"""Gene cross-validation wall time, per fold and in total, on two workloads:
  loo_clusters  clusters mode, leave-one-out: 18 clusters x 9852 spots x 249 genes (synthetic, seeded; the shape of the
                reference's test data), one pseudo-cell per cluster
  cells_10fold  cells mode, 10-fold: 20000 cells x 5000 spots x 500 genes (synthetic, seeded)
and three ways to run it:
  (a) cross_val: every fold on one handle (gene mask, device redraw, test genes projected on the device)
  (b) the naive loop: map_cells_to_space(cv_train_genes=...) + project_genes + compare_spatial_geneexp per fold
  (c) the unmodified reference Mapper(device="cuda") per fold (oracle/_ref), with the reference's host projection
(b) and (c) time their first few folds and scale to all folds.  The card's name and power limit are read in the same
call.

    python tools/cv_bench.py [--epochs 300] [--out results/cv_bench.json]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import tangram_b200 as tg  # noqa: E402
from oracle.tangram_oracle import synthetic_inputs  # noqa: E402

WORKLOADS = {
    # name: cells, spots, genes, mode, cv_mode, folds timed for (b), for (c)
    "loo_clusters": (18, 9852, 249, "clusters", "loo", 20, 5),
    "cells_10fold": (20000, 5000, 500, "cells", "10fold", 3, 2),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def adatas(N, V, K, seed=0):
    inp = synthetic_inputs(N, V, K, seed=seed)
    genes = [f"g{k:04d}" for k in range(K)]
    ad_sc = tg.MiniAnnData(X=sp.csr_matrix(inp["S"]),
                           obs=pd.DataFrame({"cl": [f"c{i}" for i in range(N)]}, index=[f"c{i}" for i in range(N)]),
                           var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=inp["G"], obs=pd.DataFrame(index=[f"s{j}" for j in range(V)]), var=pd.DataFrame(index=list(genes)))
    tg.pp_adatas(ad_sc, ad_sp)
    for ad in (ad_sc, ad_sp):
        ad.uns["training_genes"] = sorted(ad.uns["training_genes"])
    return ad_sc, ad_sp


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run(name, epochs):
    N, V, K, mode, cv_mode, nb, nc = WORKLOADS[name]
    ad_sc, ad_sp = adatas(N, V, K)
    cl = "cl" if mode == "clusters" else None
    folds = list(tg.cv_data_gen(ad_sc, ad_sp, cv_mode))
    res = {"shape": [N, V, K], "mode": mode, "cv_mode": cv_mode, "folds": len(folds), "epochs": epochs}

    with contextlib.redirect_stdout(io.StringIO()):
        dt, cv = timed(lambda: tg.cross_val(ad_sc, ad_sp, cluster_label=cl, mode=mode, cv_mode=cv_mode,
                                            num_epochs=epochs, random_state=1))
    res["a_cross_val"] = {"total_s": dt, "per_fold_s": dt / len(folds), "avg_test_score": float(cv["avg_test_score"])}

    ref_sc = tg.adata_to_cluster_expression(ad_sc, cl, True) if cl else ad_sc
    t = []
    for train, test in folds[:nb]:
        def fold():
            m = tg.map_cells_to_space(ad_sc, ad_sp, cv_train_genes=train, mode=mode, cluster_label=cl, num_epochs=epochs,
                                      random_state=1, verbose=False, density_prior=None)
            ge = tg.project_genes(m, ad_sc[:, train + test], cluster_label=cl)
            return tg.compare_spatial_geneexp(ge, ad_sp, ref_sc, train + test)
        t.append(timed(fold)[0])
    res["b_map_cells_to_space_loop"] = {"folds_timed": nb, "per_fold_s": float(np.mean(t)),
                                        "total_s_scaled": float(np.mean(t)) * len(folds)}

    from oracle import build_ref
    if build_ref.source() is None:
        res["c_reference_gpu"] = {"skipped": "no copy of the reference (oracle/build_ref.py found no Tangram checkout)"}
        return res
    ref = build_ref.load()
    genes = list(ad_sc.uns["training_genes"])
    agg = ref_sc if cl else ad_sc
    S_all = np.asarray(agg[:, genes].X.toarray() if hasattr(agg.X, "toarray") else agg[:, genes].X, dtype=np.float32)
    G_all = np.asarray(ad_sp[:, genes].X, dtype=np.float32)
    d = np.asarray(ad_sp.obs["uniform_density"], dtype=np.float32)
    col = {g: k for k, g in enumerate(genes)}
    t = []
    for train, test in folds[:nc]:
        tr, te = [col[g] for g in train], [col[g] for g in test]

        def fold():
            kw = dict(S=S_all[:, tr], G=G_all[:, tr], device="cuda", random_state=1)
            if cl:
                kw.update(d=d, lambda_d=1, d_source=np.asarray(agg.obs["cluster_density"], dtype=np.float32))
            with contextlib.redirect_stdout(io.StringIO()):
                mapping, _ = ref.Mapper(**kw).train(num_epochs=epochs, learning_rate=0.1, print_each=None)
            pred = mapping.T @ S_all[:, te]                                  # project_genes' host GEMM, test genes only
            g = G_all[:, te]
            return (pred * g).sum(0) / (np.linalg.norm(pred, axis=0) * np.linalg.norm(g, axis=0))
        t.append(timed(fold)[0])
    res["c_reference_gpu"] = {"folds_timed": nc, "per_fold_s": float(np.mean(t)), "total_s_scaled": float(np.mean(t)) * len(folds),
                              "source": build_ref.source()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=300)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "torch": torch.__version__, "workloads": {}}
    tg.cross_val  # noqa: B018  (import check before the clock starts)
    for name in a.workloads.split(","):
        out["workloads"][name] = run(name, a.epochs)
        print(json.dumps({name: out["workloads"][name]}), flush=True)
    out["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
