"""Gene projection and annotation transfer from a cell-sharded mapping, against the gather route, on W GPUs.

Launch under torchrun, one process per GPU:

    python -m torch.distributed.run --nproc-per-node=W tools/transfer_sharded_bench.py [--cells 100000] [--spots 10000]
        [--genes 20000] [--density 0.07] [--labels 32] [--reps 3] [--out results.json]

Inputs, drawn from seeds on the GPU: an N x V mapping (rows normalised to 1; each rank draws only its rows
shard_rows(N, rank, W)), T labels, and a CSR adata_sc.X of N x n_genes at the given density (the input of
tools/project_bench.py), the same on every rank.  Timed with the host clock around calls that end on host arrays, after a
barrier, one warm-up call each, the median of --reps:

  * sharded: project_genes, project_cell_annotations, cell_type_mapping, count_cell_annotations with process_group=
    (per rank, and the slowest rank), and on its own the reduction project_genes ends with (_sum_over_group of one
    spots x genes float32 array);
  * gather route: the gather of map_cells_to_space(gather=True) (every rank's block to rank 0 by gather_object), then the
    four calls without a group on rank 0.

Both routes' results are compared (largest relative difference of the sums and projection, counts equal).  The card's
name and power limit are read in the same run.  Prints one JSON object from rank 0; with --out also writes it there.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import scipy.sparse as sp
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tangram_b200 import MiniAnnData, utils  # noqa: E402
from tangram_b200 import mapping_utils as mu  # noqa: E402
from tangram_b200.sharded import shard_rows  # noqa: E402

BLOCK = 5000                                  # rows drawn per seeded block: a rank's rows do not depend on W


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def mapping_rows(r0, r1, V, dev):
    """Rows [r0, r1) of the seeded N x V mapping, as a float32 host array."""
    out = np.empty((r1 - r0, V), dtype=np.float32)
    for b in range(r0 // BLOCK, -(-r1 // BLOCK)):
        g = torch.Generator(device=dev).manual_seed(1000 + b)
        M = torch.rand((BLOCK, V), generator=g, device=dev)
        M /= M.sum(dim=1, keepdim=True)
        lo, hi = max(r0, b * BLOCK), min(r1, (b + 1) * BLOCK)
        out[lo - r0:hi - r0] = M[lo - b * BLOCK:hi - b * BLOCK].cpu().numpy()
    return out


def expression(N, K, density, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    idx, val, counts = [], [], []
    for r0 in range(0, N, 10_000):
        n = min(10_000, N - r0)
        rc = (torch.rand((n, K), generator=g, device=dev) < density).nonzero()
        counts.append(torch.bincount(rc[:, 0], minlength=n).cpu())
        idx.append(rc[:, 1].int().cpu())
        val.append(torch.rand(rc.shape[0], generator=g, device=dev).cpu())
        del rc
    torch.cuda.empty_cache()
    indptr = np.concatenate([[0], np.cumsum(torch.cat(counts).numpy())]).astype(np.int64)
    return sp.csr_matrix((torch.cat(val).numpy(), torch.cat(idx).numpy(), indptr), shape=(N, K))


def spots_adata(V, rng):
    n = rng.integers(0, 4, V)
    n[0] = 2
    names = [f"v{j}" for j in range(V)]
    features = pd.DataFrame({"segmentation_label": n,
                             "segmentation_centroid": [[(float(rng.random()), float(rng.random()))] * k for k in n]},
                            index=names)
    ad_sp = MiniAnnData(X=np.zeros((V, 1), np.float32), obs=pd.DataFrame(index=names),
                        obsm={"image_features": features, "spatial": rng.random((V, 2))})
    utils.create_segment_cell_df(ad_sp)
    return ad_sp


def timed(fn, reps, group):
    """fn() once to warm up, then `reps` timed calls (host clock, after a barrier) -> (median seconds, last result)."""
    out = fn()
    ts = []
    for _ in range(reps):
        if group is not None:
            dist.barrier(group=group)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def four_calls(ad_map, ad_sc, ad_ge, ad_sp, pg, reps):
    """-> ({call: median seconds}, {call: result}) of the four transfer calls."""
    t, res = {}, {}
    t["project_genes"], ge = timed(lambda: utils.project_genes(ad_map, ad_ge, process_group=pg), reps, pg)
    res["project_genes"] = np.asarray(ge.X)
    if pg is not None:
        # the reduction project_genes ends with, on its own: one (spots x genes) float32 array through _sum_over_group
        t["project_genes_sum_over_group"], _ = timed(lambda: mu._sum_over_group(res["project_genes"], None, pg),
                                                     reps, pg)

    def pred():
        utils.project_cell_annotations(ad_map, ad_sp, process_group=pg)
        return ad_sp.obsm["tangram_ct_pred"].to_numpy()

    def ct_map():
        utils.cell_type_mapping(ad_map, cell_types_key="cell_type", process_group=pg)
        return ad_map.varm["ct_map"].to_numpy()

    def count():
        utils.count_cell_annotations(ad_map, ad_sc, ad_sp, process_group=pg)
        return ad_sp.obsm["tangram_ct_count"].iloc[:, 4:].to_numpy(np.int64)

    for name, fn in (("project_cell_annotations", pred), ("cell_type_mapping", ct_map), ("count_cell_annotations", count)):
        t[name], res[name] = timed(fn, reps, pg)
    return t, res


def rel_max(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    ok = ~np.isnan(b)
    return float(np.max(np.abs(a[ok] - b[ok]) / np.maximum(np.abs(b[ok]), 1e-300)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=100_000)
    ap.add_argument("--spots", type=int, default=10_000)
    ap.add_argument("--genes", type=int, default=20_000)
    ap.add_argument("--density", type=float, default=0.07)
    ap.add_argument("--labels", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dev = f"cuda:{rank}"
    dist.init_process_group("nccl", device_id=torch.device(dev))
    pg = dist.group.WORLD
    N, V, K, T = a.cells, a.spots, a.genes, a.labels
    r0, r1 = shard_rows(N, rank, world)
    rng = np.random.default_rng(7)
    cells = [f"c{i}" for i in range(N)]
    labels = np.array([f"L{t:02d}" for t in range(T)], dtype=object)[rng.integers(0, T, N)]
    obs = pd.DataFrame({"cell_type": labels}, index=cells)
    ad_sp = spots_adata(V, rng)
    genes = [f"Gene{k}" for k in range(K)]
    X = expression(N, K, a.density, dev)
    ad_sc = MiniAnnData(X=np.zeros((N, 1), np.float32), obs=obs[["cell_type"]].copy())
    ad_ge = MiniAnnData(X=X, obs=pd.DataFrame(index=cells), var=pd.DataFrame(index=genes))
    uns = {"train_genes_df": pd.DataFrame(index=[g.lower() for g in genes[:200]]), "shard_rows": (r0, r1)}
    ad_map = MiniAnnData(X=mapping_rows(r0, r1, V, dev), obs=obs.iloc[r0:r1].copy(),
                         var=pd.DataFrame(index=ad_sp.obs.index), uns=uns)

    t_sharded, sharded = four_calls(ad_map, ad_sc, ad_ge, ad_sp, pg, a.reps)
    per_rank = [None] * world
    dist.all_gather_object(per_rank, t_sharded)

    dist.barrier()
    t0 = time.perf_counter()
    full = mu._gather_mapping(ad_map, obs.copy(), pg, dev)
    t_gather = time.perf_counter() - t0
    res = None
    if rank == 0:
        t_single, single = four_calls(full, ad_sc, ad_ge, ad_sp, None, a.reps)
        slowest = {k: max(r[k] for r in per_rank) for k in t_sharded}
        calls = [k for k in slowest if k != "project_genes_sum_over_group"]        # that one is inside project_genes
        res = {"card": card(), "world": world, "shape": {"cells": N, "spots": V, "genes": K, "labels": T,
                                                         "density": X.nnz / (N * K), "reps": a.reps},
               "sharded_s": {"per_rank": per_rank, "slowest_rank": slowest, "total": sum(slowest[k] for k in calls)},
               "gather_route_s": {"gather": t_gather, **t_single, "total": t_gather + sum(t_single.values())},
               "agreement": {"project_genes_max_rel": rel_max(sharded["project_genes"], single["project_genes"]),
                             "ct_pred_max_rel": rel_max(sharded["project_cell_annotations"],
                                                        single["project_cell_annotations"]),
                             "ct_map_max_abs": float(np.nanmax(np.abs(sharded["cell_type_mapping"]
                                                                      - single["cell_type_mapping"]))),
                             "counts_equal": bool(np.array_equal(sharded["count_cell_annotations"],
                                                                 single["count_cell_annotations"]))}}
        line = json.dumps(res)
        print(line, flush=True)
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                f.write(line + "\n")
    del full
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
