"""Cost of per-epoch validation: wall time of Mapper.train(E, val_each=1) against train(E), at C2 (10k x 1k x 1k) and C3
(100k x 10k x 2k), in bf16x3 and bf16, three legs each on a fresh mapper:
  plain  train(E)
  new    train(E, val_each=1): validation inside the loop (tgb200_set_validation)
  old    the one-epoch loop train(val_each=1) ran before: run(1) + validation_terms() per epoch (written out below)
The new and old legs start from the same mapping; whether their training history, mapping and val_* values agree bit for
bit (for the sparsity-weighted score: the largest difference) is recorded beside the times.  The card's name and power limit are read in the
same call.

    python tools/val_bench.py [--epochs 300] [--shapes C2,C3] [--precisions bf16x3,bf16] [--out results/val_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.tangram_oracle import synthetic_inputs  # noqa: E402
from tangram_b200 import Mapper, _lib  # noqa: E402
from tangram_b200.mapping_optimizer import _ResultBuffer  # noqa: E402

SHAPES = {"C2": (10000, 1000, 1000), "C3": (100000, 10000, 2000)}
LR = 0.1


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def old_train(m, epochs):
    """The previous Mapper._fit with print_each=None, val_each=1: one tgb200_run per epoch, then tgb200_validation_terms."""
    e = m._engine
    e.reset_adam()
    first = e.history_len()
    result = _ResultBuffer(_lib.load(), (m.n_cells, m.n_voxels), m._cfg.device)
    try:
        vals = []
        for _ in range(epochs):
            e.run(1, LR)
            vals.append(e.validation_terms())
        hist = e.history(first, epochs)
        return e.get_mapping(result.ready()), hist, np.array(vals)
    finally:
        result.release()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def run(shape, precision, epochs):
    N, V, K = SHAPES[shape]
    inp = synthetic_inputs(N, V, K, seed=0)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, device="cuda:0", random_state=1, precision=precision)
    res = {"shape": [N, V, K], "precision": precision, "epochs": epochs}

    warm = Mapper(**{**kw, "S": inp["S"][:2048]})               # module load and the kernels' first launches
    warm.train(3, print_each=None, val_each=1)
    warm.release()

    m = Mapper(**kw)
    res["plain_s"], _ = timed(lambda: m.train(epochs, print_each=None))
    m.release()

    m = Mapper(**kw)
    res["new_s"], (P_new, _) = timed(lambda: m.train(epochs, print_each=None, val_each=1))
    hist_new = m.history_matrix
    m.release()

    m = Mapper(**kw)
    res["old_s"], (P_old, hist_old, vals) = timed(lambda: old_train(m, epochs))
    m.release()

    res["new_over_plain"] = res["new_s"] / res["plain_s"]
    res["old_over_plain"] = res["old_s"] / res["plain_s"]
    res["ms_per_validated_epoch"] = {"new": 1e3 * (res["new_s"] - res["plain_s"]) / epochs,
                                     "old": 1e3 * (res["old_s"] - res["plain_s"]) / epochs}
    nv = hist_new[:, 12:16]
    res["same_as_old"] = {
        "training_history": bool(np.array_equal(hist_new[:, :12], hist_old[:, :12], equal_nan=True)),
        "mapping": bool(np.array_equal(P_new, P_old)),
        "val_total_gene_sim_entropy": bool(np.array_equal(nv[:, [0, 1, 3]], vals[:, [0, 1, 3]])),
        "val_sparsity_max_abs_diff": float(np.max(np.abs(nv[:, 2].astype(np.float64) - vals[:, 2]))),
    }
    del P_new, P_old
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=300)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--precisions", default="bf16x3,bf16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    out = {"card": card(), "torch": torch.__version__, "runs": []}
    for shape in a.shapes.split(","):
        for prec in a.precisions.split(","):
            r = run(shape, prec, a.epochs)
            out["runs"].append(r)
            print(json.dumps(r), flush=True)
    out["card_after"] = card()
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"card": out["card"], "card_after": out["card_after"]}))


if __name__ == "__main__":
    main()
