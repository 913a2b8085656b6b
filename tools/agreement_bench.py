"""The tuner's trial at C3 (100k cells x 10k voxels, R = 3 runs): one tgb200_agreement pass timed with CUDA events after
warm-up (bytes read, achieved GB/s against the H100 SXM data-sheet 3.35 TB/s), the wall time of
train_multiple_Mapper split into training, projection and scoring, and -- for scale -- the same three metrics evaluated
with numpy on this machine's host the way the reference evaluates them (float64 one-hot cube for the votes,
np.corrcoef on the flattened cube), at the largest size from a fixed ladder that fits in host memory.

    python tools/agreement_bench.py [--epochs 100] [--out results/agreement_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.stats
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.tangram_oracle import synthetic_inputs  # noqa: E402
from tangram_b200 import mapping_parameter_tuning as mpt  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def time_agreement(cube, reps, **kw):
    mpt.agreement(cube, **kw)                                   # warm-up (module load, first-touch)
    mpt.agreement(cube, **kw)
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        mpt.agreement(cube, **kw)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(np.min(ms))


def host_metrics(cube):
    """The three metrics in numpy on the host, the reference's way (float64 one-hot votes, np.corrcoef)."""
    R, N, V = cube.shape
    t = {}
    t0 = time.perf_counter()
    np.corrcoef(cube.reshape(R, -1))[np.tril_indices(R, -1)]
    t["pearson_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    onehot = np.zeros(cube.shape)
    votes = cube.argmax(axis=2)
    for r in range(R):
        onehot[r, np.arange(N), votes[r]] = 1
    scipy.stats.entropy(onehot.mean(axis=0), axis=1) / np.log(V)
    del onehot
    t["vote_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    scipy.stats.entropy(cube.mean(axis=0), axis=1) / np.log(V)
    t["consensus_s"] = time.perf_counter() - t0
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    N, V, R = 100_000, 10_000, 3
    res = {"card": card(), "shape": [R, N, V]}

    g = torch.Generator(device="cuda").manual_seed(1)
    cube = torch.empty((R, N, V), device="cuda")
    for r in range(R):
        cube[r] = torch.softmax(torch.randn((N, V), device="cuda", generator=g) * 4, dim=1)
    nbytes = 4.0 * R * N * V
    for label, kw in (("all_three", dict(vote=True, consensus=True)), ("pearson_only", {})):
        med, best = time_agreement(cube, a.reps, **kw)
        res[f"agreement_{label}_ms_median"] = med
        res[f"agreement_{label}_ms_min"] = best
        res[f"agreement_{label}_GBps"] = nbytes / (med * 1e-3) / 1e9
        res[f"agreement_{label}_of_peak"] = nbytes / (med * 1e-3) / PEAK_BPS
    res["agreement_bytes_read"] = nbytes
    del cube
    torch.cuda.empty_cache()

    inp = synthetic_inputs(N, V, a.genes, seed=3)
    K = a.genes
    data = [inp["S"], inp["G"], None, inp["d"], "cuda:0", None, None, None, None, None,
            np.arange(0, K - K // 10), np.arange(K - K // 10, K)]
    np.random.seed(0)
    det = {}
    t0 = time.perf_counter()
    metrics = mpt.train_multiple_Mapper({"num_epochs": a.epochs, "lambda_d": 1.0}, data, details=det)
    res["trial_epochs"] = a.epochs
    res["trial_wall_s"] = time.perf_counter() - t0
    res["trial_train_s"], res["trial_project_s"], res["trial_score_s"] = det["train_s"], det["project_s"], det["score_s"]
    res["trial_metrics"] = metrics
    del det
    torch.cuda.empty_cache()

    avail = os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_AVPHYS_PAGES")
    res["host_avail_GB"] = avail / 1e9
    for n in (100_000, 50_000, 25_000, 10_000, 2_000):
        if 40.0 * R * n * V < 0.6 * avail:          # float32 cube + float64 one-hot / corrcoef copies
            rng = np.random.default_rng(2)
            x = rng.standard_normal((R, n, V), dtype=np.float32) * 4
            x = np.exp(x - x.max(axis=2, keepdims=True))
            x /= x.sum(axis=2, keepdims=True)
            res["host_numpy_shape"] = [R, n, V]
            res["host_numpy"] = host_metrics(x)
            break
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
