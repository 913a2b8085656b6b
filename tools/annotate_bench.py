"""Annotation transfer at C3 (100k cells x 10k spots, T = 32 labels): one tgb200_annotate pass timed with CUDA events
after warm-up (sums only, argmax only, both; bytes read and achieved GB/s against the H100 SXM data-sheet 3.35 TB/s),
end-to-end project_cell_annotations and count_cell_annotations from a host adata_map.X (the upload included), and -- for
scale -- the reference's formulas on this machine's host (the int64 one-hot matmul, which numpy runs in float64, and
np.argmax plus the per-cell pandas loop), at the largest size from a fixed ladder that fits in host memory.

    python tools/annotate_bench.py [--reps 20] [--out results/annotate_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tangram_b200 import MiniAnnData, utils  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def time_call(fn, reps):
    fn()
    fn()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms)), float(np.min(ms))


def wall(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def adatas(X, labels):
    N, V = X.shape
    names = np.array([f"t{k}" for k in range(labels.max() + 1)], dtype=object)[labels]
    obs = pd.DataFrame({"cell_type": names}, index=[f"c{i}" for i in range(N)])
    var = pd.DataFrame(index=[f"s{j}" for j in range(V)])
    ad_map = MiniAnnData(X=X, obs=obs, var=var)
    n = np.ones(V, dtype=np.int64)
    feats = pd.DataFrame({"segmentation_label": n, "segmentation_centroid": [[(0.5, 0.5)]] * V}, index=var.index)
    ad_sp = MiniAnnData(X=np.zeros((V, 1), np.float32), obs=var.copy(),
                        obsm={"spatial": np.zeros((V, 2)), "image_features": feats})
    ad_sc = MiniAnnData(X=np.zeros((N, 1), np.float32), obs=obs.copy())
    return ad_map, ad_sp, ad_sc


def host_reference(n, V, T):
    """The reference's two hot formulas on the host: X.T @ int64 one-hot (float64 dgemm), np.argmax + iloc loop."""
    rng = np.random.default_rng(2)
    X = rng.random((n, V), dtype=np.float32)
    labels = rng.integers(0, T, n)
    one_hot = pd.DataFrame({f"t{k}": (labels == k).astype(np.int64) for k in range(T)})
    t = {}
    t0 = time.perf_counter()
    X.T @ one_hot
    t["project_matmul_s"] = time.perf_counter() - t0
    df = pd.DataFrame({f"t{k}": np.zeros(V, dtype=np.int64) for k in range(T)})
    t0 = time.perf_counter()
    vox = np.argmax(X, axis=1)
    t["argmax_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    for k, v in zip(vox, labels):
        df.iloc[k, v] += 1
    t["count_loop_s"] = time.perf_counter() - t0
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    N, V, T = 100_000, 10_000, 32
    res = {"card": card(), "shape": [N, V], "labels": T}
    g = torch.Generator(device="cuda").manual_seed(1)
    P = torch.softmax(torch.randn((N, V), device="cuda", generator=g) * 4, dim=1)
    labels = torch.randint(0, T, (N,), device="cuda", generator=g).int().cpu().numpy()
    nbytes = 4.0 * N * V
    res["bytes_read"] = nbytes
    for name, kw in (("sums", {}), ("argmax", dict(sums=False, argmax=True)), ("both", dict(argmax=True))):
        med, best = time_call(lambda: utils.annotate(P, labels, T, **kw), a.reps)
        res[f"annotate_{name}_ms_median"] = med
        res[f"annotate_{name}_ms_min"] = best
        res[f"annotate_{name}_GBps"] = nbytes / (med * 1e-3) / 1e9
        res[f"annotate_{name}_of_peak"] = nbytes / (med * 1e-3) / PEAK_BPS
    res["hbm_floor_ms"] = nbytes / PEAK_BPS * 1e3

    X = P.cpu().numpy()
    del P
    torch.cuda.empty_cache()
    ad_map, ad_sp, ad_sc = adatas(X, labels)
    utils.create_segment_cell_df(ad_sp)
    res["e2e_project_cell_annotations_s"] = wall(lambda: utils.project_cell_annotations(ad_map, ad_sp))
    res["e2e_count_cell_annotations_s"] = wall(lambda: utils.count_cell_annotations(ad_map, ad_sc, ad_sp))
    del ad_map, X

    avail = os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_AVPHYS_PAGES")
    res["host_avail_GB"] = avail / 1e9
    res["host_threads"] = torch.get_num_threads()
    for n in (100_000, 50_000, 25_000, 10_000):
        if 16.0 * n * V < 0.6 * avail:             # float32 mapping + its float64 upcast in the matmul
            res["host_reference_shape"] = [n, V]
            res["host_reference"] = host_reference(n, V, T)
            break
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
