"""Marker-gene statistics at atlas size: a seeded synthetic CSR of 250k cells x 32k genes with ~2k stored entries per cell
and 100 labels (up to 1M cells with --cells), through tgb200_group_stats and rank_genes_groups.

  * the device pass from host CSR (the C entry point on the canonical arrays), wall time around a device synchronise,
    after a warm-up, repeated;
  * the device pass from a device-resident dense block of --dense-rows cells (read in place);
  * the whole `rank_genes_groups` on the CSR (canonical-CSR checks, device pass, t-tests, BH, ranking);
  * a float64 numpy / scipy host restatement of the same statistics on the same inputs (one-hot products in row chunks);
  * bytes moved -- the CSR over the host link (int32 index + float32 value per entry, int64 indptr, int32 row tables)
    and the dense block from HBM -- and the achieved GB/s against the link's and HBM's bounds;
  * the card's name and power limit, read in the same run, and whether the GPU and host statistics agree.

    python tools/rank_genes_bench.py [--cells 250000] [--genes 32000] [--per-cell 2000] [--labels 100] [--reps 3]
                                     [--dense-rows 65536] [--out results/rank_genes_bench.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import pandas as pd
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tangram_b200 as tg  # noqa: E402
from tangram_b200 import MiniAnnData, _lib  # noqa: E402

PCIE_BPS = 64e9      # PCIe Gen5 x16, one direction, before protocol overhead
HBM_BPS = 3.35e12    # H100 SXM HBM3, NVIDIA's data sheet


def smi(fields):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


def synthetic(N, G, k, T, seed, chunk=8192):
    """Canonical CSR (int64 indptr, int32 indices, float32 data): per cell, columns a cumulative sum of random gaps of
    mean G / k (strictly increasing, those past G dropped), values log1p of a gamma draw; labels uniform in [0, T)."""
    rng = np.random.default_rng(seed)
    counts, idx, val = [], [], []
    for r0 in range(0, N, chunk):
        n = min(chunk, N - r0)
        cols = np.cumsum(rng.integers(1, 2 * G // k, size=(n, k), dtype=np.int32), axis=1, dtype=np.int32) - 1
        keep = cols < G
        counts.append(keep.sum(axis=1))
        idx.append(cols[keep])
        val.append(np.log1p(rng.gamma(1.5, 2.0, int(keep.sum()))).astype(np.float32))
    indptr = np.zeros(N + 1, np.int64)
    np.cumsum(np.concatenate(counts), out=indptr[1:])
    return indptr, np.concatenate(idx), np.concatenate(val), rng.integers(0, T, N).astype(np.int32)


def device_pass(lab, T, G, *, csr=None, X=None):
    """The bare tgb200_group_stats call -> (sum, sumsq, nnz); synchronous on the current stream."""
    s, q, n = np.empty((T, G)), np.empty((T, G)), np.empty((T, G), np.int64)
    if csr is not None:
        ip, ix, dv = csr
        x = (None, 0, _lib.ptr(ip), _lib.ptr(ix), _lib.ptr(dv), int(ix.shape[0]))
    else:
        x = (_lib.ptr(X), X.stride(0), None, None, None, 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream(0).cuda_stream)
    _lib.check(_lib.load().tgb200_group_stats(*x, len(lab), G, _lib.ptr(lab), T, _lib.ptr(s), _lib.ptr(q), _lib.ptr(n),
                                              0, 0, stream))
    return s, q, n


def timed(fn, reps):
    fn()                                          # warm-up
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts)), float(min(ts))


def host_stats(indptr, indices, data, lab, T, G, chunk=16384):
    """float64 sums, sums of squares and nonzero counts per label, one-hot products over row chunks."""
    S, Q, NZ = np.zeros((T, G)), np.zeros((T, G)), np.zeros((T, G))
    N = len(lab)
    for r0 in range(0, N, chunk):
        r1 = min(N, r0 + chunk)
        e0, e1 = indptr[r0], indptr[r1]
        X = sp.csr_matrix((data[e0:e1].astype(np.float64), indices[e0:e1], indptr[r0:r1 + 1] - e0), shape=(r1 - r0, G))
        H = sp.csr_matrix((np.ones(r1 - r0), (lab[r0:r1], np.arange(r1 - r0))), shape=(T, r1 - r0))
        S += (H @ X).toarray()
        Q += (H @ X.multiply(X)).toarray()
        X.data = (X.data != 0).astype(np.float64)
        NZ += (H @ X).toarray()
    return S, Q, NZ.astype(np.int64)


def rel_err(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=250000)
    ap.add_argument("--genes", type=int, default=32000)
    ap.add_argument("--per-cell", type=int, default=2000)
    ap.add_argument("--labels", type=int, default=100)
    ap.add_argument("--dense-rows", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("rank_genes_bench needs a CUDA device")
    N, G, T = a.cells, a.genes, a.labels
    res = {"card": smi("name,power.limit,clocks.max.sm"), "cells": N, "genes": G, "labels": T}
    t0 = time.perf_counter()
    indptr, indices, data, lab = synthetic(N, G, a.per_cell, T, a.seed)
    res["generate_s"] = time.perf_counter() - t0
    nnz = int(indices.shape[0])
    res["nnz"] = nnz
    link_bytes = 8 * nnz + 8 * (N + 1) + 4 * N
    res["csr_link_bytes"] = link_bytes

    gpu, med, best = timed(lambda: device_pass(lab, T, G, csr=(indptr, indices, data)), a.reps)
    res.update(csr_pass_s_median=med, csr_pass_s_min=best, csr_pass_GBps=link_bytes / med / 1e9,
               csr_pass_of_pcie=link_bytes / med / PCIE_BPS)

    D = min(a.dense_rows, N)
    Xd = torch.from_numpy(sp.csr_matrix((data[:indptr[D]], indices[:indptr[D]], indptr[:D + 1]), shape=(D, G))
                          .toarray()).to("cuda:0")
    dense_bytes = 4 * D * G
    dense, med, best = timed(lambda: device_pass(lab[:D], T, G, X=Xd), a.reps)
    res.update(dense_rows=D, dense_pass_s_median=med, dense_pass_s_min=best, dense_pass_GBps=dense_bytes / med / 1e9,
               dense_pass_of_hbm=dense_bytes / med / HBM_BPS)
    sub = device_pass(lab[:D], T, G, csr=(indptr[:D + 1], indices[:indptr[D]], data[:indptr[D]]))
    res["dense_equals_csr_bits"] = all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(dense, sub))
    del Xd
    torch.cuda.empty_cache()

    X = sp.csr_matrix((data, indices, indptr), shape=(N, G))
    names = [f"type{t:03d}" for t in range(T)]
    ad = MiniAnnData(X=X, obs=pd.DataFrame({"ct": pd.Categorical.from_codes(lab, names)}, index=np.arange(N).astype(str)),
                     var=pd.DataFrame(index=[f"g{k}" for k in range(G)]))
    _, med, best = timed(lambda: tg.rank_genes_groups(ad, "ct", n_genes=100), a.reps)
    res.update(rank_genes_groups_s_median=med, rank_genes_groups_s_min=best)

    t0 = time.perf_counter()
    host = host_stats(indptr, indices, data, lab, T, G)
    res["host_f64_stats_s"] = time.perf_counter() - t0
    res["agree_sum_rel"] = rel_err(gpu[0], host[0])
    res["agree_sumsq_rel"] = rel_err(gpu[1], host[1])
    res["agree_nnz_exact"] = bool(np.array_equal(gpu[2], host[2]))
    res["agree"] = res["agree_sum_rel"] < 1e-12 and res["agree_sumsq_rel"] < 1e-12 and res["agree_nnz_exact"]
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
