"""Highly-variable-gene statistics at atlas size: rank_genes_bench's seeded synthetic CSR of 250k cells x 32k genes with
~2k stored entries per cell, here with 8 batches, through tgb200_group_stats_expm1 and highly_variable_genes.

  * the expm1 pass from host CSR (the C entry point on the canonical arrays), wall time around a device synchronise,
    after a warm-up, median and minimum of --reps;
  * the expm1 pass and the plain (identity) pass from a device-resident dense block of --dense-rows cells (read in
    place), so the cost of the fp64 expm1 shows against the same bytes;
  * the whole `highly_variable_genes(n_top_genes=4000, batch_key=...)` on the CSR (seurat);
  * a float64 numpy / scipy host restatement of the same statistics (expm1 on the CSR data, per-batch column sums);
  * bytes moved -- the CSR over the host link and the dense block from HBM -- and GB/s against the link's and HBM's
    bounds, the card's name and power limit, read in the same run, and whether the GPU and host statistics agree.

    python tools/hvg_bench.py [--cells 250000] [--genes 32000] [--per-cell 2000] [--batches 8] [--reps 3]
                              [--dense-rows 65536] [--out results/hvg_bench.json]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import pandas as pd
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tangram_b200 as tg  # noqa: E402
from tangram_b200 import MiniAnnData, _lib  # noqa: E402
from rank_genes_bench import HBM_BPS, PCIE_BPS, rel_err, smi, synthetic, timed  # noqa: E402


def device_pass(lab, T, G, *, csr=None, X=None, scale=1.0):
    """The bare tgb200_group_stats_expm1 call (tgb200_group_stats with scale=None) -> (sum, sumsq, nnz)."""
    s, q, n = np.empty((T, G)), np.empty((T, G)), np.empty((T, G), np.int64)
    if csr is not None:
        ip, ix, dv = csr
        x = (None, 0, _lib.ptr(ip), _lib.ptr(ix), _lib.ptr(dv), int(ix.shape[0]))
    else:
        x = (_lib.ptr(X), X.stride(0), None, None, None, 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream(0).cuda_stream)
    args = (*x, len(lab), G, _lib.ptr(lab), T, _lib.ptr(s), _lib.ptr(q), _lib.ptr(n), 0, 0, stream)
    lib = _lib.load()
    _lib.check(lib.tgb200_group_stats(*args) if scale is None else lib.tgb200_group_stats_expm1(*args, scale))
    return s, q, n


def host_stats(indptr, indices, data, lab, T, G, chunk=16384):
    """float64 sums of expm1(x) and of its square and counts of x != 0 per batch: column sums over row chunks."""
    S, Q, NZ = np.zeros((T, G)), np.zeros((T, G)), np.zeros((T, G), np.int64)
    N = len(lab)
    for r0 in range(0, N, chunk):
        r1 = min(N, r0 + chunk)
        e0, e1 = indptr[r0], indptr[r1]
        x = data[e0:e1].astype(np.float64)
        y = np.expm1(x)
        rows = lab[np.repeat(np.arange(r0, r1), np.diff(indptr[r0:r1 + 1]))]
        cols = indices[e0:e1]
        for t in range(T):
            m = rows == t
            S[t] += np.bincount(cols[m], weights=y[m], minlength=G)
            Q[t] += np.bincount(cols[m], weights=y[m] * y[m], minlength=G)
            NZ[t] += np.bincount(cols[m], weights=x[m] != 0, minlength=G).astype(np.int64)
    return S, Q, NZ


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=250000)
    ap.add_argument("--genes", type=int, default=32000)
    ap.add_argument("--per-cell", type=int, default=2000)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--dense-rows", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("hvg_bench needs a CUDA device")
    N, G, T = a.cells, a.genes, a.batches
    res = {"card": smi("name,power.limit,clocks.max.sm"), "cells": N, "genes": G, "batches": T}
    t0 = time.perf_counter()
    indptr, indices, data, lab = synthetic(N, G, a.per_cell, T, a.seed)
    res["generate_s"] = time.perf_counter() - t0
    nnz = int(indices.shape[0])
    res["nnz"] = nnz
    link_bytes = 8 * nnz + 8 * (N + 1) + 4 * N
    res["csr_link_bytes"] = link_bytes

    gpu, med, best = timed(lambda: device_pass(lab, T, G, csr=(indptr, indices, data)), a.reps)
    res.update(csr_expm1_pass_s_median=med, csr_expm1_pass_s_min=best, csr_expm1_pass_GBps=link_bytes / med / 1e9,
               csr_expm1_pass_of_pcie=link_bytes / med / PCIE_BPS)

    D = min(a.dense_rows, N)
    Xd = torch.from_numpy(sp.csr_matrix((data[:indptr[D]], indices[:indptr[D]], indptr[:D + 1]), shape=(D, G))
                          .toarray()).to("cuda:0")
    dense_bytes = 4 * D * G
    res.update(dense_rows=D, dense_bytes=dense_bytes)
    for name, scale in (("dense_expm1_pass", 1.0), ("dense_plain_pass", None)):
        out, med, best = timed(lambda: device_pass(lab[:D], T, G, X=Xd, scale=scale), a.reps)
        res.update({f"{name}_s_median": med, f"{name}_s_min": best, f"{name}_GBps": dense_bytes / med / 1e9,
                    f"{name}_of_hbm": dense_bytes / med / HBM_BPS, f"{name}_min_of_hbm": dense_bytes / best / HBM_BPS})
        if scale is not None:
            dense = out
    sub = device_pass(lab[:D], T, G, csr=(indptr[:D + 1], indices[:indptr[D]], data[:indptr[D]]))
    res["dense_equals_csr_bits"] = all(np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(dense, sub))
    del Xd
    torch.cuda.empty_cache()

    X = sp.csr_matrix((data, indices, indptr), shape=(N, G))
    names = [f"batch{t}" for t in range(T)]
    ad = MiniAnnData(X=X, obs=pd.DataFrame({"batch": pd.Categorical.from_codes(lab, names)},
                                           index=np.arange(N).astype(str)),
                     var=pd.DataFrame(index=[f"g{k}" for k in range(G)]))
    _, med, best = timed(lambda: tg.highly_variable_genes(ad, n_top_genes=4000, batch_key="batch"), a.reps)
    res.update(highly_variable_genes_s_median=med, highly_variable_genes_s_min=best,
               highly_variable_selected=int(ad.var["highly_variable"].sum()))

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
