"""project_genes' projection at full size: a 100k x 10k mapping onto a 100k x 20k CSR X at ~7 % nonzeros (the whole
transcriptome of SURVEY 8(f) N1), through `project` (tgb200_project_map).

  * wall time of `project` with the mapping on the host and on the device (CSR on the host both times), repeated, with
    the SM clock sampled by nvidia-smi while those calls run;
  * a torch.profiler run of one host-mapping call: device time of the host-to-device copies, the CSR -> bf16-planes
    kernel, the mapping's k_split3 and the contractions, and how much of the copy time runs under kernels;
  * contraction TFLOP/s on 2 N V K (the algorithm) and on the six partial products the tensor cores run (6 x that);
  * the host GEMM the device path replaces (`adata_map.X.T @ adata_sc.X.toarray()`), on this machine's host cores:
    row-sliced to `--host-rows` cells and scaled linearly to N, densification included, repeated; with the size of
    numpy's BLAS thread pool (threadpoolctl).

    python tools/project_bench.py [--reps 3] [--host-rows 4096] [--out results/project_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import scipy.sparse as sp
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tangram_b200 import utils  # noqa: E402


def smi(fields):
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


def card():
    return smi("name,power.limit,clocks.max.sm") or torch.cuda.get_device_name(0)


class ClockSampler:
    """Samples the SM clock (MHz) every `period` seconds on a host thread while the timed calls run."""

    def __init__(self, period=0.25):
        self.period, self.mhz, self._stop = period, [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            v = smi("clocks.sm")
            if v.isdigit():
                self.mhz.append(int(v))
            self._stop.wait(self.period)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()


def blas_threads():
    """The BLAS pools numpy's matmul runs on: [(library, threads)]."""
    try:
        from threadpoolctl import threadpool_info
    except ImportError:
        return None
    return [(i.get("internal_api"), i.get("num_threads")) for i in threadpool_info() if i.get("user_api") == "blas"]


def inputs(N, V, K, density):
    g = torch.Generator(device="cuda").manual_seed(0)
    M = torch.rand((N, V), generator=g, device="cuda")
    M /= M.sum(dim=1, keepdim=True)
    Mh = M.cpu().numpy()
    del M
    idx, val, counts, step = [], [], [], 10_000
    for r0 in range(0, N, step):
        n = min(step, N - r0)
        rc = (torch.rand((n, K), generator=g, device="cuda") < density).nonzero()
        counts.append(torch.bincount(rc[:, 0], minlength=n).cpu())
        idx.append(rc[:, 1].int().cpu())
        val.append(torch.rand(rc.shape[0], generator=g, device="cuda").cpu())
        del rc
    torch.cuda.empty_cache()
    indptr = np.concatenate([[0], np.cumsum(torch.cat(counts).numpy())]).astype(np.int64)
    return Mh, sp.csr_matrix((torch.cat(val).numpy(), torch.cat(idx).numpy(), indptr), shape=(N, K))


def wall(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return ts


def union(iv):
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def overlap(u1, u2):
    i = j = 0
    s = 0.0
    while i < len(u1) and j < len(u2):
        a, b = max(u1[i][0], u2[j][0]), min(u1[i][1], u2[j][1])
        s += max(0.0, b - a)
        if u1[i][1] < u2[j][1]:
            i += 1
        else:
            j += 1
    return s


def profile(fn):
    """-> device-time breakdown (ms) of one call from its CUDA activity."""
    from torch.profiler import ProfilerActivity, profile as tprof
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    groups = {"h2d": [], "csr_split3": [], "split3": [], "gemm": [], "other": []}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        iv = (e.time_range.start, e.time_range.end)
        n = e.name
        if "HtoD" in n:
            groups["h2d"].append(iv)
        elif "k_csr_split3" in n:
            groups["csr_split3"].append(iv)
        elif "k_split3" in n:
            groups["split3"].append(iv)
        elif "k_gemm_tc" in n:
            groups["gemm"].append(iv)
        else:
            groups["other"].append(iv)
    res = {f"{k}_ms": sum(b - a for a, b in v) / 1e3 for k, v in groups.items()}
    res["gemm_launches"] = len(groups["gemm"])
    kern = union(groups["csr_split3"] + groups["split3"] + groups["gemm"])
    copies = union(groups["h2d"])
    copy_ms = sum(b - a for a, b in copies) / 1e3
    res["h2d_under_kernels_ms"] = overlap(copies, kern) / 1e3
    res["h2d_overlap_fraction"] = res["h2d_under_kernels_ms"] / copy_ms if copy_ms else 0.0
    allv = union([iv for v in groups.values() for iv in v])
    res["device_span_ms"] = (allv[-1][1] - allv[0][0]) / 1e3 if allv else 0.0
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-rows", type=int, default=4096)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    N, V, K, density = 100_000, 10_000, 20_000, 0.07
    res = {"card": card(), "shape": [N, V, K]}
    Mh, X = inputs(N, V, K, density)
    res["nnz"] = int(X.nnz)
    res["density"] = X.nnz / (N * K)
    flops = 2.0 * N * V * K
    res["flops_algorithmic"] = flops

    with ClockSampler() as clk:
        res["wall_host_mapping_s"] = wall(lambda: utils.project(Mh, X), a.reps)
        Md = torch.from_numpy(Mh).cuda()
        res["wall_device_mapping_s"] = wall(lambda: utils.project(Md, X), a.reps)
    # SM clock while the timed calls ran (copies and host work included, so the low end is not the contraction's)
    res["sm_clock_mhz_during_timed_calls"] = {"samples": len(clk.mhz), "min": min(clk.mhz, default=None),
                                              "median": float(np.median(clk.mhz)) if clk.mhz else None,
                                              "max": max(clk.mhz, default=None)}
    del Md
    torch.cuda.empty_cache()
    prof = profile(lambda: utils.project(Mh, X))
    res["profile_host_mapping"] = prof
    res["gemm_TFLOPs_algorithmic"] = flops / (prof["gemm_ms"] * 1e-3) / 1e12
    res["gemm_TFLOPs_six_products"] = 6 * flops / (prof["gemm_ms"] * 1e-3) / 1e12

    n = min(a.host_rows, N)
    res["host_rows"] = n
    Xs, Ms = X[:n], np.ascontiguousarray(Mh[:n])
    Ms[:64].T @ Xs[:64].toarray()                                          # loads the BLAS library before it is queried
    res["host_blas_threads"] = blas_threads()
    ts = []
    for _ in range(a.reps):
        t0 = time.perf_counter()
        Ms.T @ Xs.toarray()
        ts.append((time.perf_counter() - t0) * N / n)
    res["host_gemm_scaled_s"] = ts
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
