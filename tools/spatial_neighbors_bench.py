"""The spatial neighbour graph at Xenium / MERFISH / Stereo-seq size: tgb200_spatial_knn / tgb200_spatial_radius and the
whole `spatial_neighbors`, against scipy's cKDTree on the host (squidpy's own query is sklearn's tree, on one core).

For each workload:
  * device time: the C entry point on device-resident coordinates and outputs, CUDA events around it, after a warm-up,
    median of --reps (grid build, search and the device-to-device copies of the call);
  * the host-to-device copy of the coordinates and the device-to-host copy of the result, CUDA events, on their own;
  * the whole `spatial_neighbors` wall time, split into the device calls as `spatial_neighbors` makes them (host
    coordinates in, host arrays out) and the numpy / scipy assembly around them;
  * cKDTree build + query on the host with workers=1 and workers=-1 (k + 1 nearest, or query_ball_point for the
    radius), and whether its neighbours agree with the device's (indices where the data has no ties, distances always).

Workloads: 1M and 4M uniform 2-D points with k = 6; a 1M-spot Visium-like hexagonal grid in grid mode (an exact lattice,
so the k-th place has ties); radius mode at about 10 neighbours per point on 1M uniform points; and --skewed-n points
with half of them in a 1e-6 box (one cell holds that half, so its queries scan it whole).  The card's name and power
limit are read in the same run.

    python tools/spatial_neighbors_bench.py [--reps 3] [--skewed-n 200000] [--out results.json]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np
import pandas as pd
import torch
from scipy.spatial import cKDTree

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tangram_b200 as tg  # noqa: E402
from tangram_b200 import MiniAnnData, _lib  # noqa: E402
from rank_genes_bench import smi  # noqa: E402

snb = sys.modules["tangram_b200.spatial_neighbors"]


def events_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def device_split(C, k=None, r=None, reps=3):
    """ms of: the H2D copy of C, the device call on device buffers, the D2H copy of its output."""
    n, dim = C.shape
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib = _lib.load()
    Cd = torch.from_numpy(C).cuda()
    res = {"h2d_ms": events_ms(lambda: torch.from_numpy(C).to("cuda", non_blocking=False), reps)}
    if k is not None:
        idx = torch.empty((n, k), dtype=torch.int32, device="cuda")
        dst = torch.empty((n, k), dtype=torch.float64, device="cuda")
        call = lambda: _lib.check(lib.tgb200_spatial_knn(_lib.ptr(Cd), n, dim, k, _lib.ptr(idx), _lib.ptr(dst), 0,  # noqa: E731
                                                         stream))
        res["search_ms"] = events_ms(call, reps)
    else:
        ip = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        _lib.check(lib.tgb200_spatial_radius(_lib.ptr(Cd), n, dim, r, _lib.ptr(ip), None, None, 0, 0, stream))
        nnz = int(ip[-1])
        idx = torch.empty(nnz, dtype=torch.int32, device="cuda")
        dst = torch.empty(nnz, dtype=torch.float64, device="cuda")
        count = lambda: _lib.check(lib.tgb200_spatial_radius(_lib.ptr(Cd), n, dim, r, _lib.ptr(ip), None, None, 0, 0,  # noqa: E731
                                                             stream))
        fill = lambda: _lib.check(lib.tgb200_spatial_radius(_lib.ptr(Cd), n, dim, r, _lib.ptr(ip), _lib.ptr(idx),  # noqa: E731
                                                            _lib.ptr(dst), nnz, 0, stream))
        res["search_count_call_ms"] = events_ms(count, reps)
        res["search_ms"] = events_ms(fill, reps)
        res["nnz"] = nnz
    res["d2h_ms"] = events_ms(lambda: (idx.cpu(), dst.cpu()), reps)
    return res


def api_split(C, reps=3, **kw):
    """Wall seconds of the whole spatial_neighbors on a MiniAnnData, and of its device calls within it."""
    inner = {"t": 0.0}
    orig = {name: getattr(snb, name) for name in ("_knn", "_radius")}

    def timed(f):
        def g(*a, **k):
            t = time.perf_counter()
            out = f(*a, **k)
            inner["t"] += time.perf_counter() - t
            return out
        return g
    for name, f in orig.items():
        setattr(snb, name, timed(f))
    try:
        ad = MiniAnnData(X=np.zeros((C.shape[0], 1), np.float32), obsm={"spatial": C},
                         obs=pd.DataFrame(index=pd.RangeIndex(C.shape[0]).astype(str)))
        tg.spatial_neighbors(ad, **kw)                                                  # warm-up
        walls, inners = [], []
        for _ in range(reps):
            inner["t"] = 0.0
            t = time.perf_counter()
            tg.spatial_neighbors(ad, **kw)
            walls.append(time.perf_counter() - t)
            inners.append(inner["t"])
    finally:
        for name, f in orig.items():
            setattr(snb, name, f)
    w, i = float(np.median(walls)), float(np.median(inners))
    return {"wall_s": w, "device_calls_s": i, "assembly_s": w - i}, ad


def ckdtree_knn(C, k, workers):
    t = time.perf_counter()
    d, i = cKDTree(C).query(C, k=k + 1, workers=workers)
    return time.perf_counter() - t, d, i


def agree_knn(C, k, idx, dst):
    """Compare the device's k nearest with cKDTree's: distances per row always, indices (as sets) too."""
    _, d, i = ckdtree_knn(C, k, -1)
    self_col = i == np.arange(len(C))[:, None]
    ok_self = bool((self_col.sum(axis=1) == 1).all())
    if ok_self:
        wi, wd = i[~self_col].reshape(-1, k), d[~self_col].reshape(-1, k)
    else:                                          # coincident points: the tree may return another point first
        wi, wd = i[:, 1:], d[:, 1:]
    wd_sorted = np.sort(wd, axis=1)
    d_ok = bool(np.allclose(np.sort(dst, axis=1), wd_sorted, rtol=1e-12, atol=0))
    i_ok = bool(np.array_equal(idx, np.sort(wi, axis=1)))
    return {"distances_agree": d_ok, "indices_agree": i_ok}


def workload_knn(name, C, k, reps, grid=False):
    res = {"workload": name, "n": int(C.shape[0]), "k": k}
    res.update(device_split(C, k=k, reps=reps))
    kw = dict(coord_type="grid", n_neighs=k) if grid else dict(coord_type="generic", n_neighs=k)
    api, _ = api_split(C, reps=reps, **kw)
    res.update({f"api_{a}": b for a, b in api.items()})
    for w in (1, -1):
        res[f"ckdtree_workers{w}_s"] = ckdtree_knn(C, k, w)[0]
    idx, dst = snb._knn(C, k)
    res.update(agree_knn(C, k, idx, dst))
    return res


def workload_radius(name, C, r, reps):
    res = {"workload": name, "n": int(C.shape[0]), "radius": r}
    res.update(device_split(C, r=r, reps=reps))
    api, ad = api_split(C, reps=reps, coord_type="generic", radius=r)
    res.update({f"api_{a}": b for a, b in api.items()})
    for w in (1, -1):
        t = time.perf_counter()
        lists = cKDTree(C).query_ball_point(C, r, workers=w, return_sorted=False)
        res[f"ckdtree_workers{w}_s"] = time.perf_counter() - t
    counts = np.array([len(x) - 1 for x in lists])
    A = ad.obsp["spatial_connectivities"]
    res["neighbours_per_point"] = float(A.nnz / C.shape[0])
    rows = np.random.default_rng(0).choice(C.shape[0], 2000, replace=False)
    same = all(sorted(j for j in lists[i] if j != i) == list(A.indices[A.indptr[i]:A.indptr[i + 1]]) for i in rows)
    res["counts_agree"] = bool(np.array_equal(np.diff(A.indptr), counts))
    res["rows_agree_on_2000_sampled"] = bool(same)
    return res


def hex_grid(n_side):
    r, c = np.meshgrid(np.arange(n_side), np.arange(n_side), indexing="ij")
    return np.c_[(c + 0.5 * (r % 2)).ravel(), (r * np.sqrt(3) / 2).ravel()].astype(np.float64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--skewed-n", type=int, default=200_000)
    ap.add_argument("--out", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    rng = np.random.default_rng(0)
    out = {"card": smi("name,power.limit,clocks.max.sm"), "workloads": []}
    print("card:", out["card"], flush=True)
    n = 1_000_000
    skew = np.r_[rng.random((a.skewed_n - a.skewed_n // 2, 2)), 0.5 + 1e-6 * rng.random((a.skewed_n // 2, 2))]
    jobs = [
        lambda: workload_knn("uniform_1M_k6", rng.random((n, 2)), 6, a.reps),
        lambda: workload_knn("uniform_4M_k6", rng.random((4 * n, 2)), 6, a.reps),
        lambda: workload_knn("visium_hex_1M_grid", hex_grid(1000), 6, a.reps, grid=True),
        lambda: workload_radius("uniform_1M_radius_10", rng.random((n, 2)), float(np.sqrt(10 / (np.pi * n))), a.reps),
        lambda: workload_knn(f"skewed_{a.skewed_n}_k6", skew, 6, a.reps),
    ]
    for job in jobs:
        res = job()
        print(json.dumps(res), flush=True)
        out["workloads"].append(res)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
