"""state_memory="host" and "auto" against the resident handle: seconds per iteration at C3 (100k x 10k x 2k) in bf16 and
bf16x3 for "device", "host" and "auto" with 50 %, 75 % and 90 % of the rows forced resident (each auto time next to its
bound, the larger of the resident time and the staged rows' bytes over the probe's bidirectional bandwidth), with
whether every placement gives the same history and softmax(M) bits; the bytes the staging ring copies per iteration over the elapsed time (a
figure derived from the ring's copy sizes, not a measured link counter) next to a plain cudaMemcpyAsync bandwidth
probe (H2D, D2H, both at once); the seeded legacy draw into host state; and one run at a size that does not fit resident
(bf16x3 at 160k x 24k by default) with host state and with the unforced auto split (its R, device and pinned bytes),
only when MemAvailable and the free device memory hold it.  Prints one JSON object;
with --out also writes it there.

    python tools/state_host_bench.py [--steps 5] [--big-cells 160000] [--big-spots 24000] [--skip-big-host] [--out results.json]
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
from tangram_b200 import _lib  # noqa: E402
from tangram_b200.engine import HOST_STATE_BYTES_PER_ELEMENT, Engine, host_memory_available, plan_state  # noqa: E402

# bytes per mapping element the ring copies in one steady-state iteration (staged_rows): the update copies M, m / mb and
# v in and out; bf16x3 also runs the exact row pass every iteration, which copies M in once more.  Derived from the copy
# sizes, not measured on the link.
LINK_BYTES = {"bf16": (4 + 2 + 4, 4 + 2 + 4), "bf16x3": (4 + 4 + 4 + 4, 4 + 4 + 4)}    # (to the device, to the host)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def copy_probe(gib=2.0, reps=5):
    """GB/s of cudaMemcpyAsync between pinned host memory and the device: each direction alone, then both at once on two
    streams (the copy engines are independent)."""
    n = int(gib * 2**30) // 4
    h_src = torch.empty(n, dtype=torch.float32, pin_memory=True)
    h_dst = torch.empty(n, dtype=torch.float32, pin_memory=True)
    d_src = torch.empty(n, dtype=torch.float32, device="cuda")
    d_dst = torch.empty(n, dtype=torch.float32, device="cuda")
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps

    def both():
        with torch.cuda.stream(s1):
            d_dst.copy_(h_src, non_blocking=True)
        with torch.cuda.stream(s2):
            h_dst.copy_(d_src, non_blocking=True)

    nb = n * 4
    out = dict(bytes=nb,
               h2d_gbs=nb / timed(lambda: d_dst.copy_(h_src, non_blocking=True)) / 1e9,
               d2h_gbs=nb / timed(lambda: h_dst.copy_(d_src, non_blocking=True)) / 1e9)
    out["bidirectional_gbs"] = 2 * nb / timed(both) / 1e9
    del h_src, h_dst, d_src, d_dst
    torch.cuda.empty_cache()
    return out


def make_engine(N, V, K, precision, state_memory, seed=0):
    rng = np.random.default_rng(seed)
    S = rng.random((N, K), dtype=np.float32)
    G = rng.random((V, K), dtype=np.float32)
    e = Engine(N, V, K, device=0, precision=precision, state_memory=state_memory, lambda_d=1.0)
    e.set_expression(S, G)
    e.set_density(np.full(V, 1.0 / V, dtype=np.float32))
    return e


def time_steps(e, steps, warmup=2):
    e.run(warmup, 0.1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e.run(steps, 0.1)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps


AUTO_FRACTIONS = (0.5, 0.75, 0.9)


def c3_placements(precision, steps, bidir_gbs, N=100_000, V=10_000, K=2_000):
    """Resident, host and auto state (R forced to each of AUTO_FRACTIONS of the rows) at C3 from the same Philox draw:
    s/iteration, the auto bound, and whether the history and the mapping agree bit for bit with the resident handle's."""
    out = {}
    ref_map = ref_hist = None
    same = True
    ld = -(-V // 64) * 64
    placements = [("device", None), ("host", None)] + [(f"auto_{int(f * 100)}", int(f * N)) for f in AUTO_FRACTIONS]
    for where, R in placements:
        if R is not None:
            os.environ["TGB200_STATE_RESIDENT_ROWS"] = str(R)
        try:
            t0 = time.perf_counter()
            e = make_engine(N, V, K, precision, "auto" if R is not None else where)
            e.init_mapping_normal(7)
            torch.cuda.synchronize()
        finally:
            os.environ.pop("TGB200_STATE_RESIDENT_ROWS", None)
        setup = time.perf_counter() - t0
        s_it = time_steps(e, steps)
        mapping = e.get_mapping(np.empty((N, V), dtype=np.float32))
        hist = e.history(0, e.history_len())
        if ref_map is None:
            ref_map, ref_hist = mapping, hist
        else:
            same = same and bool(np.array_equal(mapping.view(np.uint32), ref_map.view(np.uint32)) and
                                 np.array_equal(hist.view(np.uint32), ref_hist.view(np.uint32)))
        del mapping
        out[where] = dict(setup_s=round(setup, 2), s_per_iter=round(s_it, 4))
        if R is not None:
            to_dev, to_host = LINK_BYTES[precision]
            staged_s = (to_dev + to_host) * (N - R) * ld / (bidir_gbs * 1e9)
            bound = max(out["device"]["s_per_iter"], staged_s)
            out[where].update(resident_rows=e.resident_rows(), ring_rows=int(e.debug("ring")[0]),
                              bound_s=round(bound, 4), of_bound=round(bound / s_it, 2))
        if where == "host":
            out[where]["ring_rows"] = int(e.debug("ring")[0])
            to_dev, to_host = LINK_BYTES[precision]
            out[where]["derived_gbs_h2d"] = round(to_dev * N * (-(-V // 64) * 64) / s_it / 1e9, 1)
            out[where]["derived_gbs_d2h"] = round(to_host * N * (-(-V // 64) * 64) / s_it / 1e9, 1)
            # the seeded legacy draw, emitted over the link into host M
            st = np.random.RandomState(3).get_state()
            t0 = time.perf_counter()
            e.init_mapping_legacy(st)
            torch.cuda.synchronize()
            out[where]["legacy_draw_s"] = round(time.perf_counter() - t0, 2)
        e.close()
    out["slowdown"] = round(out["host"]["s_per_iter"] / out["device"]["s_per_iter"], 2)
    out["same_bits"] = same
    return out


def big_run(N, V, K, steps, precision="bf16x3", placements=("host", "auto")):
    dev_b, host_b = HOST_STATE_BYTES_PER_ELEMENT[precision]
    elems = N * (-(-V // 64) * 64)
    avail = host_memory_available() or 0
    free, _ = torch.cuda.mem_get_info(0)
    res = dict(shape=[N, V, K], precision=precision, host_state_gib=round(host_b * elems / 2**30, 1),
               resident_gib_estimate=round(22 * elems / 2**30, 1), mem_available_gib=round(avail / 2**30, 1),
               device_free_gib=round(free / 2**30, 1))
    if host_b * elems + (8 << 30) > avail:
        res["run"] = "not run: MemAvailable is too small for the pinned host state plus 8 GiB of headroom"
        return res
    for where in placements:
        r = res[where] = {}
        try:
            t0 = time.perf_counter()
            free = torch.cuda.mem_get_info(0)[0]
            e = make_engine(N, V, K, precision, where)
            e.init_mapping_normal(7)
            torch.cuda.synchronize()
            r["setup_s"] = round(time.perf_counter() - t0, 1)
            r["device_used_gib"] = round((free - torch.cuda.mem_get_info(0)[0]) / 2**30, 1)
            if where == "auto":
                plan = plan_state(e.cfg, free)
                r.update(resident_rows=e.resident_rows(), of_rows=N, ring_rows=int(e.debug("ring")[0]),
                         plan_device_gib=round(plan.device_bytes / 2**30, 1), plan_reserve_gib=round(plan.reserve_bytes / 2**30, 1),
                         pinned_gib=round(plan.host_bytes / 2**30, 1))
            r["s_per_iter"] = round(time_steps(e, steps, warmup=1), 3)
            r["final_loss"] = float(e.history(e.history_len() - 1, 1)[0, 0])
            e.close()
            r["run"] = "ran"
        except _lib.TangramB200Error as ex:
            r["run"] = f"refused: {ex}"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--big-cells", type=int, default=160_000)
    ap.add_argument("--big-spots", type=int, default=24_000)
    ap.add_argument("--big-genes", type=int, default=256)
    ap.add_argument("--skip-big", action="store_true")
    ap.add_argument("--skip-big-host", action="store_true", help="at the big size, run only the auto split")
    ap.add_argument("--out")
    a = ap.parse_args()
    torch.cuda.init()
    r = dict(card=card(), copy_probe=copy_probe())
    for precision in ("bf16", "bf16x3"):
        r[f"c3_{precision}"] = c3_placements(precision, a.steps, r["copy_probe"]["bidirectional_gbs"])
    if not a.skip_big:
        r["big"] = big_run(a.big_cells, a.big_spots, a.big_genes, 2,
                           placements=("auto",) if a.skip_big_host else ("host", "auto"))
    s = json.dumps(r)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
