"""Dev tool: can the bf16 streaming update run beside a tensor-core contraction on disjoint SMs, and what would it gain?

At C3 (bf16, four cell chunks) it times, with CUDA events, on the handle's two streams:
  (a) one contraction chunk -- the backward G or the forward F' over chunk 1's rows -- with its grid capped at
      66, 60, 56, 52, 48 and 44 two-CTA clusters, and uncapped;
  (b) one update chunk (chunk 0's rows) as the product launches it, and as a persistent grid of U = 16, 24, 32, 40
      (and 132) CTAs of 512 threads, each of which holds a whole SM;
  (c) every (a) x (b) pairing at once, contraction launched first.
Whole steps at a given share are `TGB200_UPDATE_SMS=n python bench.py`.
A pairing gains what it saves against the serial sum (uncapped contraction + product update, which is what the chunk
pipeline's two streams achieve today when the contraction's full grid keeps every update CTA off the GPU), reported as
a share of the pairing's own time.  Configurations are interleaved repetition by repetition, so clock drift hits them
alike; every figure is the median.  The card's name, power limit and the SM clock sampled during the timed loop are
printed with the table; `--json PATH` also writes everything there.

Needs the debug build (-DTGB_OVERLAP_PROBE: tgb200_debug_overlap_probe and the persistent update kernel).  TGB_DBG_LIB names a prebuilt one under tools/; otherwise it is compiled into a temporary directory.
"""
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tangram_b200 import _build  # noqa: E402

if os.environ.get("TGB_DBG_LIB"):
    _build.LIB = os.path.join(ROOT, "tools", os.environ["TGB_DBG_LIB"])
else:
    _tmp = tempfile.mkdtemp(prefix="tgb_probe_")
    _build.LIB = os.path.join(_tmp, "libcfg_probe.so")
    subprocess.run([_build.find_nvcc(), "-DTGB_OVERLAP_PROBE"] + _build.NVCC_FLAGS +
                   ["-o", _build.LIB, os.path.join(_build.CSRC, "tangram_b200.cu"), "-ldl"], check=True)
_build.is_current = lambda: True

import bench  # noqa: E402
from tangram_b200 import _lib  # noqa: E402
from tangram_b200.engine import Engine  # noqa: E402

CAPS = (0, 66, 60, 56, 52, 48, 44)          # 0: as many clusters as fit
US = (0, 16, 24, 32, 40)                    # 0: the product's launch of k_adam_rows
REPS, WARM = int(os.environ.get("PROBE_REPS", 15)), 3
KINDS = {0: "G (bwd)", 1: "F' (fwd)"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    N, V, K = 100000, 10000, 2000
    inp = bench.gen_inputs("c3", 0, N)
    eng = Engine(N, V, K, precision="bf16")
    eng.set_expression(inp["S"], inp["G"]); eng.set_density(inp["d"]); eng.init_mapping_normal(1)
    eng.run(2)
    fn = eng._lib.tgb200_debug_overlap_probe
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p] + [ctypes.c_int32] * 5 + [ctypes.POINTER(ctypes.c_float)]
    out = (ctypes.c_float * 3)()

    def once(kind, cap, u, what):
        _lib.check(fn(eng._h, kind, cap, u, what, 1, out))
        return list(out)

    configs = []
    for kind in KINDS:
        configs += [(kind, c, 0, 1) for c in CAPS]
        configs += [(kind, c, u, 3) for c in CAPS for u in US]
    configs += [(0, 0, u, 2) for u in US + (132,)]
    res = {c: [] for c in configs}
    for c in configs:
        for _ in range(WARM):
            once(*c)
    clk = bench.ClockSampler(0)
    clk.start()
    for _ in range(REPS):
        for c in configs:
            res[c].append(once(*c))
    clocks = clk.stop()
    med = {c: np.median(np.array(v), axis=0) for c, v in res.items()}

    info = {"card": card(), "clocks": clocks, "reps": REPS, "chunk_rows": N // 4}
    upd = {u: float(med[(0, 0, u, 2)][2]) for u in US + (132,)}
    info["update_alone_ms"] = {str(u): round(t, 4) for u, t in upd.items()}
    print(f"card: {info['card']}  clocks: {clocks}")
    print("update chunk alone (ms): " + ", ".join(f"{'product' if u == 0 else f'U={u}'} {t:.3f}" for u, t in upd.items()))
    best = None
    for kind, name in KINDS.items():
        alone = {c: float(med[(kind, c, 0, 1)][2]) for c in CAPS}
        serial = alone[0] + upd[0]
        print(f"\n{name}: alone " + ", ".join(f"{'full' if c == 0 else c}: {t:.3f}" for c, t in alone.items())
              + f" ms; serial sum with the product update {serial:.3f} ms")
        print(f"{'cap':>5} {'U':>5} {'contr end':>10} {'upd end':>9} {'pair':>8} {'gain':>8} {'gain/pair':>9}")
        rows = []
        for c in CAPS:
            for u in US:
                ce, ue, pair = (float(x) for x in med[(kind, c, u, 3)])
                gain = serial - pair
                rows.append({"cap": c, "U": u, "contraction_end_ms": round(ce, 4), "update_end_ms": round(ue, 4),
                             "pair_ms": round(pair, 4), "gain_ms": round(gain, 4), "gain_over_pair": round(gain / pair, 4)})
                print(f"{c or 'full':>5} {u or 'prod':>5} {ce:10.3f} {ue:9.3f} {pair:8.3f} {gain:8.3f} {gain / pair:9.1%}")
                if best is None or gain / pair > best[0]:
                    best = (gain / pair, name, c, u)
        info[name] = {"alone_ms": {str(c): round(t, 4) for c, t in alone.items()}, "serial_ms": round(serial, 4), "pairs": rows}
    info["best"] = {"gain_over_pair": round(best[0], 4), "contraction": best[1], "cap": best[2], "U": best[3]}
    print(f"\nbest pairing: {best[1]} cap {best[2]} U {best[3]}: gain {best[0]:.1%} of the pair's time "
          f"({'meets' if best[0] >= 0.10 else 'misses'} the 10 % bar)")
    if "--json" in sys.argv:
        with open(sys.argv[sys.argv.index("--json") + 1], "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
