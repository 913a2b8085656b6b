"""Dev tool: where the time of the bf16 backward contraction's tiles goes, phase by phase, at C3.

Records one bf16 C3 step (the last of 20, after two warm-up steps) on a debug build (-DTGB_BWD_PHASE_PROBE), in which
thread 0 of each consumer warpgroup of k_gemm_tc<1,1,4,TcEpiDpStore> writes clock64() at six points of every tile:
  full      the tile's first operand-stage wait returns
  retired   the tile's last wgmma has retired (wgmma.wait_group 0)
  pt_full   the epilogue's wait for the tile's P~ returns
  stmatrix  the last stmatrix of dq is done
  store     the TMA stores of dq are issued
  read      cp.async.bulk.wait_group.read has returned (the buffer may be refilled)
and prints, per phase between consecutive points, the median and p90 over all (tile, warpgroup) records, in SM cycles
and in microseconds at the median SM clock sampled during the step.  Two more rows follow each warpgroup from tile to
tile on its SM: `period` (full to the next tile's full) and `boundary` (retired to the next tile's full); pairs more
than 4x the median period apart (the gaps between the step's chunk launches) are left out.  In the deferred epilogue
the four epilogue points fall inside the next tile's main loop, so there `mainloop` includes them.

TGB_DBG_LIB names a prebuilt debug library (a path, or a file under tools/); otherwise it is compiled into a temporary
directory.  `--json PATH` also writes the table there.
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
    _build.LIB = os.path.join(_tmp, "libbwd_probe.so")
    subprocess.run([_build.find_nvcc(), "-DTGB_BWD_PHASE_PROBE"] + _build.NVCC_FLAGS +
                   ["-o", _build.LIB, os.path.join(_build.CSRC, "tangram_b200.cu"), "-ldl"], check=True)
_build.is_current = lambda: True

import bench  # noqa: E402
from tangram_b200 import _lib  # noqa: E402
from tangram_b200.engine import Engine  # noqa: E402

POINTS = ("full", "retired", "pt_full", "stmatrix", "store", "read")
PHASES = [("mainloop", 0, 1), ("wait P~", 1, 2), ("ldmatrix..stmatrix", 2, 3), ("fence, barrier, store", 3, 4),
          ("wait store read", 4, 5)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    import torch
    N, V, K = 100000, 10000, 2000
    inp = bench.gen_inputs("c3", 0, N)
    eng = Engine(N, V, K, precision="bf16")
    eng.set_expression(inp["S"], inp["G"]); eng.set_density(inp["d"]); eng.init_mapping_normal(1)
    eng.run(2)
    fn = eng._lib.tgb200_debug_bwd_phase_probe
    fn.restype = ctypes.c_int
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    tiles = -(-N // 128) * -(-V // 256)
    buf = torch.zeros(tiles * 2 * 8, dtype=torch.int64, device="cuda")
    clk = bench.ClockSampler(0)
    clk.start()
    _lib.check(fn(eng._h, ctypes.c_void_p(buf.data_ptr())))
    eng.run(20)                                     # each step overwrites the records: the last one is kept
    torch.cuda.synchronize()
    _lib.check(fn(eng._h, None))
    clocks = clk.stop()
    rec = buf.view(tiles, 2, 8).cpu().numpy().view(np.uint64).astype(np.int64)
    seen = rec[:, :, 0] != 0
    mhz = clocks.get("sm_mhz") or float(card().split(",")[-1].split()[0])
    info = {"card": card(), "clocks": clocks, "tiles": int(seen[:, 0].sum()), "mhz_for_us": mhz, "phases": {}}

    def row(name, cyc):
        cyc = np.asarray(cyc, dtype=np.float64)
        med, p90 = np.median(cyc), np.percentile(cyc, 90)
        info["phases"][name] = {"median_cycles": round(med), "p90_cycles": round(p90),
                                "median_us": round(med / mhz, 3), "p90_us": round(p90 / mhz, 3), "n": int(cyc.size)}
        print(f"{name:>24} {med:10.0f} {p90:10.0f} {med / mhz:10.3f} {p90 / mhz:10.3f} {cyc.size:8d}")

    print(f"card: {info['card']}  clocks: {clocks}  tiles recorded: {info['tiles']} of {tiles}")
    print(f"{'phase':>24} {'med cyc':>10} {'p90 cyc':>10} {'med us':>10} {'p90 us':>10} {'n':>8}")
    r = rec[seen]                                   # [records, 8]
    for name, a, b in PHASES:
        row(name, r[:, b] - r[:, a])
    row("full to read", r[:, 5] - r[:, 0])
    period, boundary = [], []
    for cw in range(2):
        sel = seen[:, cw]
        x = rec[sel, cw]
        for sm in np.unique(x[:, 6]):
            y = x[x[:, 6] == sm]
            y = y[np.argsort(y[:, 0])]
            period.append(np.diff(y[:, 0]))
            boundary.append(y[1:, 0] - y[:-1, 1])
    period, boundary = np.concatenate(period), np.concatenate(boundary)
    keep = period < 4 * np.median(period)
    row("period", period[keep])
    row("boundary", boundary[keep])
    if "--json" in sys.argv:
        with open(sys.argv[sys.argv.index("--json") + 1], "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
