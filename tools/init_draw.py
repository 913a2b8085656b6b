"""Dev tool: the seeded initial mapping at C3 (100k cells x 10k voxels, 1e9 values).
  1. tgb200_init_mapping_legacy three times: device ms of jump / count + scan / emit / fix-up (CUDA events), host ms of
     the polynomials (the first call also finds phi), values recomputed on the host
  2. Mapper(random_state=42) with the host draw and with the device draw: __init__ wall time, then train(EPOCHS)
     (default precision) for the end-to-end time, and whether the two runs agree bit for bit
Prints the GPU's name, power limit and SM clock next to the numbers."""
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

import bench  # noqa: E402
from tangram_b200 import Mapper, _lib, legacy_rng  # noqa: E402
from tangram_b200.engine import Engine  # noqa: E402

N, V = 100_000, 10_000
EPOCHS = int(os.environ.get("EPOCHS", "100"))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()


print("gpu:", gpu_info())
e = Engine(N, V, 8, precision="bf16", density_mode=_lib.DENSITY_NONE)
for i in range(3):
    rs = np.random.RandomState(42)
    t0 = time.perf_counter()
    end, n_fixed = e.init_mapping_legacy(rs.get_state())
    wall = time.perf_counter() - t0
    s = e.debug("legacy_init")
    print(f"device draw {i}: wall {wall * 1e3:.1f} ms | jump {s[0]:.2f} ms, count+scan {s[1]:.2f} ms, emit {s[2]:.2f} ms, "
          f"fix-up {s[3]:.2f} ms (device) | host polynomials {s[4]:.1f} ms | {int(s[5])} draw blocks | "
          f"{n_fixed} values recomputed, {int(s[7])} changed | sm clock now: {gpu_info()}")
e.close()
del e

inp = bench.gen_inputs("c3", 0, N)
kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0)
runs = {}
for arm in ("host", "device"):
    legacy_rng._PROBE = arm == "device"          # False: Mapper keeps the host draw
    t0 = time.perf_counter()
    m = Mapper(random_state=42, device="cuda:0", **kw)
    t1 = time.perf_counter()
    out, hist = m.train(EPOCHS, print_each=None)
    t2 = time.perf_counter()
    runs[arm] = (out[:64].copy(), m.history_matrix.copy())
    print(f"{arm} draw: Mapper.__init__ {t1 - t0:.2f} s, train({EPOCHS}) {t2 - t1:.2f} s, end to end {t2 - t0:.2f} s | "
          f"{gpu_info()}")
    m.release()
    del m, out
same = all(np.array_equal(a, b, equal_nan=True) for a, b in zip(runs["host"], runs["device"]))
print("host and device runs bit-identical (first 64 rows of the mapping, loss history):", same)
