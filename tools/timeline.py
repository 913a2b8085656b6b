"""Dev tool: completion times of every launch of a few steady-state iterations on the handle's three streams
(tgb200_debug_timeline) -- shows whether the streaming Adam kernel really runs under the contractions."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from tangram_b200 import _lib
from tangram_b200.engine import Engine
name = sys.argv[1] if len(sys.argv) > 1 else "c3"
N, V, K, T, clusters, _ = bench.WORKLOADS[name]
inp = bench.gen_inputs(name, 0, N)
eng = Engine(N, V, K, precision="bf16", density_mode=_lib.DENSITY_CELLS)
eng.set_expression(inp["S"], inp["G"]); eng.set_density(inp["d"])
eng.init_mapping_normal(1234)
eng.run(5)
torch.cuda.synchronize()
eng.timeline(True)
eng.run(3)
rows = eng.timeline(False)
last = {0: 0.0, 1: 0.0, 2: 0.0, 3: 0.0}
for nm, st, ms in rows:
    print(f"{ms:9.3f} ms  stream {st}  {nm:20s}  (+{ms - last[st]:.3f} since the previous launch on this stream)")
    last[st] = ms
print(f"3 iterations: {rows[-1][2] if rows else 0:.3f} ms by the last completion")
