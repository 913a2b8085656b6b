"""Dev tool: a few iterations of every precision mode at shapes that hit the tensor-core kernels ragged in both
dimensions (last row tile partly out of range) -- for compute-sanitizer memcheck.
With TGB200_CHUNKS=2 in the environment the 2100-cell case also runs the chunked three-stream pipeline (store-only backward
contraction per chunk, streaming Adam on the update stream, next forward's chunks on the third stream).
`python tools/san_small.py rows` runs only the row-pass cases: one row width in every threads x slots bucket of
launch_softmax_rows (both edges of the widest register-cached one, and the uncached path), entropy term on and off."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
from oracle.tangram_oracle import synthetic_inputs
from tangram_b200 import Mapper
rows_only = len(sys.argv) > 1 and sys.argv[1] == "rows"
for V in (1030, 4100, 6150, 8190, 10000, 12290, 16390, 24570, 24580, 30000):
    rng = np.random.default_rng(V)
    S, G = (rng.random((5, 3)) + 0.1).astype(np.float32), (rng.random((V, 3)) + 0.1).astype(np.float32)
    for prec in ("bf16x3", "bf16"):
        for lam_r in (0.0, 1e-2):
            m = Mapper(S=S, G=G, d=(G.sum(axis=1) / G.sum()).astype(np.float32), lambda_d=1.0, lambda_r=lam_r, precision=prec, device="cuda:0")
            out, hist = m.train(2, print_each=None)
            assert np.all(np.isfinite(out)) and np.allclose(out.sum(axis=1), 1.0, atol=1e-5), (V, prec, lam_r)
            m.release()
    print("row pass, V =", V, "ok", flush=True)
for (N, V, K) in (() if rows_only else ((2100, 300, 70), (130, 65, 3))):
    inp = synthetic_inputs(N, V, K, seed=3)
    for prec in ("bf16", "bf16x3", "fp32"):
        m = Mapper(S=inp["S"], G=inp["G"], d=inp["d"], lambda_g1=1.0, lambda_d=1.0, lambda_g2=0.5, lambda_r=1e-3, precision=prec, device="cuda:0")
        out, hist = m.train(4, print_each=None)
        assert np.all(np.isfinite(out)), (N, V, K, prec)
        print(N, V, K, prec, float(hist["total_loss"][-1]), flush=True)
print("done")
