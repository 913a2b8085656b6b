"""Target for `compute-sanitizer --tool memcheck` over state_memory="host": a small run in bf16 (two pipeline chunks) and
bf16x3 mode with 300-row staging blocks, so that every pass walks several blocks of the ring (the last one partial) and the
bf16 update nests them inside each chunk.  Covers the legacy draw, train(val_each=), get_mapping, project, state() and
load_state, and checks the results against a resident handle bit for bit.

    compute-sanitizer --tool memcheck python tools/san_state_host.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.tangram_oracle import synthetic_inputs  # noqa: E402
from tangram_b200 import Mapper  # noqa: E402


def main():
    N, V, K = 8300, 200, 64
    inp = synthetic_inputs(N, V, K, seed=1)
    X = np.random.default_rng(2).standard_normal((N, 5)).astype(np.float32)
    for prec in ("bf16", "bf16x3"):
        kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-4, device="cuda:0", precision=prec,
                  random_state=4)
        res = Mapper(**kw)
        os.environ["TGB200_STATE_BLOCK_ROWS"] = "300"
        host = Mapper(**kw, state_memory="host")
        del os.environ["TGB200_STATE_BLOCK_ROWS"]
        a, _ = res.train(3, print_each=None, val_each=2)
        b, _ = host.train(3, print_each=None, val_each=2)
        host.load_state(*host.state())
        res.load_state(*res.state())
        a2, _ = res.train(2, print_each=None, resume=True)
        b2, _ = host.train(2, print_each=None, resume=True)
        same = all(np.array_equal(x.view(np.uint32), y.view(np.uint32))
                   for x, y in ((a, b), (a2, b2), (res.project(X), host.project(X))))
        print(f"{prec}: host state bit-identical to resident: {same}", flush=True)
        res.release()
        host.release()


if __name__ == "__main__":
    main()
