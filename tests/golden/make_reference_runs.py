"""Golden outputs of the REAL reference Mapper (loaded by path, device='cpu') for the tests that compare against a run of
the reference itself: tests/test_oracle.py (autograd gradient, second train() call) and tests/test_parity_gpu.py (30-epoch
trajectory).  Inputs are regenerated in the tests from oracle.synthetic_inputs and the reference's own seeded draw of M0
(np.random.seed(random_state); np.random.normal(0, 1, (N, V)), mapping_optimizer.py:147-157), so only outputs are stored;
the 3000 x 700 mapping is stored as a fixed, seeded sample of rows plus its column sums.

    python tests/golden/make_reference_runs.py <checkout of the original Tangram project>
"""
import importlib.util
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle.tangram_oracle import synthetic_inputs  # noqa: E402

spec = importlib.util.spec_from_file_location("ref_mo", os.path.join(sys.argv[1], "tangram", "mapping_optimizer.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

# tests/test_oracle.py::test_oracle_matches_live_reference_autograd
inp = synthetic_inputs(500, 130, 70, seed=9)
r = ref.Mapper(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_g2=0.2, lambda_r=1e-4, random_state=5)
loss = r._loss_fn(verbose=False)[0]
loss.backward()
np.savez_compressed(os.path.join(HERE, "ref_autograd.npz"), loss=np.array(float(loss)), grad=r.M.grad.detach().numpy())

# tests/test_oracle.py::test_second_train_call_restarts_adam_like_the_reference
inp = synthetic_inputs(60, 25, 12, seed=4)
r = ref.Mapper(device="cpu", S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, random_state=7)
r.train(4, print_each=None)
r_out, r_hist = r.train(3, print_each=None)
np.savez_compressed(os.path.join(HERE, "ref_second_train.npz"), out=r_out,
                    total_loss=np.array([float(x) for x in r_hist["total_loss"]]))

# tests/test_parity_gpu.py::test_live_reference_on_the_same_gpu
inp = synthetic_inputs(3000, 700, 300, seed=31)
r = ref.Mapper(device="cpu", random_state=42, S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0)
rout, rhist = r.train(num_epochs=30, learning_rate=0.1, print_each=None)
rows = np.sort(np.random.default_rng(0).choice(3000, 96, replace=False))
np.savez_compressed(os.path.join(HERE, "ref_trajectory.npz"), total_loss=np.array([float(x) for x in rhist["total_loss"]]),
                    main_loss=np.array(rhist["main_loss"], dtype=np.float64), rows=rows, out_rows=rout[rows],
                    out_colsum=rout.sum(axis=0))
for f in ("ref_autograd.npz", "ref_second_train.npz", "ref_trajectory.npz"):
    print(f, os.path.getsize(os.path.join(HERE, f)))
