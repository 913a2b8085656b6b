"""The sharded tuner trial on two GPUs (NCCL), launched as a torchrun subprocess like
tests/test_sharded_validation_multigpu.py; skipped with fewer than two devices.

train_multiple_Mapper(process_group=) on the `default` and `spatial` trial inputs of tests/golden/tuning.npz, bf16x3:
* the five metrics are bit-identical on both ranks, and both ranks leave numpy's generator in the same state, the state
  the unsharded trial leaves;
* the metrics are within test_trial_matches_the_reference_trial's tolerance (1e-4) of the reference's, with the same
  allowance for rows whose vote flipped (each moves the mean vote entropy by at most 1/N, and may only flip at a near-tie
  of the reference mapping), the rows of the cell cube gathered from both ranks;
* they are within the same tolerance of the unsharded trial run on rank 0, with the allowance counted from the rows
  whose vote differs between the sharded and the unsharded cubes.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import contextlib, io, os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TGB_ROOT"])
from tangram_b200 import mapping_parameter_tuning as mpt
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = f"cuda:{rank}"
dist.init_process_group("nccl", device_id=torch.device(dev))
Z = np.load(os.path.join(os.environ["TGB_ROOT"], "tests", "golden", "tuning.npz"))
METRICS = ["cell_map_consistency", "cell_map_agreement", "cell_map_certainty", "gene_expr_consistency",
           "gene_expr_correctness"]
DATA_KEYS = ["S", "G", "d_source", "d", "device", "print_each", "voxel_weights", "ct_encode", "neighborhood_filter",
             "spatial_weights", "train_genes_idx", "val_genes_idx"]
TOL = 1e-4


def inputs(name):
    p = f"t_{name}_"
    data = [Z[p + "in_" + k] if p + "in_" + k in Z.files else None for k in DATA_KEYS]
    data[DATA_KEYS.index("device")] = dev
    config = {k[len(p + "cfg_"):]: Z[k].item() for k in Z.files if k.startswith(p + "cfg_")}
    return data, config, int(Z[p + "seed"])


def rng_state():
    _, key, pos, has_gauss, gauss = np.random.get_state()
    return key.tobytes() + np.array([pos, has_gauss, gauss], dtype=np.float64).tobytes()


def gathered(x):
    got = [None] * world
    dist.all_gather_object(got, x)
    return got


def within(what, got, want, flipped, N):
    for k in METRICS:
        allow = TOL + (flipped / N if k == "cell_map_agreement" else 0.0)
        assert abs(got[k] - want[k]) < allow, (what, k, got[k], want[k])


for name in ("default", "spatial"):
    data, config, seed = inputs(name)
    np.random.seed(seed)
    det = {}
    with contextlib.redirect_stdout(io.StringIO()):
        got = mpt.train_multiple_Mapper(config, data, details=det, process_group=dist.group.WORLD)
    state = rng_state()
    metrics = gathered(np.array([got[k] for k in METRICS]).tobytes())
    assert all(m == metrics[0] for m in metrics), f"{name}: metrics differ between ranks"
    assert all(s == state for s in gathered(state)), f"{name}: generator states differ between ranks"
    r0, r1 = det["shard_rows"]
    assert det["cell_cube"].shape[1] == r1 - r0 and det["gene_cube"].shape[1] == np.shape(data[1])[0]
    parts = gathered((r0, det["cell_cube"].cpu().numpy()))
    cube = np.concatenate([c for _, c in sorted(parts, key=lambda t: t[0])], axis=1)
    N = cube.shape[1]
    assert N == np.shape(data[0])[0]

    ref = dict(zip(METRICS, Z[f"t_{name}_metrics"]))
    votes, gap = cube.argmax(axis=2), Z[f"t_{name}_gap"]
    flipped = votes != Z[f"t_{name}_argmax"]
    assert np.all(gap[flipped] < 1e-4), gap[flipped]
    n_flipped = int(flipped.any(axis=0).sum())
    within(f"{name} against the reference", got, ref, n_flipped, N)

    if rank == 0:
        np.random.seed(seed)
        udet = {}
        with contextlib.redirect_stdout(io.StringIO()):
            want = mpt.train_multiple_Mapper(config, data, details=udet)
        assert rng_state() == state, f"{name}: the sharded trial left numpy's generator elsewhere"
        n_diff = int((udet["cell_cube"].cpu().numpy().argmax(axis=2) != votes).any(axis=0).sum())
        within(f"{name} against the unsharded trial", got, want, n_diff, N)
        print(f"{name}: sharded {got}; unsharded {want}; {n_flipped} rows flipped against the reference, {n_diff} "
              f"against the unsharded trial", flush=True)
    dist.barrier()
dist.destroy_process_group()
print("SHARDED TRIAL OK", flush=True)
'''


def _launch(tmp_path, nproc):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, TGB_ROOT=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", "29543", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1200)
    print(res.stdout[-4000:], res.stderr[-4000:])
    return res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_trial(tmp_path):
    res = _launch(tmp_path, 2)
    assert res.returncode == 0 and res.stdout.count("SHARDED TRIAL OK") == 2
