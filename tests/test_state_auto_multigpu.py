"""state_memory="auto" on a two-GPU NCCL group (one process per GPU, torch.distributed.run): each rank plans its own shard
on its own device, here with a different forced split per rank, and every rank's mapping rows, history and projection
equal those of the resident sharded run, bit for bit, in bf16 and bf16x3 mode.  Skipped with fewer than two GPUs."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TGB_ROOT"])
from oracle.tangram_oracle import synthetic_inputs
from tangram_b200 import Mapper
rank = int(os.environ["RANK"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rank}"))
N, V, K = 9001, 300, 100
inp = synthetic_inputs(N, V, K, seed=8)
S = inp["S"]
for prec in ("bf16", "bf16x3"):
    kw = dict(S=S, G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_g2=0.3, device=f"cuda:{rank}", random_state=5,
              precision=prec, process_group=dist.group.WORLD)
    res = Mapper(**kw)
    os.environ["TGB200_STATE_BLOCK_ROWS"] = "1111"
    os.environ["TGB200_STATE_RESIDENT_ROWS"] = str(1500 + 2001 * rank)
    host = Mapper(**kw, state_memory="auto")
    del os.environ["TGB200_STATE_BLOCK_ROWS"], os.environ["TGB200_STATE_RESIDENT_ROWS"]
    assert host.resident_rows == 1500 + 2001 * rank
    a, _ = res.train(6, print_each=None, val_each=3)
    b, _ = host.train(6, print_each=None, val_each=3)
    r0, r1 = res._rows
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), prec
    assert np.array_equal(res.history_matrix.view(np.uint32), host.history_matrix.view(np.uint32)), prec
    pa, pb = res.project(S[r0:r1]), host.project(S[r0:r1])
    assert np.array_equal(pa.view(np.uint32), pb.view(np.uint32)), prec
    res.release()
    host.release()
dist.barrier()
dist.destroy_process_group()
print("STATE AUTO MULTIGPU OK", flush=True)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_auto_state_matches_resident(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, TGB_ROOT=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29543", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    print(res.stdout[-3000:], res.stderr[-3000:])
    assert res.returncode == 0 and res.stdout.count("STATE AUTO MULTIGPU OK") == 2
