"""Validation and cross-validation of a cell-sharded mapping on two GPUs (NCCL), launched as a torchrun subprocess like
tests/test_multigpu.py; skipped with fewer than two devices.

* Mapper(process_group=).train(12, val_each=3) in fp32, bf16x3 and bf16 against the unsharded Mapper from the same M0:
  val_* lists within 1e-5 relative (bf16: within the 1e-3 test_multigpu.py allows its losses), bit-identical on both
  ranks, and validation_terms() identical on both ranks;
* cross_val(mode="cells", cv_mode="10fold" / "loo", process_group=) against the unsharded cross_val: cv_dict and the
  per-gene test scores within 1e-5, identical on both ranks.  The 10-fold run draws its initial mappings from numpy's
  global generator (no random_state), so every fold after the first also checks that each rank's generator ends where
  the unsharded draw leaves it.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import contextlib, io, os, sys, numpy as np, pandas as pd, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TGB_ROOT"])
from oracle.tangram_oracle import synthetic_inputs
import tangram_b200 as tg
from tangram_b200 import Mapper
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = f"cuda:{rank}"
dist.init_process_group("nccl", device_id=torch.device(dev))
KEYS = ["val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy"]


def same_on_every_rank(x, what):
    got = [None] * world
    dist.all_gather_object(got, np.asarray(x, dtype=np.float32).tobytes())
    assert all(g == got[0] for g in got), f"{what} differs between ranks"


N, V, K = 3001, 700, 300
inp = synthetic_inputs(N, V, K, seed=5)
M0 = np.random.default_rng(2).standard_normal((N, V)).astype(np.float32)
kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-3, lambda_g2=0.3, device=dev, M0=M0)
for prec, tol in (("fp32", 1e-5), ("bf16x3", 1e-5), ("bf16", 1e-3)):
    m = Mapper(process_group=dist.group.WORLD, precision=prec, **kw)
    assert m._sharded == (world > 1) and m._own_comm == (world > 1)
    _, hist = m.train(12, print_each=None, val_each=3)
    vt = m.validation_terms()
    m.release()
    u = Mapper(precision=prec, **kw)
    _, ref = u.train(12, print_each=None, val_each=3)
    u.release()
    worst = 0.0
    for k in KEYS:
        got, want = np.array(hist[k]), np.array(ref[k])
        assert got.shape == want.shape == (4,), (k, got, want)
        err = np.abs(got - want) / np.maximum(np.abs(want), 1e-30) if prec != "bf16" else np.abs(got - want)
        worst = max(worst, float(err.max()))
        assert np.all(err <= tol), (prec, k, got, want)
        same_on_every_rank(hist[k], f"{prec} {k}")
    same_on_every_rank([vt[k] for k in KEYS], f"{prec} validation_terms()")
    print(f"rank {rank} {prec}: val_* against the unsharded mapper, largest {'rel' if prec != 'bf16' else 'abs'} "
          f"difference {worst:.3e}", flush=True)

# cross-validation: a small synthetic AnnData pair
Nc, Vc, Kc = 1203, 300, 24
ic = synthetic_inputs(Nc, Vc, Kc, seed=9)
genes = [f"g{i}" for i in range(Kc)]


def adatas():
    ad_sc = tg.MiniAnnData(X=ic["S"].copy(), obs=pd.DataFrame(index=[f"c{i}" for i in range(Nc)]), var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=ic["G"].copy(), obs=pd.DataFrame(index=[f"v{i}" for i in range(Vc)]), var=pd.DataFrame(index=genes))
    tg.pp_adatas(ad_sc, ad_sp)
    return ad_sc, ad_sp


def cv(cv_mode, random_state, pg):
    np.random.seed(11)
    with contextlib.redirect_stdout(io.StringIO()):
        return tg.cross_val(*adatas(), mode="cells", num_epochs=30, device=dev, cv_mode=cv_mode, random_state=random_state,
                            density_prior="uniform", lambda_d=1.0, return_gene_pred=cv_mode == "loo", precision="fp32",
                            process_group=pg)


for cv_mode, random_state in (("10fold", None), ("loo", 7)):
    got, want = cv(cv_mode, random_state, dist.group.WORLD), cv(cv_mode, random_state, None)
    if cv_mode == "loo":
        (got, ge, df), (want, ge_w, df_w) = got, want
        assert list(ge.var.index) == list(ge_w.var.index) and list(df.index) == list(df_w.index)
        np.testing.assert_allclose(ge.var["test_score"].to_numpy(), ge_w.var["test_score"].to_numpy(), atol=1e-5)
        np.testing.assert_allclose(df["score"].to_numpy(), df_w["score"].to_numpy(), atol=1e-5)
        same_on_every_rank(ge.var["test_score"].to_numpy(), "loo test scores")
        same_on_every_rank(np.asarray(ge.X), "loo gene predictions")
    for k in ("avg_test_score", "avg_train_score"):
        assert abs(got[k] - want[k]) <= 1e-5, (cv_mode, k, got[k], want[k])
    same_on_every_rank([got["avg_test_score"], got["avg_train_score"]], f"{cv_mode} cv_dict")
    print(f"rank {rank} cross_val {cv_mode}: {got} (unsharded {want})", flush=True)
dist.barrier()
dist.destroy_process_group()
print("SHARDED VALIDATION OK", flush=True)
'''


def _launch(tmp_path, nproc):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, TGB_ROOT=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr",
           "127.0.0.1", "--master-port", "29541", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1200)
    print(res.stdout[-4000:], res.stderr[-4000:])
    return res


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_validation_and_cross_val(tmp_path):
    res = _launch(tmp_path, 2)
    assert res.returncode == 0 and res.stdout.count("SHARDED VALIDATION OK") == 2
