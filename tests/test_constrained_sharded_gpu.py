"""Cell-sharded constrained mode (MapperConstrained(process_group= / shard=), map_cells_to_space(mode="constrained",
process_group=)) on the GPU.  On one GPU, two or three shard handles play the ranks and the test plays the all-reduce by
summing their exchange buffers (tgb200_step_begin -> sum -> tgb200_step_end); they must reproduce one unsharded handle.
The seeded draw of a shard must be its slice of the unsharded draw, bit for bit.  The two-GPU NCCL run is skipped below
two GPUs."""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle.tangram_oracle import synthetic_inputs
from tangram_b200 import MapperConstrained, legacy_rng
from tangram_b200.sharded import shard_rows
from tests.helpers import max_rel, rel_fro

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# every constrained term on: density, entropy, voxel-gene, count (sum f ~ N / 2 stays above target_count), f-regulariser
LAMBDAS = dict(lambda_d=1.0, lambda_g1=1.0, lambda_g2=0.3, lambda_r=1e-3, lambda_count=0.5, lambda_f_reg=0.7)
HIST_GLOBAL = [0, 1, 2, 3, 4, 10, 11]          # loss terms, count_reg, lambda_f_reg: computed from the all-reduced buffer


def _mapping(m):
    return m._engine.get_mapping(np.empty((m.n_cells, m.n_voxels), dtype=np.float32))


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_shards_on_one_gpu_reproduce_the_unsharded_handle(precision, world):
    N, V, K, steps = 2341, 300, 120, 6              # N is not a multiple of 256: ragged shards and tiles
    inp = synthetic_inputs(N, V, K, seed=31)
    rng = np.random.default_rng(8)
    M0 = rng.standard_normal((N, V)).astype(np.float32)
    F0 = rng.standard_normal(N).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], target_count=N / 4, device="cuda:0", precision=precision, M0=M0, F0=F0,
              **LAMBDAS)
    whole = MapperConstrained(**kw)
    whole._engine.run(steps, 0.1)
    ref_P, (ref_M, ref_F, _) = _mapping(whole), whole.state()
    ref_h = whole._engine.history()
    whole.release()

    parts = [MapperConstrained(shard=shard_rows(N, r, world), **kw) for r in range(world)]
    assert [p._rows for p in parts] == [shard_rows(N, r, world) for r in range(world)] and all(p._sharded for p in parts)
    bufs = [p._engine.exchange_tensor() for p in parts]
    for _ in range(steps):
        for p in parts:
            p._engine.step_begin()
        torch.cuda.synchronize()
        total = sum(bufs[1:], bufs[0].clone())
        for b in bufs:
            b.copy_(total)
        torch.cuda.synchronize()
        for p in parts:
            p._engine.step_end(0.1)
    states = [p.state() for p in parts]
    got_P = np.concatenate([_mapping(p) for p in parts])
    got_M = np.concatenate([s[0] for s in states])
    got_F = np.concatenate([s[1] for s in states])
    assert all(s[2] == steps for s in states)
    tol = 2e-2 if precision == "bf16" else 2e-5
    assert rel_fro(got_P, ref_P) < tol and rel_fro(got_M, ref_M) < tol and rel_fro(got_F, ref_F) < tol
    hists = [p._engine.history() for p in parts]
    assert max_rel(hists[0][:, 0], ref_h[:, 0]) < (1e-3 if precision == "bf16" else 1e-5)
    for h in hists[1:]:                               # every rank logs the same global loss, bit for bit
        assert np.array_equal(h[:, HIST_GLOBAL], hists[0][:, HIST_GLOBAL], equal_nan=True)
    assert not np.isnan(hists[0][:, HIST_GLOBAL]).any()
    for p in parts:
        p.release()


def _same_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


@pytest.mark.parametrize("host_draw", [False, True])
def test_seeded_draw_of_every_shard_is_its_slice_of_the_unsharded_draw(host_draw, monkeypatch):
    """random_state=7: each shard's M rows and F entries are the unsharded handle's, bit for bit, and numpy's global
    generator ends where the unsharded construction leaves it.  N V is odd, so the second draw starts on a cached normal.
    host_draw forces the host path (as on a numpy whose arithmetic differs from the device formula): same bits."""
    N, V, K = 301, 77, 40
    inp = synthetic_inputs(N, V, K, seed=2)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], target_count=60, device="cuda:0", precision="fp32", random_state=7)
    whole = MapperConstrained(**kw)                  # the device draw: the reference for both paths
    want_state = np.random.get_state()
    want_M, want_F, _ = whole.state()
    whole.release()
    if host_draw:
        monkeypatch.setattr(legacy_rng, "_PROBE", False)
        again = MapperConstrained(**kw)
        assert _same_state(np.random.get_state(), want_state)
        M, F, _ = again.state()
        assert np.array_equal(M.view(np.uint32), want_M.view(np.uint32))
        assert np.array_equal(F.view(np.uint32), want_F.view(np.uint32))
        again.release()
    for world in (2, 3):
        for r in range(world):
            r0, r1 = shard_rows(N, r, world)
            np.random.seed(123)                       # construction must not depend on where the generator was
            m = MapperConstrained(shard=(r0, r1), **kw)
            assert _same_state(np.random.get_state(), want_state)
            M, F, step = m.state()
            assert M.shape == (r1 - r0, V) and F.shape == (r1 - r0,) and step == 0
            assert np.array_equal(M.view(np.uint32), want_M[r0:r1].view(np.uint32))
            assert np.array_equal(F.view(np.uint32), want_F[r0:r1].view(np.uint32))
            m.release()


def test_map_cells_to_space_constrained_on_a_one_rank_gloo_group():
    """The public entry point with process_group= in constrained mode (plumbing: one rank holds every cell) against the
    same call without a group."""
    import pandas as pd
    import torch.distributed as dist

    import tangram_b200 as tg
    N, V, K = 400, 90, 50
    inp = synthetic_inputs(N, V, K, seed=12)
    genes = [f"Gene{i}" for i in range(K)]
    ad_sc = tg.MiniAnnData(X=inp["S"].copy(), obs=pd.DataFrame(index=[f"c{i}" for i in range(N)]), var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=inp["G"].copy(), obs=pd.DataFrame(index=[f"v{i}" for i in range(V)]), var=pd.DataFrame(index=genes))
    tg.pp_adatas(ad_sc, ad_sp)
    kw = dict(mode="constrained", target_count=80, lambda_f_reg=1, lambda_count=1, device="cuda:0", num_epochs=12,
              random_state=3, verbose=False, precision="fp32")
    ref = tg.map_cells_to_space(ad_sc, ad_sp, **kw)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=0, world_size=1)
    try:
        got = tg.map_cells_to_space(ad_sc, ad_sp, process_group=dist.group.WORLD, **kw)
        full = tg.map_cells_to_space(ad_sc, ad_sp, process_group=dist.group.WORLD, gather=True, **kw)
    finally:
        dist.destroy_process_group()
    assert got.X.shape == (N, V) and got.uns["shard_rows"] == (0, N) and list(got.obs.index) == list(ref.obs.index)
    assert rel_fro(got.X, ref.X) < 1e-6
    assert rel_fro(np.asarray(got.obs["F_out"]), np.asarray(ref.obs["F_out"])) < 1e-6
    a, b = got.uns["train_genes_df"].sort_index(), ref.uns["train_genes_df"].sort_index()
    assert list(a.index) == list(b.index) and np.allclose(a["train_score"], b["train_score"], rtol=1e-6, atol=0)
    assert got.uns["training_history"]["total_loss"] == ref.uns["training_history"]["total_loss"]
    assert full.X.shape == (N, V) and "shard_rows" not in full.uns
    assert rel_fro(np.asarray(full.obs["F_out"]), np.asarray(ref.obs["F_out"])) < 1e-6


WORKER = r'''
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TGB_ROOT"])
from oracle.tangram_oracle import OracleMapperConstrained, synthetic_inputs
from tangram_b200 import MapperConstrained
from tangram_b200.sharded import shard_rows
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rank}"))
N, V, K = 3001, 700, 300
inp = synthetic_inputs(N, V, K, seed=5)
rng = np.random.default_rng(2)
M0, F0 = rng.standard_normal((N, V)).astype(np.float32), rng.standard_normal(N).astype(np.float32)
kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-3, lambda_g2=0.3, lambda_count=0.5,
          lambda_f_reg=0.7, target_count=N / 4)
o = OracleMapperConstrained(M0=M0, F0=F0, **kw)
ref, refF, oh = o.train(8, print_each=None)
for prec, tol in (("fp32", 2e-5), ("bf16", 5e-2)):
    m = MapperConstrained(device=f"cuda:{rank}", M0=M0, F0=F0, precision=prec, process_group=dist.group.WORLD, **kw)
    out, F_out, hist = m.train(8, print_each=None)
    r0, r1 = shard_rows(N, rank, world)
    assert out.shape == (r1 - r0, V) and F_out.shape == (r1 - r0,)
    err = np.linalg.norm(out - ref[r0:r1]) / np.linalg.norm(ref[r0:r1])
    errF = np.linalg.norm(F_out - refF[r0:r1]) / np.linalg.norm(refF[r0:r1])
    dl = max(abs(float(a) - b) / abs(b) for a, b in zip(m.history_matrix[:, 0], o.float_history["total_loss"]))
    print(f"rank {rank} {prec}: rel-Frobenius {err:.3e} F_out {errF:.3e} max rel loss diff {dl:.3e}", flush=True)
    assert err < tol and errF < tol and dl < (1e-5 if prec == "fp32" else 1e-3)
    assert m._own_comm, "NCCL group: the exchange must run inside tgb200_run on the handle's own communicator"
    m.release()
import pandas as pd
import tangram_b200 as tg
Na, Va, Ka = 1203, 300, 120
ia = synthetic_inputs(Na, Va, Ka, seed=9)
genes = [f"g{i}" for i in range(Ka)]
ad_sc = tg.MiniAnnData(X=ia["S"].copy(), obs=pd.DataFrame(index=[f"c{i}" for i in range(Na)]), var=pd.DataFrame(index=genes))
ad_sp = tg.MiniAnnData(X=ia["G"].copy(), obs=pd.DataFrame(index=[f"v{i}" for i in range(Va)]), var=pd.DataFrame(index=genes))
tg.pp_adatas(ad_sc, ad_sp)
akw = dict(mode="constrained", target_count=200, lambda_f_reg=1, lambda_count=1, device=f"cuda:{rank}", num_epochs=10,
           random_state=7, verbose=False, precision="fp32", process_group=dist.group.WORLD)
part = tg.map_cells_to_space(ad_sc, ad_sp, **akw)
full = tg.map_cells_to_space(ad_sc, ad_sp, gather=True, **akw)
d = np.asarray(ad_sp.obs["rna_count_based_density"], dtype=np.float32)
oa = OracleMapperConstrained(ia["S"], ia["G"], d, lambda_d=1, lambda_g1=1, lambda_g2=0, lambda_r=0, lambda_count=1,
                             lambda_f_reg=1, target_count=200, random_state=7)
ra, rF, _ = oa.train(10, print_each=None)
a0, a1 = part.uns["shard_rows"]
assert (a0, a1) == shard_rows(Na, rank, world) and list(part.obs.index) == [f"c{i}" for i in range(a0, a1)]
assert np.linalg.norm(part.X - ra[a0:a1]) / np.linalg.norm(ra[a0:a1]) < 1e-4
assert np.linalg.norm(np.asarray(part.obs["F_out"]) - rF[a0:a1]) / np.linalg.norm(rF[a0:a1]) < 1e-4
assert (full is None) == (rank != 0)
if rank == 0:
    assert full.X.shape == (Na, Va) and np.linalg.norm(full.X - ra) / np.linalg.norm(ra) < 1e-4
    assert np.linalg.norm(np.asarray(full.obs["F_out"]) - rF) / np.linalg.norm(rF) < 1e-4
    assert len(full.uns["train_genes_df"]) == Ka
dist.barrier()
dist.destroy_process_group()
print("MULTIGPU CONSTRAINED OK", flush=True)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_nccl_sharded_constrained_matches_oracle(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, TGB_ROOT=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29534", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    print(res.stdout[-3000:], res.stderr[-3000:])
    assert res.returncode == 0 and res.stdout.count("MULTIGPU CONSTRAINED OK") == 2
