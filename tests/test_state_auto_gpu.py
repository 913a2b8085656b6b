"""state_memory="auto" on one H100: rows [0, R) of M and Adam's moments on the device, rows [R, N) in pinned host memory
streamed through the ring, give the resident handle's results bit for bit.  TGB200_STATE_RESIDENT_ROWS forces the split
and TGB200_STATE_BLOCK_ROWS small blocks, so that every pass has resident pieces and several staged blocks (and, in bf16
mode, a chunk that straddles R).

The bit-identity cases are the host-state suite's (tests/test_state_host_gpu.py) with R inside the mapping; the split
points R = 0, R = N, R inside a cell chunk, R off the block grid and R = N - 1 run on a two-chunk bf16 mapper.  R = N is
the device handle: the same launches, no ring.  An unforced auto mapper on a device whose free memory a filler tensor
shrinks keeps part of its rows, runs every pass, and stays within the library's plan of its device memory."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.tangram_oracle import synthetic_inputs
from tangram_b200 import Mapper, MapperConstrained, _lib, legacy_rng
from tangram_b200.engine import Engine, plan_state
from tests.test_state_host_gpu import CASES, regulariser_kw, same_bits, same_rng_state

pytestmark = pytest.mark.gpu


def _build(cls, kw, state_memory, seed, monkeypatch, resident=None, block_rows=None):
    st = np.random.get_state()
    if resident is not None:
        monkeypatch.setenv("TGB200_STATE_RESIDENT_ROWS", str(resident))
    if block_rows:
        monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", str(block_rows))
    try:
        m = cls(**kw, random_state=seed, state_memory=state_memory)
    finally:
        monkeypatch.delenv("TGB200_STATE_RESIDENT_ROWS", raising=False)
        monkeypatch.delenv("TGB200_STATE_BLOCK_ROWS", raising=False)
    return m, np.random.get_state()


def _compare(res, auto, N, V, X, val=True):
    """Train both from the same draw and compare every output as bits."""
    out_r, h_r = res.train(6, print_each=None, val_each=2 if val else None)
    out_a, h_a = auto.train(6, print_each=None, val_each=2 if val else None)
    assert same_bits(out_r, out_a)
    assert same_bits(res.history_matrix, auto.history_matrix)      # every column, validation 12-15 included
    for a, b in zip(res.state(), auto.state()):
        assert same_bits(np.asarray(a), np.asarray(b))
    assert same_bits(res.project(X), auto.project(X))
    if val:
        assert h_r["val_total_loss"] == h_a["val_total_loss"]
        assert same_bits(np.array(list(res.validation_terms().values()), dtype=np.float32),
                         np.array(list(auto.validation_terms().values()), dtype=np.float32))
    t_r = torch.empty((N, V), dtype=torch.float32, device="cuda:0")
    t_a = torch.empty_like(t_r)
    res.train(4, print_each=None, resume=True, out=t_r)
    auto.train(4, print_each=None, resume=True, out=t_a)
    assert torch.equal(t_r.view(torch.int32), t_a.view(torch.int32))
    assert same_bits(res.history_matrix, auto.history_matrix)
    for a, b in zip(res.state(), auto.state()):
        assert same_bits(np.asarray(a), np.asarray(b))


def _mapper_kw(case):
    precision, N, V, K, clusters, regs, chunks = CASES[case]
    inp = synthetic_inputs(N, V, K, seed=N + V, n_types=6 if regs else 0, clusters=clusters)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, device="cuda:0", precision=precision)
    if clusters:
        kw["d_source"] = inp["d_source"]
    if regs:
        kw.update(regulariser_kw(N, V, inp))
    return kw, N, V, chunks


@pytest.mark.parametrize("case", list(CASES))
def test_mapper_auto_state_is_bit_identical(case, monkeypatch):
    assert legacy_rng.device_draw_supported()
    kw, N, V, chunks = _mapper_kw(case)
    R, blk = N * 3 // 5 + 7, N // 9 + 3                   # off the block and chunk grids
    X = np.random.default_rng(3).standard_normal((N, 7)).astype(np.float32)
    res, rng_res = _build(Mapper, kw, "device", 11, monkeypatch)
    auto, rng_auto = _build(Mapper, kw, "auto", 11, monkeypatch, resident=R, block_rows=blk)
    try:
        assert auto.resident_rows == R and res.resident_rows == N
        assert int(auto._engine.debug("ring")[0]) == blk
        assert int(auto._debug("shape")[4]) == chunks
        assert same_rng_state(rng_res, rng_auto)                  # numpy's generator after the legacy draw
        assert same_bits(res.state()[0], auto.state()[0])         # the draw itself
        _compare(res, auto, N, V, X)
    finally:
        res.release()
        auto.release()


# R on a two-chunk bf16 mapper of 9000 rows (chunk boundary 4608) with 700-row blocks
SPLITS = {"R0": 0, "R_inside_chunk0": 2100, "R_inside_chunk1": 6001, "R_off_block_grid": 4608 + 333, "R_N_minus_1": 8999}


@pytest.mark.parametrize("split", list(SPLITS))
def test_split_points_are_bit_identical(split, monkeypatch):
    kw, N, V, _ = _mapper_kw("bf16_2chunks")
    R = SPLITS[split]
    X = np.random.default_rng(4).standard_normal((N, 5)).astype(np.float32)
    res, _ = _build(Mapper, kw, "device", 7, monkeypatch)
    auto, _ = _build(Mapper, kw, "auto", 7, monkeypatch, resident=R, block_rows=700)
    try:
        assert auto.resident_rows == R
        assert int(auto._engine.debug("ring")[0]) == min(700, N - R)
        _compare(res, auto, N, V, X)
    finally:
        res.release()
        auto.release()


@pytest.mark.parametrize("case", ["bf16_2chunks", "bf16x3"])
def test_all_resident_is_the_device_handle(case, monkeypatch):
    """R = N (forced, and unforced on an idle H100): no ring, and the device handle's launches and bits."""
    kw, N, V, _ = _mapper_kw(case)
    res, _ = _build(Mapper, kw, "device", 5, monkeypatch)
    forced, _ = _build(Mapper, kw, "auto", 5, monkeypatch, resident=N)
    free, _ = _build(Mapper, kw, "auto", 5, monkeypatch)
    try:
        plan = plan_state(free._cfg, torch.cuda.mem_get_info(0)[0])
        assert plan.resident_rows == N and plan.host_bytes == 0 and plan.block_rows == 0
        for m in (forced, free):
            assert m.resident_rows == N and int(m._engine.debug("ring")[0]) == 0
        outs = [m.train(5, print_each=None, val_each=2)[0] for m in (res, forced, free)]
        assert same_bits(outs[0], outs[1]) and same_bits(outs[0], outs[2])
        assert res.kernel_launches() == forced.kernel_launches() == free.kernel_launches()
    finally:
        for m in (res, forced, free):
            m.release()


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_constrained_auto_state_is_bit_identical(precision, monkeypatch):
    N, V, K = 3000, 300, 80
    inp = synthetic_inputs(N, V, K, seed=17)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-4, device="cuda:0", precision=precision,
              target_count=N // 3)
    res, rng_res = _build(MapperConstrained, kw, "device", 4, monkeypatch)
    auto, rng_auto = _build(MapperConstrained, kw, "auto", 4, monkeypatch, resident=1234, block_rows=555)
    try:
        assert auto.resident_rows == 1234
        assert same_rng_state(rng_res, rng_auto)
        out_r, F_r, _ = res.train(6, print_each=None)
        out_a, F_a, _ = auto.train(6, print_each=None)
        assert same_bits(out_r, out_a) and same_bits(F_r, F_a)
        assert same_bits(res.history_matrix, auto.history_matrix)
        out_r, F_r, _ = res.train(3, print_each=None, resume=True)
        out_a, F_a, _ = auto.train(3, print_each=None, resume=True)
        assert same_bits(out_r, out_a) and same_bits(F_r, F_a)
        for a, b in zip(res.state(), auto.state()):
            assert same_bits(np.asarray(a), np.asarray(b))
    finally:
        res.release()
        auto.release()


def test_fp32_auto_state_is_refused():
    with pytest.raises(ValueError, match="state_memory='auto' needs precision"):
        Engine(100, 64, 8, device=0, precision="fp32", state_memory="auto")
    lib = _lib.load()
    cfg = _lib.Config(struct_size=ctypes.sizeof(_lib.Config), device=0, n_cells=100, n_voxels=64, n_genes=8,
                      precision=_lib.PREC["fp32"], density_mode=_lib.DENSITY_NONE, lambda_g1=1.0,
                      state_memory=_lib.STATE_MEMORY["auto"])
    h = ctypes.c_void_p()
    assert lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)) == -4           # TGB200_ERR_UNSUPPORTED
    assert b"auto" in lib.tgb200_last_error() and not h


@pytest.fixture
def nccl_group(monkeypatch):
    """A one-rank NCCL process group on cuda:0."""
    import torch.distributed as dist
    monkeypatch.setenv("NCCL_SOCKET_IFNAME", "lo")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_sharded_auto_state_is_bit_identical(precision, nccl_group, monkeypatch):
    N, V, K = 9000, 256, 64
    inp = synthetic_inputs(N, V, K, seed=23)
    M0 = np.random.default_rng(5).standard_normal((N, V)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_g2=0.3, device="cuda:0", M0=M0,
              precision=precision, shard=(1000, 8000), process_group=nccl_group)
    res = Mapper(**kw)
    monkeypatch.setenv("TGB200_STATE_RESIDENT_ROWS", "3001")
    monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", "900")
    auto = Mapper(**kw, state_memory="auto")
    monkeypatch.delenv("TGB200_STATE_RESIDENT_ROWS")
    monkeypatch.delenv("TGB200_STATE_BLOCK_ROWS")
    try:
        assert res._own_comm and auto._own_comm and auto.resident_rows == 3001
        out_r, _ = res.train(5, print_each=None, val_each=2)
        out_a, _ = auto.train(5, print_each=None, val_each=2)
        assert same_bits(out_r, out_a)
        assert same_bits(res.history_matrix, auto.history_matrix)
        assert same_bits(res.project(inp["S"][1000:8000]), auto.project(inp["S"][1000:8000]))
    finally:
        res.release()
        auto.release()


@pytest.mark.parametrize("mode", ["cells", "constrained"])
def test_map_cells_to_space_auto_state_is_bit_identical(mode, monkeypatch):
    import pandas as pd

    import tangram_b200 as tg
    N, V, K = 1200, 150, 60
    inp = synthetic_inputs(N, V, K, seed=31)
    genes = [f"Gene{i}" for i in range(K)]
    ad_sc = tg.MiniAnnData(X=inp["S"].copy(), obs=pd.DataFrame(index=[f"c{i}" for i in range(N)]), var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=inp["G"].copy(), obs=pd.DataFrame(index=[f"v{i}" for i in range(V)]), var=pd.DataFrame(index=genes))
    tg.pp_adatas(ad_sc, ad_sp)
    kw = dict(mode=mode, device="cuda:0", num_epochs=12, random_state=3, verbose=False, precision="bf16x3")
    if mode == "constrained":
        kw.update(target_count=300, lambda_f_reg=1, lambda_count=1)
    ref = tg.map_cells_to_space(ad_sc, ad_sp, **kw)
    monkeypatch.setenv("TGB200_STATE_RESIDENT_ROWS", "701")
    monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", "150")
    got = tg.map_cells_to_space(ad_sc, ad_sp, state_memory="auto", **kw)
    assert same_bits(got.X, ref.X)
    a, b = got.uns["train_genes_df"], ref.uns["train_genes_df"]
    assert list(a.index) == list(b.index) and same_bits(a["train_score"].to_numpy(), b["train_score"].to_numpy())
    assert got.uns["training_history"]["total_loss"] == ref.uns["training_history"]["total_loss"]
    if mode == "constrained":
        assert same_bits(np.asarray(got.obs["F_out"]), np.asarray(ref.obs["F_out"]))


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_small_device_budget(precision, monkeypatch):
    """A filler tensor leaves room for about half of the rows: the unforced plan keeps part of them, every pass that
    reads the state runs, and the device memory the handle takes stays within the plan (device_bytes at creation, plus
    the reserve after training with validation, the projection, get_mapping and state())."""
    monkeypatch.delenv("TGB200_STATE_RESIDENT_ROWS", raising=False)
    monkeypatch.delenv("TGB200_STATE_BLOCK_ROWS", raising=False)
    N, V, K = 40000, 8192, 64
    inp = synthetic_inputs(N, 64, K, seed=9)
    G = np.random.default_rng(2).random((V, K), dtype=np.float32)
    d = np.full(V, 1.0 / V, np.float32)
    kw = dict(S=inp["S"], G=G, d=d, lambda_d=1.0, device="cuda:0", precision=precision)
    torch.cuda.init()
    probe = _lib.Config(struct_size=ctypes.sizeof(_lib.Config), device=0, n_cells=N, n_voxels=V, n_genes=K,
                        precision=_lib.PREC[precision], density_mode=_lib.DENSITY_CELLS, lambda_g1=1.0, lambda_d=1.0,
                        state_memory=_lib.STATE_MEMORY["device"])
    full = plan_state(probe, 1 << 50)
    row = 8192 * (10 if precision == "bf16" else 12)
    want_free = full.device_bytes - N * row // 2 + full.reserve_bytes         # about half of the rows fit
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info(0)
    assert free0 > want_free
    filler = torch.empty(free0 - want_free, dtype=torch.uint8, device="cuda:0")
    try:
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info(0)
        auto = Mapper(**kw, random_state=1, state_memory="auto")
        try:
            plan = plan_state(auto._cfg, free1)
            R = auto.resident_rows
            assert 0 < R < N and R == plan.resident_rows
            torch.cuda.synchronize()
            used = free1 - torch.cuda.mem_get_info(0)[0]
            print(f"{precision}: R = {R} of {N}, created with {used / 2**30:.2f} GiB, plan "
                  f"{plan.device_bytes / 2**30:.2f} + {plan.reserve_bytes / 2**30:.2f} GiB")
            assert used <= plan.device_bytes
            out, _ = auto.train(4, print_each=None, val_each=2)
            assert np.isfinite(out).all() and not np.isnan(auto.history_matrix[::2, 12:16]).any()
            auto.validation_terms()
            P = auto.project(np.random.default_rng(1).standard_normal((N, 16)).astype(np.float32))
            assert np.isfinite(P).all()
            auto.state()
            torch.cuda.synchronize()
            used = free1 - torch.cuda.mem_get_info(0)[0]
            print(f"{precision}: after the passes {used / 2**30:.2f} GiB")
            assert used <= plan.device_bytes + plan.reserve_bytes
        finally:
            auto.release()
    finally:
        del filler
        torch.cuda.empty_cache()
