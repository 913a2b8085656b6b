"""state_memory="host" on one H100: M and Adam's moments in pinned host memory (TGB200_STATE_HOST), streamed through the
device ring of row blocks, give the resident handle's results bit for bit, and the device keeps only the contraction
operands and the ring.  TGB200_STATE_BLOCK_ROWS forces small blocks, so that every pass walks several of them (and, in
bf16 mode, several inside each pipeline chunk, with a partial block at each chunk's end).

Every case builds a resident and a host-state mapper from the same seed, with the seeded legacy draw made on the device,
and compares as uint32: the drawn M and numpy's generator state after the draw, the history of train(val_each=) with its
validation columns 12-15, the returned softmax(M) (host array and train(out=)), state(), project(X) and a resume=True
continuation.  The cases cover bf16 at one, two and four pipeline chunks, bf16x3, clusters mode with d_source, every
regulariser at once, constrained mode in both precisions, and a sharded mapper on a one-rank NCCL group.
"""
import numpy as np
import pytest
import torch

from oracle.tangram_oracle import grid_graph, synthetic_inputs
from tangram_b200 import Mapper, MapperConstrained, legacy_rng
from tangram_b200.engine import Engine

pytestmark = pytest.mark.gpu


def same_bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def same_rng_state(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def regulariser_kw(N, V, inp):
    conn, _ = grid_graph(V)
    rs = np.asarray(conn.sum(axis=1)).ravel()
    sw = conn.multiply(1.0 / rs[:, None]).tocsr()
    return dict(lambda_g2=0.4, lambda_r=1e-4, lambda_l1=1e-6, lambda_l2=1e-7, lambda_neighborhood_g1=0.5,
                voxel_weights=conn, lambda_ct_islands=0.2, neighborhood_filter=conn, ct_encode=inp["ct_encode"],
                lambda_getis_ord=0.3, spatial_weights=sw)


# name: (precision, N, V, K, clusters, regularisers, pipeline chunks of the bf16 handle)
CASES = {
    "bf16_1chunk": ("bf16", 2000, 300, 80, False, False, 1),
    "bf16_2chunks": ("bf16", 9000, 200, 64, False, False, 2),
    "bf16_4chunks": ("bf16", 33000, 96, 48, False, False, 4),
    "bf16_regs": ("bf16", 9000, 256, 64, False, True, 2),
    "bf16x3": ("bf16x3", 3000, 300, 80, False, False, 1),
    "bf16x3_regs": ("bf16x3", 2500, 256, 64, False, True, 1),
    "bf16_clusters": ("bf16", 96, 5000, 120, True, False, 1),
    "bf16x3_clusters": ("bf16x3", 96, 5000, 120, True, False, 1),
}


def _build(cls, kw, state_memory, seed, block_rows=None, monkeypatch=None):
    st = np.random.get_state()
    if block_rows:
        monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", str(block_rows))
    try:
        m = cls(**kw, random_state=seed, state_memory=state_memory)
    finally:
        if block_rows:
            monkeypatch.delenv("TGB200_STATE_BLOCK_ROWS")
    if block_rows:
        assert int(m._engine.debug("ring")[0]) == block_rows
    return m, np.random.get_state(), st


@pytest.mark.parametrize("case", list(CASES))
def test_mapper_host_state_is_bit_identical(case, monkeypatch):
    assert legacy_rng.device_draw_supported()
    precision, N, V, K, clusters, regs, chunks = CASES[case]
    inp = synthetic_inputs(N, V, K, seed=N + V, n_types=6 if regs else 0, clusters=clusters)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, device="cuda:0", precision=precision)
    if clusters:
        kw["d_source"] = inp["d_source"]
    if regs:
        kw.update(regulariser_kw(N, V, inp))
    X = np.random.default_rng(3).standard_normal((N, 7)).astype(np.float32)
    res, rng_res, _ = _build(Mapper, kw, "device", 11)
    host, rng_host, _ = _build(Mapper, kw, "host", 11, block_rows=N // 5 + 3, monkeypatch=monkeypatch)
    try:
        assert int(res._debug("ring")[0]) == 0
        assert int(host._debug("shape")[4]) == chunks == int(res._debug("shape")[4])
        assert same_rng_state(rng_res, rng_host)                  # numpy's generator after the legacy draw
        assert same_bits(res.state()[0], host.state()[0])         # the draw itself
        out_r, h_r = res.train(6, print_each=None, val_each=2)
        out_h, h_h = host.train(6, print_each=None, val_each=2)
        assert same_bits(out_r, out_h)
        assert same_bits(res.history_matrix, host.history_matrix)  # every column, validation 12-15 included
        assert not np.isnan(host.history_matrix[::2, 12:16]).any()
        assert h_r["val_total_loss"] == h_h["val_total_loss"]
        for a, b in zip(res.state(), host.state()):
            assert same_bits(np.asarray(a), np.asarray(b))
        assert same_bits(res.project(X), host.project(X))
        assert same_bits(np.array(list(res.validation_terms().values()), dtype=np.float32),
                         np.array(list(host.validation_terms().values()), dtype=np.float32))
        t_r = torch.empty((N, V), dtype=torch.float32, device="cuda:0")
        t_h = torch.empty_like(t_r)
        res.train(4, print_each=None, resume=True, out=t_r)
        host.train(4, print_each=None, resume=True, out=t_h)
        assert torch.equal(t_r.view(torch.int32), t_h.view(torch.int32))
        assert same_bits(res.history_matrix, host.history_matrix)
        for a, b in zip(res.state(), host.state()):
            assert same_bits(np.asarray(a), np.asarray(b))
    finally:
        res.release()
        host.release()


def test_load_state_round_trip(monkeypatch):
    """state() of a host-state mapper loaded into a resident one (and back) continues with the same bits."""
    N, V, K = 2400, 200, 64
    inp = synthetic_inputs(N, V, K, seed=5)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, device="cuda:0", precision="bf16", random_state=2)
    monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", "1000")
    host = Mapper(**kw, state_memory="host")
    monkeypatch.delenv("TGB200_STATE_BLOCK_ROWS")
    res = Mapper(**kw)
    try:
        host.train(5, print_each=None)
        res.load_state(*host.state())
        host.load_state(*host.state())
        a, _ = res.train(3, print_each=None, resume=True)
        b, _ = host.train(3, print_each=None, resume=True)
        assert same_bits(a, b)
    finally:
        res.release()
        host.release()


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_constrained_host_state_is_bit_identical(precision, monkeypatch):
    N, V, K = 3000, 300, 80
    inp = synthetic_inputs(N, V, K, seed=17)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-4, device="cuda:0", precision=precision,
              target_count=N // 3)
    res, rng_res, _ = _build(MapperConstrained, kw, "device", 4)
    host, rng_host, _ = _build(MapperConstrained, kw, "host", 4, block_rows=777, monkeypatch=monkeypatch)
    try:
        assert same_rng_state(rng_res, rng_host)
        for a, b in zip(res.state(), host.state()):
            assert same_bits(np.asarray(a), np.asarray(b))
        out_r, F_r, _ = res.train(6, print_each=None)
        out_h, F_h, _ = host.train(6, print_each=None)
        assert same_bits(out_r, out_h) and same_bits(F_r, F_h)
        assert same_bits(res.history_matrix, host.history_matrix)
        out_r, F_r, _ = res.train(3, print_each=None, resume=True)
        out_h, F_h, _ = host.train(3, print_each=None, resume=True)
        assert same_bits(out_r, out_h) and same_bits(F_r, F_h)
        for a, b in zip(res.state(), host.state()):
            assert same_bits(np.asarray(a), np.asarray(b))
    finally:
        res.release()
        host.release()


def test_fp32_host_state_is_refused():
    import ctypes

    from tangram_b200 import _lib
    with pytest.raises(ValueError, match="state_memory='host' needs precision"):
        Engine(100, 64, 8, device=0, precision="fp32", state_memory="host")
    lib = _lib.load()
    cfg = _lib.Config(struct_size=ctypes.sizeof(_lib.Config), device=0, n_cells=100, n_voxels=64, n_genes=8,
                      precision=_lib.PREC["fp32"], density_mode=_lib.DENSITY_NONE, lambda_g1=1.0,
                      state_memory=_lib.STATE_MEMORY["host"])
    h = ctypes.c_void_p()
    assert lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)) == -4           # TGB200_ERR_UNSUPPORTED
    assert b"fp32" in lib.tgb200_last_error() and not h


@pytest.mark.parametrize("precision,limit", [("bf16", 6.0), ("bf16x3", 12.0)])
def test_device_footprint(precision, limit):
    """About 20k x 8k: the device memory a host-state handle takes at creation, per mapping element."""
    N, V, K = 20000, 8192, 64
    torch.cuda.init()
    torch.cuda.synchronize()
    free0, _ = torch.cuda.mem_get_info(0)
    e = Engine(N, V, K, device=0, precision=precision, state_memory="host")
    try:
        torch.cuda.synchronize()
        free1, _ = torch.cuda.mem_get_info(0)
        per_element = (free0 - free1) / (N * V)
        print(f"{precision}: {per_element:.2f} B per element on the device")
        assert per_element < limit
    finally:
        e.close()


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
def test_sharded_host_state_is_bit_identical(precision, nccl_group):
    """A shard on a one-rank NCCL group (its own communicator, the exchange inside tgb200_run) with host state gives the
    resident shard's bits, validation included."""
    N, V, K = 9000, 256, 64
    inp = synthetic_inputs(N, V, K, seed=23)
    M0 = np.random.default_rng(5).standard_normal((N, V)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_g2=0.3, device="cuda:0", M0=M0,
              precision=precision, shard=(1000, 8000), process_group=nccl_group)
    res = Mapper(**kw)
    host = Mapper(**kw, state_memory="host")
    try:
        assert res._own_comm and host._own_comm
        out_r, _ = res.train(5, print_each=None, val_each=2)
        out_h, _ = host.train(5, print_each=None, val_each=2)
        assert same_bits(out_r, out_h)
        assert same_bits(res.history_matrix, host.history_matrix)
        assert same_bits(res.project(inp["S"][1000:8000]), host.project(inp["S"][1000:8000]))
    finally:
        res.release()
        host.release()


@pytest.mark.parametrize("mode", ["cells", "constrained"])
def test_map_cells_to_space_host_state_is_bit_identical(mode, monkeypatch):
    """The public entry point forwards state_memory: the AnnData, the per-gene scores and the history are those of the
    resident call, bit for bit."""
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
    monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", "250")
    got = tg.map_cells_to_space(ad_sc, ad_sp, state_memory="host", **kw)
    assert same_bits(got.X, ref.X)
    a, b = got.uns["train_genes_df"], ref.uns["train_genes_df"]
    assert list(a.index) == list(b.index) and same_bits(a["train_score"].to_numpy(), b["train_score"].to_numpy())
    assert got.uns["training_history"]["total_loss"] == ref.uns["training_history"]["total_loss"]
    if mode == "constrained":
        assert same_bits(np.asarray(got.obs["F_out"]), np.asarray(ref.obs["F_out"]))
