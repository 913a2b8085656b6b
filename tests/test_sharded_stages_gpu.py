"""Each stage of one cell-sharded iteration checked against float64, on one GPU, and tgb200_run's own exchange through a
one-rank NCCL communicator.

W shard handles hold rows shard_rows(N, r, W) of the N cells (n_cells_global = N); the test plays the all-reduce the way
NCCL does it, an fp32 sum of the exchange buffers in rank order copied back into every shard.  At step 1 and step 3:

1. the exchange buffer after step_begin, before the sum: Y_r = P_r^T S_ext,r of the shard's own P, with the forward bound
   of its mode and the shard's own chain (its forward splits -- summed into the buffer by k_sum_planes -- or its bf16
   cell chunks, which accumulate into it directly);
2. the tail: sum_i h_i (the device's own row entropies), sum |M| and sum M^2 over the shard's rows against float64 sums
   within 4 (V + N_r) u sum |term|; tail[3..7] (constrained mode only) exactly 0;
3. the loss stage on the summed buffer: the history row (all 16 columns) and dY_ext bit-identical on every shard, and
   against float64 autograd of the loss of the summed Y_ext with N_global cells and the concatenated M (the KL column
   checks the n_cells_global normalisation of the density);
4. backward and update of every shard from its own inputs, with the checks of tests/test_stages_gpu.py.

Every case asserts, from debug("shape"), the internal path it is there for, so that a change of the split heuristics
cannot quietly take it elsewhere.  Then W = 2, 3, 4 shards against the unsharded handle, the seeded draw of ragged shards
against the unsharded draw, and the sharded handle's refusals.

The one-rank NCCL tests drive tgb200_run's sharded branch (the exchange inside the loop, the buffer moved into NCCL memory
and registered, tgb200_set_comm lending, swapping and dropping communicators) and Mapper(process_group=) on a one-rank
NCCL group.  With one rank the all-reduce is the identity: a missing or mis-sized reduction has no effect there, and only
tests/test_multigpu.py, on two GPUs, can see one.

Observed maxima over all cases, shards and steps, as fractions of each bound (H100 80GB HBM3, 700 W power limit):

    stage                            elementwise   rel-Fro   bias
    exchange Y_r, fp32               0.011         0.038     0.020
    exchange Y_r, bf16x3             0.023         0.13      0.13
    exchange Y_r, bf16               0.56          0.56      0.56     (all-positive density column, 8250-cell chunk)
    tail sum h, sum |M|, sum M^2     0.0003        -         -
    history row of the summed Y      0.0061        -         -
    dY_ext, fp32 / bf16x3            0.12          0.014     0.080
    dY_ext, bf16                     0.97          0.37      0.029    (the bound is dY's own bf16 rounding)
    backward dP, bf16x3              0.021         0.096     0.11
    row-dot                          0.019         0.048     0.059
    update step, fp32 / bf16x3       -             0.11      0.16
    update step, bf16                -             0.56      0.23
    bf16 carry lseT / P~/z~ / h      0.055         0.43      0.017
    row pass log z / 1/z / P         0.35          0.095     0.021

Against the unsharded handle after six steps the largest rel-Frobenius difference is 2.2e-7 in fp32 and bf16x3 (bound
2e-5) and 1.7e-4 in bf16 (bound 2e-2, on m).
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs
from tangram_b200.sharded import shard_rows
from tests.helpers import max_rel, rel_fro
from tests.test_stages_gpu import (ALL_TERMS, LR, U, Run, _bf16_forward_consts, _bf16_round, _check_backward_fp32,
                                   _check_backward_x3, _check_bf16_update_step, _check_carry, _check_forward,
                                   _check_loss_stage, _check_row_pass, _fp32_forward_consts, _state, _torch,
                                   _x3_forward_consts)

pytestmark = pytest.mark.gpu
ERR_STATE, ERR_UNSUPPORTED = -3, -4
ROW_TERMS = dict(lambda_r=1e-3, lambda_l1=1e-7, lambda_l2=1e-7)


class ShardRun:
    """W shard Runs over shard_rows(N, r, W) of one set of inputs and initial mapping, plus the global view the loss
    checkers read (N = N_global)."""

    def __init__(self, precision, N, V, K, W, seed=0, T=0, clusters=False, lam=None):
        self.precision, self.W = precision, W
        self.shards = [Run(precision, N, V, K, seed=seed, T=T, clusters=clusters, lam=lam, rows=shard_rows(N, r, W))
                       for r in range(W)]
        s0 = self.shards[0]
        self.Ke, self.V = s0.Ke, V
        self.glob = SimpleNamespace(precision=precision, N=N, V=V, K=K, T=T, clusters=clusters, lam=s0.lam,
                                    graphs=s0.graphs, G=s0.G, d=s0.d)
        self.bufs = [s.e.exchange_tensor() for s in self.shards]
        self.Ysum = None

    def all_reduce(self):
        """fp32 sum of the exchange buffers in rank order, copied back into every shard; keeps the sum's Y_ext."""
        torch = _torch()
        torch.cuda.synchronize()
        total = self.bufs[0].clone()
        for b in self.bufs[1:]:
            total += b
        for b in self.bufs:
            b.copy_(total)
        torch.cuda.synchronize()
        self.Ysum = total[:self.V * self.Ke].view(self.V, self.Ke).double()

    def step(self):
        for s in self.shards:
            s.e.step_begin()
        self.all_reduce()
        for s in self.shards:
            s.e.step_end(LR)

    def close(self):
        for s in self.shards:
            s.e.close()


def _check_tail(s, M, stats, mode):
    """tail[0..2] = sum_i h_i, sum |M|, sum M^2 over the shard's rows (zero unless a row term needs them), tail[3..7] = 0."""
    tail = s.e.debug("tail").astype(np.float64)
    lam = s.lam
    rows = bool(lam.get("lambda_r") or lam.get("lambda_l1") or lam.get("lambda_l2"))
    aux = bool(lam.get("lambda_l1") or lam.get("lambda_l2"))
    Mv = M[:, :s.V]
    terms = [stats[:, 3] if rows else None, Mv.abs().sum(dim=1) if aux else None, (Mv * Mv).sum(dim=1) if aux else None]
    worst = 0.0
    for k, term in enumerate(terms):
        if term is None:
            assert tail[k] == 0, f"{mode} tail[{k}] = {tail[k]} where no row term needs it"
            continue
        ref, scale = float(term.sum()), float(term.abs().sum())
        bound = 4 * (s.V + s.N) * U * scale
        worst = max(worst, abs(tail[k] - ref) / bound)
        assert abs(tail[k] - ref) <= bound, f"{mode} tail[{k}]: {tail[k]} vs {ref} (bound {bound:.3g})"
    assert not np.any(tail[3:]), f"{mode} tail[3..7] = {tail[3:]} in cells mode"
    print(f"[stage] {mode} tail: max err/bound {worst:.3g}")


def _run_sharded_stages(sr, steps=3, checked=(1, 3)):
    torch = _torch()
    sh = sr.shards
    prec = sr.precision
    for step in range(1, steps + 1):
        pre = [_state(s) for s in sh]
        ts = [s.e.get_state() for s in sh]
        for s in sh:
            s.e.step_begin()
        check = step in checked
        lseT = []
        for i, s in enumerate(sh):
            if not check:
                break
            mode = f"{prec} W{sr.W}[{step}] shard {i}"
            Yr = s.buf("Y", s.Ke)
            stats = s.buf("stats", 4)
            if prec == "bf16":
                if step > 1:
                    _check_carry(s, pre[i][0], f"{mode} carry")
                Ss = _bf16_round(s.S.float() * s.buf("inv_zt").float()[:, None])
                _check_forward(s, Yr, s.nv("Pb")[:, :s.V], *_bf16_forward_consts(s), f"{mode} exchange Y", S=Ss)
                lseT.append(s.buf("lseT"))
            else:
                P = s.nv("Pb" if prec == "bf16x3" else "Pf")
                Pref = _check_row_pass(s, pre[i][0], P, stats, f"{mode} row pass")
                consts = _x3_forward_consts(s) if prec == "bf16x3" else _fp32_forward_consts(s)
                _check_forward(s, Yr, Pref, *consts, f"{mode} exchange Y")
            _check_tail(s, pre[i][0], stats, mode)
        sr.all_reduce()
        for s in sh:
            s.e.step_end(LR)
        if not check:
            continue
        hist = [s.e.history()[-1] for s in sh]
        dY = [s.buf("dY", s.Ke) for s in sh]
        for i in range(1, len(sh)):
            assert np.array_equal(hist[i].view(np.uint32), hist[0].view(np.uint32)), \
                f"step {step}: shard {i} logs {hist[i]}, shard 0 {hist[0]}"
            assert torch.equal(dY[i], dY[0]), f"step {step}: dY_ext of shard {i} differs from shard 0's"
        M_all = torch.cat([p[0] for p in pre])
        _check_loss_stage(sr.glob, sr.Ysum, dY[0], hist[0], M_all, f"{prec} W{sr.W}[{step}] summed")
        for i, s in enumerate(sh):
            mode = f"{prec} W{sr.W}[{step}] shard {i}"
            if prec == "bf16":
                _check_bf16_update_step(s, pre[i], ts[i], lseT[i], mode)
            elif prec == "bf16x3":
                _check_backward_x3(s, pre[i], ts[i], s.buf("stats", 4), s.nv("Pb"), dY[0], mode)
            else:
                _check_backward_fp32(s, pre[i], ts[i], s.buf("stats", 4), s.nv("Pf"), dY[0], mode)


def _ragged(sr, sizes):
    assert [s.N for s in sr.shards] == list(sizes)


def _hits_fp32_splits(sr):
    """SIMT forward splits on every shard: k_sum_planes writes the exchange buffer"""
    _ragged(sr, (781, 780, 780))
    assert all(s.splits > 1 and s.nchunks == 1 for s in sr.shards), [s.splits for s in sr.shards]


def _hits_x3_chain_cut(sr):
    """bf16x3 with one split filling the GPU (264 output tiles): only the 2048-cell cut splits a shard's forward, into
    three chains, and k_sum_planes sums the chain-cut planes.  (At a small V x K the splits that fill the SMs cut the
    chain below 2048 cells first, and the cut itself would not be the reason for the planes.)"""
    _ragged(sr, (4102, 4101))
    for s in sr.shards:
        assert s.splits == 3 and -(-s.N // s.splits) <= 2048, (s.N, s.splits)


def _hits_ke2112(sr):
    """Ke = 2112 > 2048: the backward's one uncut chain on a shard"""
    assert all(s.Ke == 2112 for s in sr.shards)


def _hits_bf16_mixed(sr):
    """rank 0 (8192 cells) runs the 2-chunk pipeline (no planes), rank 1 (8191) one chunk with forward splits"""
    a, b = sr.shards
    assert (a.N, a.nchunks, a.splits) == (8192, 2, 1), (a.N, a.nchunks, a.splits)
    assert b.N == 8191 and b.nchunks == 1 and b.splits > 1, (b.N, b.nchunks, b.splits)


def _hits_bf16_4chunks(sr):
    assert all(s.N == 33000 and s.nchunks == 4 and s.splits == 1 for s in sr.shards)


def _hits_bf16_single_chunk(sr):
    _ragged(sr, (781, 780, 780))
    assert all(s.nchunks == 1 for s in sr.shards)


def _hits_clusters(sr):
    """clusters mode: the density column is sum_i P_ij d_source,i over the pre-sharded rows of d_source, not divided by N"""
    from tangram_b200 import _lib
    assert all(s.e.cfg.density_mode == _lib.DENSITY_SOURCE for s in sr.shards)


def _hits_v5(sr):
    assert all(s.V == 5 and s.ld == 64 for s in sr.shards)


STAGE_CASES = [
    # precision, W, N, V, K, T, clusters, lambdas, the path it must hit
    ("fp32", 3, 2341, 300, 120, 6, False, ALL_TERMS, _hits_fp32_splits),
    ("bf16x3", 2, 8203, 4224, 1994, 6, False, ALL_TERMS, _hits_x3_chain_cut),
    ("bf16x3", 2, 2001, 100, 2100, 0, False, {}, _hits_ke2112),
    ("bf16", 2, 16383, 300, 70, 0, False, ROW_TERMS, _hits_bf16_mixed),
    ("bf16", 2, 66000, 130, 40, 0, False, {"lambda_r": 1e-3}, _hits_bf16_4chunks),
    ("bf16", 3, 2341, 300, 120, 6, False, ALL_TERMS, _hits_bf16_single_chunk),
    ("bf16x3", 2, 1200, 263, 100, 0, True, {}, _hits_clusters),
    ("bf16x3", 2, 601, 5, 60, 0, False, {}, _hits_v5),
]


@pytest.mark.parametrize("precision,W,N,V,K,T,clusters,lam,hits", STAGE_CASES,
                         ids=["fp32-splits", "x3-chain-cut", "x3-Ke2112", "bf16-mixed-chunks", "bf16-4-chunks",
                              "bf16-all-terms", "x3-clusters", "x3-V5"])
def test_sharded_stages(precision, W, N, V, K, T, clusters, lam, hits):
    sr = ShardRun(precision, N, V, K, W, seed=N + V + K, T=T, clusters=clusters, lam=lam)
    try:
        hits(sr)
        _run_sharded_stages(sr)
    finally:
        sr.close()


# ------------------------------------------------------------------------------------------------ against the unsharded handle
def _state_and_mapping(run):
    e = run.e
    M, m, v = (np.empty((run.N, run.V), dtype=np.float32) for _ in range(3))
    step = e.get_state(M, m, v)
    return dict(M=M, m=m, v=v, P=e.get_mapping(np.empty_like(M))), step


@pytest.mark.parametrize("W", [2, 3, 4])
@pytest.mark.parametrize("precision,N,V,K", [("fp32", 2341, 300, 120), ("bf16x3", 2341, 300, 120),
                                             ("bf16", 2341, 300, 120), ("bf16", 16383, 300, 70)])
def test_shards_reproduce_the_unsharded_handle(precision, N, V, K, W):
    """Every term on, N ragged: the shards' mapping, M, m, v and history against one unsharded handle (the same arithmetic
    up to the order of the cell sums), and every shard's history bit-identical to shard 0's."""
    steps, T = 6, 6
    whole = Run(precision, N, V, K, seed=17, T=T, lam=ALL_TERMS)
    for _ in range(steps):
        whole.e.step_begin()
        whole.e.step_end(LR)
    ref, _ = _state_and_mapping(whole)
    ref_h = whole.e.history()
    whole.e.close()
    sr = ShardRun(precision, N, V, K, W, seed=17, T=T, lam=ALL_TERMS)
    try:
        for _ in range(steps):
            sr.step()
        got = [_state_and_mapping(s) for s in sr.shards]
        assert all(step == steps for _, step in got)
        tol = 2e-2 if precision == "bf16" else 2e-5
        for k in ("P", "M", "m", "v"):
            err = rel_fro(np.concatenate([g[k] for g, _ in got]), ref[k])
            print(f"[sharded] {precision} N={N} W={W} {k}: rel-Frobenius {err:.3g} (bound {tol:.3g})")
            assert err < tol, f"{k}: rel-Frobenius {err:.3g}"
        hists = [s.e.history() for s in sr.shards]
        assert max_rel(hists[0][:, 0], ref_h[:, 0]) < (1e-3 if precision == "bf16" else 1e-5)
        for h in hists[1:]:
            assert np.array_equal(h.view(np.uint32), hists[0].view(np.uint32)), "every shard logs the same history, bit for bit"
    finally:
        sr.close()


# ------------------------------------------------------------------------------------------------------ draws and refusals
def test_seeded_draw_of_ragged_shards_is_the_unsharded_draw():
    """init_mapping_normal(seed, first_row=r0) on each of three ragged shards (V % 4 != 0, so a row does not start on a
    float4 of the stream) gives rows [r0, r1) of the unsharded draw, bit for bit."""
    from tangram_b200.engine import Engine
    N, V, K, W, seed = 1001, 77, 30, 3, 11
    whole = Engine(N, V, K)
    whole.init_mapping_normal(seed)
    want = np.empty((N, V), dtype=np.float32)
    whole.get_state(M=want)
    whole.close()
    assert np.isfinite(want).all() and want.std() > 0.5
    for r in range(W):
        r0, r1 = shard_rows(N, r, W)
        e = Engine(r1 - r0, V, K, n_cells_global=N)
        e.init_mapping_normal(seed, first_row=r0)
        got = np.empty((r1 - r0, V), dtype=np.float32)
        e.get_state(M=got)
        e.close()
        assert np.array_equal(got.view(np.uint32), want[r0:r1].view(np.uint32)), f"shard {r} rows [{r0}, {r1})"


def test_sharded_handle_refusals():
    """A sharded handle refuses validation (set_validation(k > 0), validation_terms) with UNSUPPORTED, and its exchange
    buffer is V Ke + 8 floats: Y_ext and the tail."""
    from tangram_b200 import _lib
    s = Run("bf16x3", 1000, 70, 40, seed=1, rows=(0, 600))
    e, lib = s.e, s.e._lib
    assert lib.tgb200_set_validation(e._h, 1, None) == ERR_UNSUPPORTED
    assert lib.tgb200_set_validation(e._h, 0, None) == 0
    out = np.zeros(4, dtype=np.float32)
    assert lib.tgb200_validation_terms(e._h, _lib.ptr(out), None) == ERR_UNSUPPORTED
    p, n = ctypes.c_void_p(), ctypes.c_int64()
    assert lib.tgb200_exchange_buffer(e._h, ctypes.byref(p), ctypes.byref(n)) == 0
    assert n.value == 70 * s.Ke + 8 and e.exchange_tensor().numel() == n.value
    assert lib.tgb200_run(e._h, 1, LR, None) == ERR_STATE          # no communicator: the caller drives the exchange
    e.close()


# ------------------------------------------------------------------------------------- tgb200_run on a one-rank communicator
class _Nccl:
    """One-rank NCCL communicators and the handles that use them: handles are closed before the communicators are
    destroyed."""

    def __init__(self, lib):
        self.lib, self.comms, self.engines = lib, [], []

    def comm(self):
        from tangram_b200 import _lib
        uid = np.zeros(128, dtype=np.uint8)
        _lib.check(self.lib.tgb200_comm_unique_id(_lib.ptr(uid), uid.nbytes))
        c = ctypes.c_void_p()
        _lib.check(self.lib.tgb200_comm_create(_lib.ptr(uid), 0, 1, 0, ctypes.byref(c)))
        self.comms.append(c)
        return c

    def track(self, run):
        self.engines.append(run.e)
        return run

    def close(self):
        for e in self.engines:
            e.close()
        for c in self.comms:
            self.lib.tgb200_comm_destroy(c)


@pytest.fixture
def nccl(monkeypatch):
    from tangram_b200 import _lib
    _torch()                                  # the libnccl.so.2 torch loaded is the one the library binds
    lib = _lib.load()
    monkeypatch.setenv("NCCL_SOCKET_IFNAME", "lo")
    uid = np.zeros(128, dtype=np.uint8)
    if lib.tgb200_comm_unique_id(_lib.ptr(uid), uid.nbytes) != 0:
        pytest.skip(f"no NCCL in this process: {lib.tgb200_last_error().decode()}")
    n = _Nccl(lib)
    yield n
    n.close()


def _same(a, b, what):
    """bit-identical history, M, m, v and mapping of two handles"""
    (sa, ta), (sb, tb) = _state_and_mapping(a), _state_and_mapping(b)
    assert ta == tb, f"{what}: step {ta} vs {tb}"
    ha, hb = a.e.history(), b.e.history()
    assert np.array_equal(ha.view(np.uint32), hb.view(np.uint32)), f"{what}: history"
    for k in ("M", "m", "v", "P"):
        assert np.array_equal(sa[k].view(np.uint32), sb[k].view(np.uint32)), \
            f"{what}: {k} differs in {int((sa[k] != sb[k]).sum())} elements"


def _manual(run, n):
    for _ in range(n):
        run.e.step_begin()
        run.e.step_end(LR)


RUN_CASES = [("fp32", 1200, 300, 120, 1), ("bf16x3", 1200, 300, 120, 1), ("bf16", 1200, 300, 120, 1),
             ("bf16", 9000, 300, 70, 2), ("bf16", 33000, 130, 40, 4)]


@pytest.mark.parametrize("precision,Nr,V,K,chunks", RUN_CASES, ids=["fp32", "bf16x3", "bf16", "bf16-2chunks", "bf16-4chunks"])
def test_run_with_a_one_rank_communicator_is_the_manual_loop(nccl, precision, Nr, V, K, chunks):
    """A shard (n_cells_global = 2 N_r) holding a one-rank communicator, driven by run(6) and by run(3) + run(3), against
    its twin driven by six step_begin / step_end pairs: history, M, m, v and mapping bit-identical.  In bf16 with 2 and 4
    cell chunks run() also issues the next forward beside the exchange."""
    lam = dict(ROW_TERMS, lambda_g2=0.3)

    def shard():
        return nccl.track(Run(precision, 2 * Nr, V, K, seed=Nr, lam=lam, rows=(0, Nr)))

    a6, a33, twin = shard(), shard(), shard()
    assert twin.nchunks == chunks
    c = nccl.comm()
    a6.e.set_comm(c, 0, 1)
    a33.e.set_comm(c, 0, 1)
    a6.e.run(6, LR)
    a33.e.run(3, LR)
    a33.e.run(3, LR)
    _manual(twin, 6)
    _same(a6, twin, "run(6)")
    _same(a33, twin, "run(3) + run(3)")


def _buffer_moved(run, comm):
    """Lend `comm` (None: drop it); the exchange buffer keeps its contents bit for bit and exchange_tensor() views the
    buffer the handle uses.  -> whether its address changed (a buffer re-allocated at the address just freed keeps it)."""
    torch = _torch()
    before = run.e.exchange_tensor()
    old_ptr, old = before.data_ptr(), before.clone()
    run.e.set_comm(comm, 0, 1)
    now = run.e.exchange_tensor()
    assert torch.equal(now.view(torch.int32), old.view(torch.int32)), "the exchange buffer's contents changed"
    x0 = float(now[0])
    now[0] = 12345.0
    torch.cuda.synchronize()
    assert run.e.debug("Y")[0] == 12345.0, "exchange_tensor() does not view the handle's buffer"
    now[0] = x0
    torch.cuda.synchronize()
    return now.data_ptr() != old_ptr


def test_communicator_lifecycle(nccl):
    """Lend c1, swap to c2, drop it: the exchange buffer survives each move bit for bit, exchange_tensor() follows it,
    run() without a communicator is a STATE error, and training (run() while a communicator is lent, the manual loop
    after) still equals the twin's manual loop."""
    Nr, V, K = 1000, 300, 120

    def shard():
        return nccl.track(Run("bf16x3", 2 * Nr, V, K, seed=4, lam=ROW_TERMS, rows=(0, Nr)))

    h, twin = shard(), shard()
    lib = h.e._lib
    assert lib.tgb200_run(h.e._h, 1, LR, None) == ERR_STATE
    _manual(h, 2)
    _manual(twin, 2)
    for name, comm in (("c1", nccl.comm()), ("c2", nccl.comm()), ("none", None)):
        moved = _buffer_moved(h, comm)
        print(f"[sharded] set_comm({name}): exchange buffer address {'changed' if moved else 'unchanged'}")
        if comm is None:
            assert lib.tgb200_run(h.e._h, 1, LR, None) == ERR_STATE
            _manual(h, 2)
        else:
            h.e.run(2, LR)
        _manual(twin, 2)
        _same(h, twin, f"after set_comm({name})")


def test_mapper_on_a_one_rank_nccl_group(nccl):
    """Mapper(process_group=, shard=) on a one-rank NCCL group gets its own communicator, and its train() equals the
    manual loop on the same shard bit for bit."""
    import torch.distributed as dist

    from tangram_b200 import Mapper
    N, V, K = 2400, 300, 120
    inp = synthetic_inputs(N, V, K, seed=21)
    M0 = np.random.default_rng(5).standard_normal((N, V)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-3, lambda_g2=0.3, device="cuda:0", M0=M0,
              shard=(600, 1800))
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1)
    try:
        m = Mapper(process_group=dist.group.WORLD, **kw)
        twin = Mapper(**kw)
        try:
            assert m._sharded and m._own_comm and twin._sharded and not twin._own_comm
            out, _ = m.train(6, print_each=None)
            twin._engine.reset_adam()
            for _ in range(6):
                twin._engine.step_begin()
                twin._engine.step_end(0.1)
            want = twin._engine.get_mapping(np.empty_like(out))
            assert np.array_equal(out.view(np.uint32), want.view(np.uint32))
            assert np.array_equal(m.history_matrix.view(np.uint32), twin._engine.history().view(np.uint32))
        finally:
            m.release()
            twin.release()
    finally:
        dist.destroy_process_group()
