"""Each stage of the bf16x3 and fp32 iterations checked against float64 at the benchmark's own sizes -- C3 (100k cells x
10k voxels x 2k genes) and, in bf16x3, C5 (50k x 5k x 2k with the spatial terms) -- and on a mapping of 224,000 x 10,000
(2.25e9 elements), where bf16x3's three P planes of N x ld elements start at element 0, 2.25e9 and 4.5e9 of one
allocation, so that every access to the mid and lo planes, and to dP past row 213,722, is a 64-bit offset.

bf16x3 is the default precision of map_cells_to_space, Mapper and MapperConstrained; fp32 is bench.py's --precision fp32.
tests/test_fullsize_gpu.py holds them only in aggregate (Y within 1e-5, loss and mapping within 1e-4 of the oracle), and
tests/test_stages_gpu.py / tests/test_clusters_stages_gpu.py check their stages at a few thousand rows at most.  Here the
path each size takes is asserted first (debug("shape") against the launch arithmetic of tc_forward_splits,
tc_splits_for_chain and the SIMT forward's grid), then every stage is checked on row blocks with the plumbing of
tests/test_scale_stages_gpu.py: debug() buffers read once into float32 host arrays, uploaded a block at a time, checked in
float64; _Blocks accumulates the statistics across blocks; the forward's reference P^T S_ext is summed over every row.

Bounds (u = 2^-24, u_b = 2^-8), each from the kernel that runs:

* Row pass (k_softmax_rows, fp32 P; in bf16x3 split3 into three bf16 planes that reconstruct it exactly):
  _check_row_pass_tight's bounds of the bucket row_pass_layout picks at this ld (C3: 1024 threads x 3 float4, C5:
  512 x 3), P within cP P (no bf16 rounding), statistics 0.5 / 0.25.
* bf16x3 forward: _x3_contraction_consts(chain, splits) with the handle's own chain (2048 cells, the cut of
  tc_splits_for_chain) and split count (49 at C3, 25 at C5, 110 at 224k), against P^T S_ext of the device's own P.
* fp32 forward (k_gemm_simt, EpiStorePartial): one round-to-nearest FFMA chain of `chain` cells per output (100,000 at
  C3, where 79 x 16 output tiles already fill the grid and splits = 1; 112,000 at 224k, 2 splits) plus the fp32 sum of
  the splits.  Elementwise (2 chain + splits + 4) u, 1.2e-2 at C3: a worst case that proves little.  The statistics carry
  the check.  Each FFMA rounds its partial sum s_k to nearest, an error uniform within half an ulp, so
  E[e_k^2] <= u^2 s_k^2 / 3; with same-sign terms s_k ~ (k / n) s_n and the n errors independent, sum_k E[e_k^2] ~
  u^2 s_n^2 n / 9, an rms of sqrt(n) u / 3 of sum |a b| (at C4's 256-cell chain tests/test_clusters_stages_gpu.py
  observes 0.33 sqrt(n) u).  rel-Fro <= sqrt(chain) u + (splits + 4) u is three times that.  Round to nearest is
  unbiased, so the signed mean over `count` outputs is held to the split sum's (splits + 4) u plus four standard errors,
  4 sqrt(chain) u / (3 sqrt(count)).  A dropped 128-cell k-block (1.3e-3 relative) is 65 times the rel-Fro bound.
* Loss stage: _check_loss_stage_tight (loss_layout), at C5 with the neighbourhood, islands and Getis-Ord terms on the
  benchmark's grid graph, L2 and entropy from the row pass.
* bf16x3 dP (TcEpiDpStoreF32, one uncut wgmma chain over Ke): _x3_contraction_consts(Ke)'s elementwise bound,
  X3_BWD_FRO / X3_BWD_BIAS, pad columns exactly zero.
* bf16x3 row-dot: (64 + 2 + r_parts + 1) u sum |P dP| against the device's own P and dP.  fp32 row-dot (EpiRowDot, a
  V-long FFMA chain of P dY_ext, dotted with S_ext over Ke): _check_backward_fp32_rows' (2 (Ke + V) + 8) u, 4 sqrt(Ke + V) u
  and 4 u + 4 sqrt((Ke + V) / rows) u over the rows checked.
* Update (k_adam_rows_exact through staged_rows in bf16x3, the fused EpiAdam in fp32): _check_update's elementwise
  bounds on M, m, v, pad columns zero, and the step's rel-Fro 256 u and bias 32 u plus the rounding of M' itself: at
  10,000 voxels g is far below Adam's eps, so a step is a few thousand ulps of M or less.  Its u |M'| adds to the
  rel-Fro bound as in _late_step_consts; to the bias, four standard errors of a uniform rounding where the step spans
  more than 32 ulps, and u |M'| only where it does not (there the rounding need not cancel: below half an ulp M' = M).
  In bf16x3 without gradient terms (C3, 224k) M, m, v also equal torch.optim.Adam bit for bit in every row block.

Observed maxima over C3, C5 and the 2^31 windows, steps 1..3, as fractions of each bound (H100 80GB HBM3, 700 W power
limit):

    stage                               elementwise   rel-Fro   bias
    row pass log z, bf16x3 / fp32          0.21          0.15      0.066
    row pass 1 / z                         0.14          0.073     0.024
    row pass P                             0.34          0.097     0.008
    row pass h (C5)                        0.084         0.04      0.0033
    forward Y genes, bf16x3                0.036         0.19      0.19
    forward Y density / ct, bf16x3         0.0065        0.011     0.0027
    forward Y genes, fp32                  0.0014        0.15      0.034
    forward Y density, fp32                0.0018        0.26      0.12
    dY_ext genes                           0.034         0.0076    0.00024
    dY_ext density                         0.24          0.25      0.0099
    dP, bf16x3                             0.0063        0.075     0.11
    row-dot, bf16x3                        0.073         0.032     0.0035
    row-dot, fp32                          0.0035        0.046     0.025
    update M / m / v                       0.19          0.053     0.0042
    update step                            -             0.39      0.0053
    history columns                        9.4e-05       -         -

The forward's statistics are what holds fp32 at C3: its elementwise bound is 1.2e-2 relative, its rel-Fro bound 1.9e-5.
The step's bias bound is still dominated by its steps within 32 ulps of M'; its rel-Fro carries the check.

Each case prints its path ("[path]") and its peak device use, sampled device-wide at every block upload and state copy,
and the process's peak host RSS ("[memory]"): 44.7 GiB at C3 in bf16x3, 15.0 GiB at C5, 34.1 GiB at C3 in fp32, 58.5 /
37.5 GiB for run() against step pairs (two handles), 49.4 GiB past 2^31 in bf16x3 and 35.4 GiB in fp32; host RSS 25 GiB
through the benchmark-size cases, 40 GiB once the bf16x3 host-state handle pins its 27 GB.  The benchmark-size cases and
run() take about 4 minutes, the two cases past 2^31 another 6, so the file about 10 minutes.

Planted errors, each built into a copy of the library and run once at its case (H100 80GB HBM3, 700 W):

* A stale dP tile: TcEpiDpStoreF32 never stores the 128 x 256 dP tile at column tile 0 of the last full row tile
  (rows 99,840..99,967 at C3); the row-dot still sums it.  The C3 bf16x3 case fails at step 1: dP at 8,500 times its
  bound, first at row 99,840.  tests/test_fullsize_gpu.py at C3 fails too: the bf16x3 mapping's rel-Frobenius against
  the oracle is 8.1e-4 (bound 1e-4; 1.7e-7 without the error), while Y (2.9e-6) and the loss trajectory (5.9e-6) stay
  within theirs.
* A 32-bit plane offset: split3 stores the lo plane at (uint32_t)(2 plane + offset), so at 224k, where 2 plane is
  4.5e9 elements, every row's lo plane lands in plane 0 from element 206,536,704 on and the real lo plane is never
  written.  The 224k bf16x3 case fails at step 1: the row pass's P at 2,200 times its bound, on row 0.
  tests/test_fullsize_gpu.py passes with it: at C3, C4 and C5 2 plane + offset stays below 2^32, so the library
  computes what it computed before.
* A skipped ragged tile: the fp32 EpiAdam returns on the last column tile, voxels 9,984..10,111 of which 16 are live.
  The C3 fp32 case fails at step 1: update M at 1.7 times its bound, first at voxel 9,986 of row 0 (M there keeps its
  old value; m and v, 0 before the first step, would fail by far more).  tests/test_fullsize_gpu.py has no fp32 leg, so
  it cannot see this error.
"""
import ctypes
import hashlib

import numpy as np
import pytest

from tests.test_clusters_stages_gpu import (BIAS, FRO, _Blocks, _cdiv, _check_loss_stage_tight, _row_pass_consts,
                                            _row_pass_h_bound, row_pass_layout)
from tests.test_scale_stages_gpu import (BLOCK, CROSS, GIB, _big_windows, _big_work, _bench_work, _blocks, _finish,
                                         _HostRows, _need, _pre_state, _report_memory, _round_up, _sample)
from tests.test_stages_gpu import (B1, B2, EPS, LR, U, X3_BWD_BIAS, X3_BWD_FRO, _adam64, _check, _check_forward,
                                   _grad_terms, _torch, _x3_contraction_consts)

__all__ = ["_report_memory"]       # the autouse fixture that prints each case's "[memory]" line


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


pytestmark = [pytest.mark.gpu, pytest.mark.skipif(_no_gpu(), reason="needs an H100 GPU")]


# ------------------------------------------------------------------------------------------------------------- plumbing
def _plan(N, V, K, T, precision, lam=None, state_memory="device"):
    """tgb200_plan_state for a handle of this shape: its device bytes (operands and resident state), the reserve it
    leaves free and the pinned host bytes of its host rows"""
    from tangram_b200 import _lib
    from tangram_b200.engine import plan_state
    cfg = _lib.Config()
    cfg.struct_size = ctypes.sizeof(_lib.Config)
    cfg.n_cells, cfg.n_voxels, cfg.n_genes, cfg.n_types, cfg.n_cells_global = N, V, K, T, N
    cfg.precision, cfg.density_mode = _lib.PREC[precision], _lib.DENSITY_CELLS
    cfg.state_memory = _lib.STATE_MEMORY[state_memory]
    for k, x in (lam or {}).items():
        setattr(cfg, k, x)
    return plan_state(cfg, 1 << 62)


def _planned_gib(N, V, K, T, precision, lam=None, state_memory="device"):
    """device memory planned for a handle of this shape (operands, resident state and the reserve)"""
    p = _plan(N, V, K, T, precision, lam, state_memory)
    return (p.device_bytes + p.reserve_bytes) / GIB


class _PreRows:
    """The handle's pre-step M, m, v (float32) on the rows of `wins` and its step count: all of it on the device
    (_pre_state), or read one component at a time through one host buffer and cut down to the windows."""

    def __init__(self, r, wins, on_device):
        torch = _torch()
        if on_device:
            (M, m, v), self.t = _pre_state(r)
            self.parts = [(0, r.N, (M, m, v))]
            return
        buf = np.empty((r.N, r.V), dtype=np.float32)
        keep = {w: [] for w in wins}
        for name in "Mmv":
            self.t = r.e.get_state(**{name: buf})
            torch.cuda.synchronize()
            for a, b in wins:
                keep[(a, b)].append(buf[a:b].copy())
        del buf
        self.parts = [(a, b, tuple(keep[(a, b)])) for a, b in wins]

    def get(self, a, b):
        torch = _torch()
        for w0, w1, xs in self.parts:
            if w0 <= a and b <= w1:
                out = tuple(torch.from_numpy(x[a - w0:b - w0]).to("cuda") if isinstance(x, np.ndarray) else x[a - w0:b - w0]
                            for x in xs)
                _sample()
                return out
        raise KeyError((a, b))


def _chain(r):
    """cells per forward chain: the tensor-core k-split rounds to 64-cell k-blocks, the SIMT one to 16"""
    return min(r.N, _round_up(_cdiv(r.N, r.splits), 64 if r.precision == "bf16x3" else 16))


def _assert_path(r, ld, Ke, splits):
    """debug("shape") against the launch arithmetic: ld, Ke, one cell chunk, the forward's split count and chain (bf16x3:
    at most 2048 cells), the row-dot's partials (bf16x3: one per 256-voxel tile; fp32: one per 128-column SIMT tile)"""
    chain = _chain(r)
    last = r.N - (r.splits - 1) * chain
    assert (r.ld, r.Ke, r.nchunks) == (ld, Ke, 1), (r.ld, r.Ke, r.nchunks)
    assert r.splits == splits and 0 < last <= chain, f"{r.splits} forward splits of {chain} cells, the last {last}"
    if r.precision == "bf16x3":
        assert chain <= 2048 and r.rparts == _cdiv(r.V, 256), (chain, r.rparts)
    else:
        assert r.rparts == _cdiv(r.Ke, 128), r.rparts
    print(f"[path] {r.name} {r.precision}: ld {r.ld}, Ke {r.Ke}, one cell chunk, {r.splits} forward splits of {chain} "
          f"cells (the last {last}), {r.rparts} row-dot partials")


# ------------------------------------------------------------------------------------------------------------- stages
def _row_pass_blocks(r, pre, P, stats, wins, res, mode):
    """tests/test_clusters_stages_gpu.py::_check_row_pass_tight on row blocks: log z, 1 / z, P (fp32, or bf16x3's three
    planes summed), pad columns zero, h where the entropy term is on"""
    torch = _torch()
    V = r.V
    lz = _Blocks(f"{mode} log z", 1.0, FRO, BIAS)
    iz_ = _Blocks(f"{mode} 1 / z", 1.0, FRO, BIAS)
    pp = _Blocks(f"{mode} P", 1.0, FRO, BIAS)
    hh = _Blocks(f"{mode} h", 1.0, FRO, BIAS) if r.lam.get("lambda_r") else None
    for a, b in _blocks(wins, BLOCK):
        M = pre.get(a, b)[0].double()
        st = stats[a:b]
        Pr, mx, logz, cz, c_logz, cP, dist = _row_pass_consts(r, M)
        assert torch.equal(st[:, 0], mx), f"{mode}: row max, rows {a}..{b}"
        lz.add(st[:, 2], logz, c_logz)
        iz = torch.exp(-logz)
        iz_.add(st[:, 1], iz, (cz + U) * iz)
        x = P.get(a, b)
        pp.add(x[:, :V], Pr, cP * Pr)
        assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of P, rows {a}..{b}"
        if hh is not None:
            logP = torch.log_softmax(M, dim=1)
            hh.add(st[:, 3], (Pr * logP).sum(dim=1), _row_pass_h_bound(r, Pr, logP, cP, dist, c_logz))
        del M, Pr, x, cP, dist
    _finish(res, *[x for x in (lz, iz_, pp, hh) if x is not None])


def _fp32_forward(r, Y, ref, mode):
    """the fp32 forward's gene, density and cell-type columns with the docstring's chain-structure statistics"""
    K, T = r.K, r.T
    chain = _chain(r)
    Yref, scale = ref
    ce, cf = (2 * chain + r.splits + 4) * U, np.sqrt(chain) * U + (r.splits + 4) * U
    out = {}
    parts = [("Y genes", Y[:, :K], Yref[:, :K], scale[:, :K]),
             ("Y density", Y[:, K] + Y[:, K + 1], Yref[:, K] + Yref[:, K + 1], scale[:, K] + scale[:, K + 1])]
    if T:
        parts.append(("Y ct", Y[:, K + 2:K + 2 + T], Yref[:, K + 2:K + 2 + T], scale[:, K + 2:K + 2 + T]))
    for what, got, want, sc in parts:
        cb = (r.splits + 4) * U + 4 * np.sqrt(chain) * U / (3 * np.sqrt(got.numel()))
        out[what] = _check(f"{mode} {what}", got, want, sc, ce, cf, cb)
    assert _torch().count_nonzero(Y[:, K + 2 + T:]) == 0, "Y_ext past the last used column"
    return out


class _Update:
    """tests/test_stages_gpu.py::_check_update on row blocks: M, m, v elementwise (pad columns zero), the step's
    statistics accumulated"""

    def __init__(self, mode):
        self.acc = [_Blocks(f"{mode} update {x}", 1.0, 1.0, 1.0) for x in ("M", "m", "v")]
        self.step = _Blocks(f"{mode} update step", 1e30, 256 * U, 32 * U)
        self.mode, self.rnd2, self.near, self.far2 = mode, 0.0, 0.0, 0.0

    def add(self, r, pre, post, g, dg, t, a, b):
        torch = _torch()
        V = r.V
        M0, m0, v0 = (x.double() for x in pre)
        Mr, mr, vr, dM, dm, dv = _adam64(M0, m0, v0, g, dg, t)
        for acc, x, ref, bound, name in zip(self.acc, post, (Mr, mr, vr), (dM, dm, dv), "Mmv"):
            assert torch.count_nonzero(x[:, V:]) == 0, f"{self.mode}: pad columns of {name}, rows {a}..{b}"
            acc.add(x[:, :V], ref, bound)
        stepref = M0 - Mr
        scale = stepref.abs() + dM
        self.step.add(M0 - post[0][:, :V], stepref, scale)
        # The rounding of M' itself, up to u |M'| (tests/test_stages_gpu.py::_late_step_consts): at 10,000 voxels
        # g = P (dP - r) is far below Adam's eps, so a step is a few thousand ulps of M or less and M''s rounding is a
        # visible part of its error.  Its square adds to the rel-Fro bound.  For the bias: round to nearest of a step of
        # many ulps is unbiased, so those elements add four standard errors of a uniform rounding (u |M'| / sqrt(3) of
        # each); a step within 32 ulps of M' (64 u |M'|, an ulp being at most 2 u |M'|) lands on the grid in a pattern
        # that need not cancel (below half an ulp M' = M and the step is lost, one-sided), so those add u |M'| each.
        rnd = U * post[0][:, :V].abs()
        live = scale > 0
        x = rnd[live] / scale[live]
        near = stepref.abs()[live] < 64 * rnd[live]
        self.rnd2 += float((rnd * rnd).sum())
        self.near += float(x[near].sum())
        self.far2 += float((x[~near] ** 2).sum())

    def done(self, res):
        st = self.step
        if st.s2:
            st.c_fro += (self.rnd2 / st.s2) ** 0.5
            st.c_bias += (self.near + 4 * (self.far2 / 3) ** 0.5) / st.n
        _finish(res, *self.acc, st)


def _torch_adam(pre, post, g, t, what):
    """one torch.optim.Adam step (foreach=False, on CUDA) from the device's fp32 state and gradient equals M, m, v"""
    torch = _torch()
    M0, m0, v0 = (x.contiguous() for x in pre)
    p = torch.nn.Parameter(M0.clone())
    opt = torch.optim.Adam([p], lr=LR, betas=(B1, B2), eps=EPS, foreach=False, fused=False)
    p.grad = g
    opt.state[p] = {"step": torch.tensor(float(t)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    opt.step()
    V = M0.shape[1]
    for name, got, want in (("v", post[2], opt.state[p]["exp_avg_sq"]), ("m", post[1], opt.state[p]["exp_avg"]),
                            ("M", post[0], p.detach())):
        diff = got[:, :V].float() != want
        assert not bool(diff.any()), f"{what}: {name} differs from torch's Adam in {int(diff.sum())} of {diff.numel()} elements"


def _backward_x3(r, pre, t, stats, rdot, P, dY, post, wins, res, mode):
    """dP, the row-dot and the exact update on row blocks"""
    torch = _torch()
    V, N, ld, Ke = r.V, r.N, r.ld, r.Ke
    dpa = _Blocks(f"{mode} dP (Ke {Ke})", _x3_contraction_consts(Ke)[0], X3_BWD_FRO, X3_BWD_BIAS)
    rda = _Blocks(f"{mode} row-dot ({r.rparts} partials)", 1.0, FRO, BIAS)
    upd = _Update(mode)
    dpf = _HostRows(r.e, "dpf", N, ld, wins)
    exact = 0
    for a, b in _blocks(wins, BLOCK):
        S = r.S[a:b]
        q = dpf.get(a, b)
        assert torch.count_nonzero(q[:, V:]) == 0, f"{mode}: pad columns of dP, rows {a}..{b}"
        q = q[:, :V]
        dpa.add(q, S @ dY.t(), S.abs() @ dY.abs().t())
        p = P.get(a, b)[:, :V]
        pd = p * q
        rda.add(rdot[a:b], pd.sum(dim=1), (64 + 2 + r.rparts + 1) * U * pd.abs().sum(dim=1))
        del pd
        st, rd = stats[a:b], rdot[a:b]
        pb = pre.get(a, b)
        g = _grad_terms(r, pb[0].double(), p, q - rd[:, None], st[:, 0] + st[:, 2], st[:, 3])
        if r.lam:
            dg = 8 * U * (g.abs() + p * (q.abs() + rd.abs()[:, None] + 1.0))
        else:
            dg = 4 * U * (g.abs() + p * (q.abs() + rd.abs()[:, None]))
        pst = [x.get(a, b) for x in post]
        upd.add(r, pb, pst, g, dg, t + 1, a, b)
        del g, dg
        if not r.lam:
            _torch_adam(pb, pst, (q.float() - rd.float()[:, None]) * p.float(), t, f"{mode} rows {a}..{b}")
            exact += b - a
        del p, q, pst, pb
    _finish(res, dpa, rda)
    upd.done(res)
    if exact:
        print(f"[stage] {mode} update: M, m, v of {exact} rows bit-identical to torch.optim.Adam")


def _backward_fp32(r, pre, t, stats, rdot, P, dY, post, wins, res, mode):
    """tests/test_clusters_stages_gpu.py::_check_backward_fp32_rows on row blocks: the row-dot, and the fused EpiAdam
    update with dP recomputed in float64 from the device's S_ext and dY_ext"""
    V, Ke = r.V, r.Ke
    n = Ke + V
    rows = sum(b - a for a, b in wins)
    rda = _Blocks(f"{mode} row-dot ({r.rparts} partials)", (2 * n + 8) * U, 4 * np.sqrt(n) * U,
                  4 * U + 4 * np.sqrt(n / rows) * U)
    upd = _Update(mode)
    for a, b in _blocks(wins, BLOCK):
        S = r.S[a:b]
        dPref = S @ dY.t()
        scale = S.abs() @ dY.abs().t()
        p = P.get(a, b)[:, :V]
        rd, st = rdot[a:b], stats[a:b]
        rda.add(rd, (p * dPref).sum(dim=1), (p * scale).sum(dim=1))
        pb = pre.get(a, b)
        g = _grad_terms(r, pb[0].double(), p, dPref - rd[:, None], st[:, 0] + st[:, 2], st[:, 3])
        dg = p * (2 * Ke + 8) * U * scale + 8 * U * (g.abs() + p * (dPref.abs() + rd.abs()[:, None] + 1.0))
        del scale
        upd.add(r, pb, [x.get(a, b) for x in post], g, dg, t + 1, a, b)
        del g, dg, dPref, p, pb
    _finish(res, rda)
    upd.done(res)


def _stage_step(r, step, wins, pre_on_device=True, M_loss64=False):
    """one step_begin / step_end pair with every stage checked on the rows of `wins` (the forward's Y in full)"""
    torch = _torch()
    V, N, ld, Ke = r.V, r.N, r.ld, r.Ke
    x3 = r.precision == "bf16x3"
    pre = _PreRows(r, wins, pre_on_device)
    t = pre.t
    assert t == step - 1
    mode = f"{r.name} {r.precision}[{step}]"
    res = {}
    M_loss = pre.parts[0][2][0].double() if M_loss64 else torch.zeros((1, V), dtype=torch.float64, device="cuda")
    r.e.step_begin()
    r.e.step_end(LR)
    stats, rdot = r.buf("stats", 4), r.buf("rdot")
    Yref = torch.zeros((V, Ke), dtype=torch.float64, device="cuda")
    Ysc = torch.zeros_like(Yref)

    def fwd(a, b, x):
        Pb = torch.from_numpy(x[:, :V]).to("cuda").double()
        Yref.addmm_(Pb.t(), r.S[a:b])
        Ysc.addmm_(Pb.t(), r.S[a:b].abs())

    P = _HostRows(r.e, "Pb" if x3 else "Pf", N, ld, wins, visit=fwd)
    _row_pass_blocks(r, pre, P, stats, wins, res, f"{mode} row pass")
    Y = r.buf("Y", Ke)
    if x3:
        out = _check_forward(r, Y, None, *_x3_contraction_consts(_chain(r), r.splits), mode=mode, ref=(Yref, Ysc))
    else:
        out = _fp32_forward(r, Y, (Yref, Ysc), mode)
    res.update({f"{mode} {k}": x for k, x in out.items()})
    del Yref, Ysc
    dY = r.buf("dY", Ke)
    threads, _, per = row_pass_layout(ld)
    _check_loss_stage_tight(r, Y, dY, r.e.history()[-1], M_loss, stats, per + 2 + int(np.log2(threads)), mode)
    del Y, M_loss
    post = [_HostRows(r.e, name, N, ld, wins) for name in "Mmv"]
    (_backward_x3 if x3 else _backward_fp32)(r, pre, t, stats, rdot, P, dY, post, wins, res, mode)
    del pre, post, P, dY
    torch.cuda.empty_cache()
    return res


# ======================================================================================== 1, 2. the benchmark's sizes
# id: (workload, precision, ld, Ke, forward splits)
BENCH = {"c3-bf16x3": ("c3", "bf16x3", 10048, 2048, 49), "c5-bf16x3": ("c5", "bf16x3", 5056, 2048, 25),
         "c3-fp32": ("c3", "fp32", 10048, 2048, 1)}


@pytest.mark.parametrize("case", list(BENCH))
def test_stages_at_benchmark_size(case):
    """bench.gen_inputs' workload: the row pass, the forward, the loss stage, dP (bf16x3), the row-dot and the update at
    steps 1, 2 and 3 on every row."""
    import bench
    name, precision, ld, Ke, splits = BENCH[case]
    N, V, K, T = bench.WORKLOADS[name][:4]
    lam = dict(bench.C5_LAMBDAS) if name == "c5" else {}
    # the handle, the pre-step state (3 N x V floats) and the float64 block temporaries; host: P, dP and the post-step
    # state read back as float32
    _need(_planned_gib(N, V, K, T, precision, lam) + 12 * N * V / GIB + 8, 24 * N * V / GIB + 8)
    r = _bench_work(name, precision=precision)
    _assert_path(r, ld, Ke, splits)
    for step in (1, 2, 3):
        _stage_step(r, step, [(0, r.N)], M_loss64=name == "c5")
    r.e.close()


# ============================================================================================ 4. run() = step pairs
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
def test_c3_run_matches_step_pairs(precision):
    """C3: run(3) leaves M, m, v, every debug buffer and the history bit-identical to three step_begin / step_end pairs."""
    import bench
    torch = _torch()
    N, V, K, T = bench.WORKLOADS["c3"][:4]
    _need(2 * _planned_gib(N, V, K, T, precision) + 2, 16 * N * V / GIB + 8)
    a = _bench_work("c3", precision=precision)
    for _ in range(3):
        a.e.step_begin()
        a.e.step_end(LR)
    b = _bench_work("c3", precision=precision)
    b.e.run(3)
    _sample()
    names = ["Y", "dY", "M", "m", "v", "stats", "rdot"] + (["Pb", "dpf"] if precision == "bf16x3" else ["Pf"])
    for name in names:
        x, y = a.e.debug(name), b.e.debug(name)
        assert np.array_equal(x, y, equal_nan=True), f"{name}: run() and step_begin / step_end differ in {int((x != y).sum())} elements"
        del x, y
    assert np.array_equal(a.e.history(), b.e.history(), equal_nan=True), "history"
    print(f"[stage] c3 {precision}: run(3) and three step pairs bit-identical in {', '.join(names)} and the history")
    a.e.close()
    b.e.close()
    del a, b
    torch.cuda.empty_cache()


# ================================================================================================== 3. past 2^31
def _state_digests(r):
    """SHA-256 of M, m, v (N x V float32, read one at a time through one host buffer) and the step count"""
    torch = _torch()
    buf = np.empty((r.N, r.V), dtype=np.float32)
    out = []
    for name in "Mmv":
        t = r.e.get_state(**{name: buf})
        torch.cuda.synchronize()
        out.append(hashlib.sha256(buf.data).hexdigest())
    del buf
    return out, t


def _big_case(precision):
    N, V, K = 224_000, 10_000, 200
    assert (CROSS[0] * 10048 < 2 ** 31 < CROSS[1] * 10048), "element 2^31 of an N x 10048 operand is in CROSS"
    # host: the stage checks read P (bf16x3: three bf16 planes staged into float32, 10 bytes per element) and one N x V
    # float32 state component at a time; then the bf16x3 host-state handle pins M, m, v (its plan's host bytes) beside
    # the N x V float32 buffer its digests go through.  8 GiB on top of the larger of the two: the process itself
    # (torch, the CUDA context, the inputs) and the window rows.
    stage = (10 if precision == "bf16x3" else 4) * N * V / GIB
    pinned = 0.0
    if precision == "bf16x3":
        pinned = _plan(N, V, K, 0, precision, state_memory="host").host_bytes / GIB + 4 * N * V / GIB
    _need(_planned_gib(N, V, K, 0, precision) + 8, max(stage, pinned) + 8)
    r = _big_work(precision=precision)
    _, wins = _big_windows(r)
    chain = _chain(r)
    # More row windows, at the rows where a forward chain starts: the first two chains' boundaries, the last chain and
    # (fp32) the second split.  The checks on windows are per row and do not depend on where the forward cuts its chains
    # (the forward is checked in full, over every row), so these only spread the rows checked across the mapping.
    for c in sorted({chain, 2 * chain, (r.splits - 1) * chain}):
        if c < N:
            wins.append((c - 64, min(N, c + 64)))
    wins = sorted(set(wins))
    return (N, V, K), r, wins


def test_bf16x3_past_2_31_elements(monkeypatch):
    """224,000 x 10,000 x 200, bf16x3, resident: P's planes 1 and 2 start past element 2^31 and byte 2^32; steps 1..3
    checked on the first rows, the chain boundaries, rows 213,700..213,760 and the last rows (Y in full); and
    state_memory="host" and "auto" (its host rows from row 200,000) reproduce the resident handle's M, m, v and history bit
    for bit after 3 steps."""
    (N, V, K), r, wins = _big_case("bf16x3")
    _assert_path(r, 10048, 256, 110)
    plane = N * r.ld
    assert plane > 2 ** 31 and 2 * plane > 2 ** 32, "P's plane 1 starts past element 2^31 and byte 2^32"
    print(f"[path] big bf16x3: P planes at elements 0, {plane}, {2 * plane} (bytes 0, {2 * plane}, {4 * plane}); "
          f"windows {wins}")
    for step in (1, 2, 3):
        _stage_step(r, step, wins, pre_on_device=False)
    ref = _state_digests(r)
    hist = r.e.history()
    r.e.close()
    del r
    _torch().cuda.empty_cache()
    for sm, forced in (("host", None), ("auto", "200000")):
        if forced:
            monkeypatch.setenv("TGB200_STATE_RESIDENT_ROWS", forced)
        o = _big_work(sm, precision="bf16x3")
        if forced:
            assert o.e.resident_rows() == int(forced) < CROSS[0]
        for _ in range(3):
            o.e.step_begin()
            o.e.step_end(LR)
        _sample()
        assert _state_digests(o) == ref, f"state_memory={sm}: M, m, v differ from the resident handle's"
        assert np.array_equal(o.e.history(), hist, equal_nan=True), f"state_memory={sm}: history"
        o.e.close()
        del o
        _torch().cuda.empty_cache()
        print(f"[stage] bf16x3 state_memory={sm}: M, m, v and history bit-identical to the resident handle")


def test_fp32_past_2_31_elements():
    """224,000 x 10,000 x 200, fp32: Pf, M, m and v pass element 2^31 inside row 213,722 (byte 2^33); steps 1..3 checked
    on the windows of the bf16x3 case plus the second forward split's first rows (Y in full).  fp32 refuses host and
    auto state, in Engine and in tgb200_plan_state."""
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    (N, V, K), r, wins = _big_case("fp32")
    _assert_path(r, 10048, 256, 2)
    print(f"[path] big fp32: windows {wins}")
    for step in (1, 2, 3):
        _stage_step(r, step, wins, pre_on_device=False)
    r.e.close()
    for sm in ("host", "auto"):
        with pytest.raises(ValueError, match="needs precision"):
            Engine(N, V, K, precision="fp32", state_memory=sm)
        with pytest.raises(_lib.TangramB200Error, match="needs precision bf16 or bf16x3"):
            _planned_gib(N, V, K, 0, "fp32", state_memory=sm)
    print("[stage] fp32: state_memory='host' and 'auto' refused")
