"""Each stage of the bf16 iteration checked against float64 at the benchmark's own sizes -- C3 (100k cells x 10k voxels x
2k genes) and C5 (50k x 5k x 2k with the spatial terms) -- and on a mapping of more than 2^31 elements, where every
element offset, TMA coordinate and stream position has to be 64 bits wide.

At these sizes one float64 N x ld tensor is 8 GB, so every N x V check runs on row blocks: debug() buffers are read once
into float32 host arrays, uploaded a block at a time, checked in float64 and freed; the pre-step M, m, v come from
get_state into device tensors; _Blocks (tests/test_clusters_stages_gpu.py) accumulates the rel-Frobenius and bias
statistics across blocks, and the forward's reference P~^T bf16(S / z~) and its magnitude are summed over row blocks.
test_row_blocks_match_full_tensors proves the machinery at 9000 x 300 x 70: one block of every row and blocks of 997
rows give the same max ratio, rel-Frobenius and bias to float64 rounding, and the full-tensor helpers of
tests/test_stages_gpu.py pass on the same steps.

At V = 10,000 the V-scaled bounds of tests/test_stages_gpu.py are about 6e-4 relative, loose enough to let a dropped
float4 through.  The bounds here follow the reductions the kernels run (u = 2^-24, u_b = 2^-8, UM = 2^-21 for MUFU
ex2 / rcp, doubled):

* Row pass at step 1 (k_softmax_rows into bf16 P~): the bucket-table bounds of test_clusters_stages_gpu.py
  (row_pass_layout), P~ with one bf16 rounding on top.
* Carry (k_row_norm, steps >= 2): z~ was summed by the streaming update (k_adam_rows), a lane per 8 columns of every
  256, then a warp tree of 5, each term an ex2.approx of an fma'd argument.  Its depth D is the path's: PLAIN (no
  entropy / L1 / L2 term, C3) sums each 8-column group as a tree of 3 and adds ceil(V / 256) groups in turn,
  D = ceil(V / 256) + 8; the general path (C5, the 9000-row case) adds every element in turn, D = 8 ceil(V / 256) + 5:
      cz_i = D u + UM sum_j P_ij (2 + |M_ij| + |lseA_i|)                              (relative to z)
  lseT = lseA + log z~: cz + 2 u |log z~| + u |lseT|;  P~ / z~: (u_b + UM (3 + |M| + |lseA|) + cz + 2 u) P;
  h = px / z~ - lseT with px = sum_j pt_j M_j a serial fmaf chain of the same depth:
      (cz + cpx + 4 u) (sum_j P_j |M_j| + |lse|),   cpx = (D + 1) u + UM (2 + max_j |M_j| + |lseA|).
  At C3 cz ~ 6e-6 against (V + 8) u = 6e-4.
* Forward: from its own operands P~ and bf16(S / z~), the contraction bounds of _bf16_forward_consts over one 25k-cell
  chunk; Y is checked in full (it sums every row).
* Loss stage: _check_loss_stage_tight (loss_layout), the neighbourhood, cell-type-island and Getis-Ord terms on the
  benchmark's grid graph at C5.
* dq = bf16(S_ext dY_ext^T - c) (TcEpiDpStore): a one-pass wgmma chain over Ke (the forward's constant with chain Ke),
  the fp32 subtraction of the centre c and the bf16 rounding:
      |dq - ref| <= (u_b + 2 u) |ref| + (1 + 2 u_b) ce(Ke) |S| |dY|^T      (pad columns: bf16(-c))
* Row-dot: each lane chains 64 FMAs over a 256-column tile, a quad sum adds 2, k_rowdot_finalize_staged sums r_parts
  partials and scales by 1 / z~: |r' - ref| <= (64 + 2 + r_parts + 2) u sum_j |P~_j dq_j| / z~; rdot = c + r' adds u |rdot|.
* Update: _check_update_bf16's elementwise bounds; P~ after it as in test_stages_gpu; z~ with cz above.
Statistics: 0.5 / 0.25 of an elementwise worst case, 0.75 / 0.1 where a bf16 rounding is the floor, 0.5 / 0.5 where the
MUFU term dominates (ex2.approx may err one-sidedly).

Observed maxima over C3, C5 and the 2^31 windows, steps 1..3, as fractions of each bound (H100 80GB HBM3, 700 W power
limit):

    stage                          elementwise   rel-Fro   bias
    row pass log z / 1 / z / h       0.21          0.15      0.054
    row pass P~                      1.0           0.57      0.0073   (its own bf16 rounding: u_b is the bound)
    carry lseT / h                   0.11          0.085     0.0034
    carry P~ / z~                    0.99          0.56      0.0073
    forward Y genes / density / ct   0.41          0.4       0.4      (run()'s prefetched forward: 0.38)
    dY_ext genes / density           0.98          0.66      0.11
    dq                               0.99          0.65      0.031
    row-dot r' / rdot                0.29          0.32      0.015
    update M / v / m                 1.0           0.42      0.0075   (m: its bf16 rounding)
    update step                      -             0.11      0.0024
    P~ after the update              0.99          0.57      0.0071
    z~                               0.077         0.055     0.015

The file takes 8.8 minutes and at most 27 GiB of host memory (peak RSS).  Each case prints its peak device use, sampled
device-wide at every block upload and state copy ("[memory]"): 1.6 GiB for the 9000-row case, 32.6 GiB at C3, 12.7 GiB at
C5, 33.7 GiB for run() and the shares, 64.6 GiB past 2^31.

Planted errors, each built into a copy of the library and run once at its case:

* A stale dq tile: TcEpiDpStore never stores the 128 x 256 dq tile at column tile 0 of the last full row tile (rows
  99,840..99,967 at C3, in the last chunk).  The C3 stage check fails at step 1: dq at 255 times its bound.
  tests/test_fullsize_gpu.py at C3 still passes with it: bf16 Y against float64 1.0e-3 (bound 3e-3), loss trajectory
  3.3e-5 (1e-3), mapping rel-Frobenius 8.1e-4 (2e-2).
* A forward column tile stored instead of added: chunk 2's contraction stores the tile of voxels 0..127 x genes 0..255
  of Y_ext over the sum of chunks 0 and 1.  The C3 stage check fails at step 1: Y genes at 2,700 times its bound.
* A 32-bit wrap: the streaming update stores P~ at its byte offset modulo 2^32, so the rows from 213,722 on write over
  rows 0..~10,280 of the same allocation.  The 2^31 case fails at step 1: P~ after the update, on the first rows, at
  2.0e5 times its bound.
"""
import os

import numpy as np
import pytest

from tests.test_clusters_stages_gpu import (BIAS, FRO, _Blocks, _cdiv, _check_loss_stage_tight, _row_pass_consts,
                                            _row_pass_h_bound, row_pass_layout)
from tests.test_stages_gpu import (LR, U, UB, UM, Run, _bf16_adam64, _bf16_forward_consts, _bf16_round, _bf16_update_grad,
                                   _check_bf16_update_step, _check_carry, _check_forward, _torch, _x3_contraction_consts)


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


pytestmark = [pytest.mark.gpu, pytest.mark.skipif(_no_gpu(), reason="needs an H100 GPU")]
BLOCK = 2048            # rows per block: float64 temporaries of 2048 x 10048 are 165 MB each
GIB = 2.0 ** 30
_PEAK = {"device": 0}     # device memory in use (device-wide, total - free), sampled at every block upload and state copy


def _sample():
    free, total = _torch().cuda.mem_get_info()
    _PEAK["device"] = max(_PEAK["device"], total - free)


@pytest.fixture(autouse=True)
def _report_memory(request):
    """print each case's sampled peak device use and the process's peak host RSS"""
    import resource
    _PEAK["device"] = 0
    yield
    rss = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024
    print(f"\n[memory] {request.node.name}: peak device use {_PEAK['device'] / GIB:.1f} GiB (sampled), "
          f"peak host RSS of the process so far {rss / GIB:.1f} GiB")


# ------------------------------------------------------------------------------------------------------------- plumbing
def _blocks(wins, block):
    return [(a, min(w1, a + block)) for w0, w1 in wins for a in range(w0, w1, block)]


class _HostRows:
    """Rows `wins` of a debug() buffer of N x cols floats, read once into a float32 host array.  visit(a, b, x) sees
    every row block of the whole buffer before it is cut down to the windows."""

    def __init__(self, e, name, N, cols, wins, visit=None, block=BLOCK):
        x = e.debug(name).reshape(N, cols)
        if visit is not None:
            for a in range(0, N, block):
                visit(a, min(N, a + block), x[a:a + block])
        full = len(wins) == 1 and wins[0] == (0, N)
        self.parts = [(a, b, x[a:b] if full else x[a:b].copy()) for a, b in wins]
        del x

    def get(self, a, b):
        torch = _torch()
        for w0, w1, x in self.parts:
            if w0 <= a and b <= w1:
                out = torch.from_numpy(x[a - w0:b - w0]).to("cuda").double()
                _sample()
                return out
        raise KeyError((a, b))


def _pre_state(r):
    """the handle's M, m, v (N x V float32) on the device and its step count"""
    torch = _torch()
    M, m, v = (torch.empty((r.N, r.V), dtype=torch.float32, device="cuda") for _ in range(3))
    t = r.e.get_state(M=M, m=m, v=v)
    torch.cuda.synchronize()
    _sample()
    return (M, m, v), t


def _same_state(o, ref, what):
    """o's M, m, v equal the device tensors `ref`, bit for bit (one N x V buffer at a time)"""
    torch = _torch()
    x = torch.empty_like(ref[0])
    for name, want in zip("Mmv", ref):
        o.e.get_state(**{k: (x if k == name else None) for k in "Mmv"})
        torch.cuda.synchronize()
        _sample()
        assert torch.equal(x, want), f"{what}: {name} differs in {int((x != want).sum())} elements"


def _finish(res, *accs):
    for acc in accs:
        res[acc.what] = acc.done()


# ------------------------------------------------------------------------------------------------- after step_begin
def _after_begin(r, pre, step, wins, block, res, mode):
    """Reads P~ once: the forward's reference summed over every row, and on the rows of `wins` the row pass (step 1) or
    the carry (steps >= 2).  -> snapshot for _after_end."""
    torch = _torch()
    V, N, ld = r.V, r.N, r.ld
    stats = r.buf("stats", 4)
    izt = r.buf("inv_zt")
    snap = {"lseT": r.buf("lseT"), "c": r.buf("rcenter"), "stats": stats, "izt": izt, "lseA": r.buf("lseA")}
    if step == 1:
        assert bool((izt == 1).all()), "z~ = 1 on a fresh P"
        assert bool((snap["c"] == 0).all()), "no centre before the first backward"
    Yref = torch.zeros((V, r.Ke), dtype=torch.float64, device="cuda")
    Ysc = torch.zeros_like(Yref)

    def fwd(a, b, x):
        P = torch.from_numpy(x[:, :V]).to("cuda").double()
        Ss = _bf16_round(r.S[a:b].float() * izt[a:b].float()[:, None])       # k_scale_rows_bf16
        Yref.addmm_(P.t(), Ss)
        Ysc.addmm_(P.t(), Ss.abs())

    Pt = _HostRows(r.e, "Pb", N, ld, wins, visit=fwd, block=block)
    snap["Pt"], snap["Yref"] = Pt, (Yref, Ysc)
    if step == 1:
        _row_pass_blocks(r, pre, Pt, stats, wins, block, res, f"{mode} row pass")
    else:
        _carry_blocks(r, pre, Pt, snap, wins, block, res, f"{mode} carry")
    return snap


def _row_pass_blocks(r, pre, Pt, stats, wins, block, res, mode):
    """tests/test_clusters_stages_gpu.py::_check_row_pass_tight on row blocks, P~ with its bf16 rounding (p_extra u_b)"""
    torch = _torch()
    V = r.V
    lz = _Blocks(f"{mode} log z", 1.0, FRO, BIAS)
    iz_ = _Blocks(f"{mode} 1 / z", 1.0, FRO, BIAS)
    pp = _Blocks(f"{mode} P", 1.0, 0.75, 0.1)
    hh = _Blocks(f"{mode} h", 1.0, FRO, BIAS) if r.lam.get("lambda_r") else None
    for a, b in _blocks(wins, block):
        M = pre[0][a:b].double()
        st = stats[a:b]
        P, mx, logz, cz, c_logz, cP, dist = _row_pass_consts(r, M)
        assert torch.equal(st[:, 0], mx), f"{mode}: row max, rows {a}..{b}"
        lz.add(st[:, 2], logz, c_logz)
        iz = torch.exp(-logz)
        iz_.add(st[:, 1], iz, (cz + U) * iz)
        x = Pt.get(a, b)
        pp.add(x[:, :V], P, (cP + UB) * P)
        assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of P~, rows {a}..{b}"
        if hh is not None:
            logP = torch.log_softmax(M, dim=1)
            hh.add(st[:, 3], (P * logP).sum(dim=1), _row_pass_h_bound(r, P, logP, cP, dist, c_logz))
        del M, P, x, cP, dist
    _finish(res, *[x for x in (lz, iz_, pp, hh) if x is not None])


def _sum_depth(r):
    """serial adds + tree levels of the streaming update's per-row sums (adam_rows.cuh, a lane per 8 columns of every
    256): the PLAIN path (no entropy / L1 / L2 term) sums each 8-column group as a tree of 3 and adds the groups in turn,
    ceil(V / 256) + 3; the general path adds every element in turn, 8 ceil(V / 256); then a warp tree of 5"""
    n = _cdiv(r.V, 256)
    plain = not (r.lam.get("lambda_r") or r.lam.get("lambda_l1") or r.lam.get("lambda_l2"))
    return (n + 3 if plain else 8 * n) + 5


def _cz(r, P, M, lseA):
    """relative error bound of a z~ the streaming update summed: depth u + UM sum_j P_j (2 + |M_j| + |lseA|)"""
    return _sum_depth(r) * U + UM * (P * (2 + M.abs() + lseA.abs()[:, None])).sum(dim=1)


def _carry_blocks(r, pre, Pt, snap, wins, block, res, mode):
    """lseT, P~ / z~ and h after k_row_norm against float64 softmax / logsumexp of the pre-step M (the docstring's cz)"""
    torch = _torch()
    V = r.V
    lseT, izt, lseA, stats = snap["lseT"], snap["izt"], snap["lseA"], snap["stats"]
    ls = _Blocks(f"{mode} lseT", 1.0, 0.5, 0.5)
    pz = _Blocks(f"{mode} P~ / z~", 1.0, 0.75, 0.1)
    hh = _Blocks(f"{mode} h", 1.0, 0.5, 0.5) if r.lam.get("lambda_r") else None
    for a, b in _blocks(wins, block):
        M = pre[0][a:b].double()
        lse = torch.logsumexp(M, dim=1)
        P = torch.softmax(M, dim=1)
        la = lseA[a:b]
        cz = _cz(r, P, M, la)
        ls.add(lseT[a:b], lse, cz + 2 * U * (lse - la).abs() + U * lse.abs())
        x = Pt.get(a, b)
        z = x[:, :V] * izt[a:b, None]
        pz.add(z, P, (UB + UM * (3 + M.abs() + la.abs()[:, None]) + cz[:, None] + 2 * U) * P)
        assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of P~, rows {a}..{b}"
        if hh is not None:
            h = (P * torch.log_softmax(M, dim=1)).sum(dim=1)
            # px = sum_j pt_j M_j, a serial fmaf chain of the same depth, each pt off by UM (2 + |M_j| + |lseA|)
            cpx = (_sum_depth(r) + 1) * U + UM * (2 + M.abs().max(dim=1).values + la.abs())
            hs = (P * M.abs()).sum(dim=1) + lse.abs()
            hh.add(stats[a:b, 3], h, (cz + cpx + 4 * U) * hs)
        del M, P, x, z
    _finish(res, *[x for x in (ls, pz, hh) if x is not None])


# --------------------------------------------------------------------------------------------------- after step_end
def _dq_consts(Ke):
    """one wgmma pass over a chain of Ke products (the bf16 forward's constant, _bf16_forward_consts, with chain Ke)"""
    return _x3_contraction_consts(Ke)[0] - 2 * 5 * _cdiv(Ke, 16) * U


def _after_end(r, pre, t, snap, step, wins, block, res, mode, M_loss=None):
    """The forward (in full), the loss stage, and on the rows of `wins` dq, the row-dot, the streaming update and the
    P~ / z~ it left."""
    torch = _torch()
    V, N, ld, Ke = r.V, r.N, r.ld, r.Ke
    Y = r.buf("Y", Ke)
    fc = _bf16_forward_consts(r)
    res.update({f"{mode} {k}": x for k, x in _check_forward(r, Y, None, *fc, mode=mode, ref=snap["Yref"]).items()})
    dY = r.buf("dY", Ke)
    stats = snap["stats"]
    # per-row |M|, M^2: the row pass at step 1, the previous streaming update (8 columns per lane) after it
    threads, _, per = row_pass_layout(ld)
    row_depth = per + 2 + int(np.log2(threads)) if step == 1 else 8 * _cdiv(V, 256) + 5
    if M_loss is None:
        M_loss = torch.zeros((1, V), dtype=torch.float64, device="cuda")
    _check_loss_stage_tight(r, Y, dY, r.e.history()[-1], M_loss, stats, row_depth, mode)
    del Y
    dYp = torch.zeros((ld, Ke), dtype=torch.float64, device="cuda")
    dYp[:V] = dY
    del dY
    rowc, rdot, rc_after = r.buf("rowc", 4), r.buf("rdot"), r.buf("rcenter")
    zsum, lseA = r.buf("zsum"), r.buf("lseA")
    assert torch.equal(rowc[:, 0], snap["lseT"]), "rowc carries the row's exact log-sum-exp"
    assert torch.equal(lseA, snap["lseT"]), "after step_end lseA is the offset the new P~ was written with"
    assert torch.equal(rc_after, rdot), "the next centre is this row-dot"
    c, izt = snap["c"], snap["izt"]
    ce = _dq_consts(Ke)
    dqa = _Blocks(f"{mode} dq (Ke {Ke})", 1.0, 0.75, 0.1)
    sa = _Blocks(f"{mode} row-dot r' ({r.rparts} partials)", 1.0, FRO, BIAS)
    ra = _Blocks(f"{mode} rdot = c + r'", 1.0, FRO, BIAS)
    dq = _HostRows(r.e, "dq", N, ld, wins, block=block)
    Pt = snap.pop("Pt")
    for a, b in _blocks(wins, block):
        Sb = _bf16_round(r.S[a:b])
        ref = Sb @ dYp.t() - c[a:b, None]
        sc = Sb.abs() @ dYp.abs().t()
        q = dq.get(a, b)
        dqa.add(q, ref, (UB + 2 * U) * ref.abs() + (1 + 2 * UB) * ce * sc)
        del ref, sc, Sb
        p = Pt.get(a, b)
        pq = p * q
        s_ref = pq.sum(dim=1) * izt[a:b]
        s_b = (64 + 2 + r.rparts + 2) * U * pq.abs().sum(dim=1) * izt[a:b]
        sa.add(rowc[a:b, 1], s_ref, s_b)
        ra.add(rdot[a:b], c[a:b] + s_ref, s_b + U * (c[a:b] + s_ref).abs())
        del p, q, pq
    _finish(res, dqa, sa, ra)
    del Pt, dYp
    post = [_HostRows(r.e, n, N, ld, wins, block=block) for n in ("M", "m", "v")]
    Pn = _HostRows(r.e, "Pb", N, ld, wins, block=block)
    _update_blocks(r, pre, post, Pn, dq, rowc, lseA, zsum, t + 1, wins, block, res, mode)
    del post, Pn, dq
    _torch().cuda.empty_cache()


def _update_blocks(r, pre, post, Pn, dq, rowc, lseA, zsum, t, wins, block, res, mode):
    """tests/test_stages_gpu.py::_check_bf16_update_step / _check_update_bf16 on row blocks (not late, not tiny), with
    the z~ bound cz of the docstring"""
    torch = _torch()
    V = r.V
    accM = _Blocks(f"{mode} update M", 1.0, FRO, BIAS)
    accv = _Blocks(f"{mode} update v", 1.0, 1.0, 1.0)
    accm = _Blocks(f"{mode} update m (bf16)", 1.0, 1.0, 1.0)
    step = _Blocks(f"{mode} update step", 1e30, 8 * UM, 2 * UM)
    pn = _Blocks(f"{mode} P~ after the update", 1.0, 0.75, 0.1)
    zz = _Blocks(f"{mode} z~", 1.0, 0.5, 0.5)
    mb_sum, mb_n, dM2, dMrel = 0.0, 0, 0.0, 0.0
    for a, b in _blocks(wins, block):
        M0, m0, v0 = (x[a:b].double() for x in pre)
        rc = rowc[a:b]
        q = dq.get(a, b)[:, :V]
        P, g, dg = _bf16_update_grad(r, M0, q, rc)
        del q, P
        Mr, mr, vr, dM, dm, dv = _bf16_adam64(M0, m0, v0, g, dg, t)
        del g, dg
        M1, m1, v1 = (x.get(a, b) for x in post)
        for x, name in ((M1, "M"), (m1, "m"), (v1, "v")):
            assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of {name}, rows {a}..{b}"
        accv.add(v1[:, :V], vr, dv)
        accM.add(M1[:, :V], Mr, dM)
        accm.add(m1[:, :V], mr, UB * mr.abs() + dm * (1 + UB))
        live = mr.abs() > 0
        mb_sum += float(((m1[:, :V] - mr)[live] / mr[live].abs() * torch.sign(mr[live])).sum())
        mb_n += int(live.sum())
        stepref = M0 - Mr
        step.add(M0 - M1[:, :V], stepref, stepref.abs() + dM)
        dM2 += float((dM * dM).sum())
        sc = stepref.abs() + dM
        dMrel += float((dM[sc > 0] / sc[sc > 0]).sum())
        del sc
        del m0, v0, mr, vr, dm, dv, m1, v1, stepref, M0, Mr, dM
        Mn = M1[:, :V]
        la = lseA[a:b]
        Pref = torch.exp(Mn - la[:, None])
        x = Pn.get(a, b)
        pn.add(x[:, :V], Pref, (UB + UM * (2 + Mn.abs() + la.abs()[:, None])) * Pref)
        assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of P~ after the update, rows {a}..{b}"
        zs = Pref.sum(dim=1)
        zz.add(zsum[a:b], zs, _cz(r, Pref / zs[:, None], Mn, la) * zs)
        del Mn, M1, Pref, x
    # The step's rel-Fro: 8 UM where g is large against Adam's eps (tests/test_stages_gpu.py); at 10k voxels g = P (dq - r')
    # is ~1e-9, as small as eps, so the step passes on g's own error (MUFU ex2 of |M - lse| ~ 10, the cancellation in
    # dq - r'), one-sidedly where ex2.approx errs one way; the bounds are then half the rel-Fro and a quarter of the mean
    # of the elementwise bound dM, as for every other worst case here (observed at C3: 0.11 and 0.14 of them)
    step.c_fro = max(step.c_fro, 0.5 * (dM2 / step.s2) ** 0.5 if step.s2 else 0.0)
    step.c_bias = max(step.c_bias, 0.25 * dMrel / step.n if step.n else 0.0)
    _finish(res, accM, accv, accm, step, pn, zz)
    bias = mb_sum / mb_n if mb_n else 0.0
    print(f"[stage] {mode} update m (bf16 round to nearest) bias {bias:.3g} (bound {UB / 16:.3g})")
    assert abs(bias) <= UB / 16, f"{mode} update m: rounding bias {bias:.3g}"
    res[f"{mode} update m bias"] = (0.0, 0.0, bias)


def _stage_step(r, step, wins, block=BLOCK, M_loss64=False):
    """one step_begin / step_end pair with every stage checked on the rows of `wins` -> {label: statistics}"""
    pre, t = _pre_state(r)
    assert t == step - 1
    mode = f"{r.name} bf16[{step}]"
    res = {}
    r.e.step_begin()
    snap = _after_begin(r, pre, step, wins, block, res, mode)
    r.e.step_end(LR)
    M_loss = pre[0].double() if M_loss64 else None
    _after_end(r, pre, t, snap, step, wins, block, res, mode, M_loss=M_loss)
    del pre, snap, M_loss
    _torch().cuda.empty_cache()
    return res


# ================================================================================================ 1. the machinery
def test_row_blocks_match_full_tensors():
    """9000 x 300 x 70 with the entropy term, two cell chunks.  The row-block checks over one block of every row and over
    blocks of 997 rows agree to float64 rounding (max ratio, rel-Frobenius, bias).  Where the full-tensor helpers of
    tests/test_stages_gpu.py measure the same quantity against the same scale -- the forward from P~ and bf16(S / z~),
    the update step -- their statistics agree with the row blocks' too; their other checks (V-scaled bounds) pass on the
    same steps."""
    torch = _torch()
    N, V, K = 9000, 300, 70
    r = Run("bf16", N, V, K, seed=N + V, lam={"lambda_r": 1e-3})
    r.name, r.rparts = "rows9000", int(r.e.debug("shape")[3])
    assert r.nchunks == 2
    wins = [(0, N)]
    for step in range(1, 4):
        pre, t = _pre_state(r)
        pre64 = tuple(x.double() for x in pre)
        res = [{}, {}]
        mode = f"rows9000 bf16[{step}]"
        r.e.step_begin()
        snaps = [_after_begin(r, pre, step, wins, blk, res[i], mode) for i, blk in enumerate((N, 997))]
        if step > 1:
            _check_carry(r, pre64[0], f"{mode} carry (full tensor)")
        lseT_now = r.buf("lseT")
        Pt_fwd = r.nv("Pb")[:, :V]
        Ss = _bf16_round(r.S.float() * r.buf("inv_zt").float()[:, None])
        r.e.step_end(LR)
        full = {f"{mode} {k}": x for k, x in
                _check_forward(r, r.buf("Y", r.Ke), Pt_fwd, *_bf16_forward_consts(r), f"{mode} (full tensor)", S=Ss).items()}
        full[f"{mode} update step"] = _check_bf16_update_step(r, pre64, t, lseT_now, f"{mode} (full tensor)")
        for i, blk in enumerate((N, 997)):
            _after_end(r, pre, t, snaps[i], step, wins, blk, res[i], mode, M_loss=pre64[0])
        assert res[0].keys() == res[1].keys() and set(full) <= set(res[0]), (sorted(full), sorted(res[0]))
        for what, want in [(w, res[0][w]) for w in res[0]] + list(full.items()):
            for x, y in zip(res[1][what], want):
                assert abs(x - y) <= 1e-9 * max(abs(x), abs(y)) + 1e-12, f"{what}: row blocks {res[1][what]}, against {want}"
        del pre, pre64, snaps
        torch.cuda.empty_cache()


# ======================================================================================== 2. the benchmark's sizes
class _Work:
    """An Engine on a workload's inputs plus the float64 copies the stage checks read (S_ext on the device)"""

    def __init__(self, name, N, V, K, T, inp, lam, graphs=None, state_memory="device", init=None, precision="bf16"):
        import torch
        from tangram_b200 import _lib
        from tangram_b200.engine import Engine
        self.name, self.precision, self.N, self.V, self.K, self.T, self.lam = name, precision, N, V, K, T, dict(lam)
        self.clusters, self.graphs, self.inp = False, graphs or {}, inp
        self.e = Engine(N, V, K, n_types=T, precision=precision, density_mode=_lib.DENSITY_CELLS, state_memory=state_memory, **lam)
        self.e.set_expression(inp["S"], inp["G"])
        self.e.set_density(inp["d"])
        for which, g in self.graphs.items():
            self.e.set_graph(which, g)
        if T:
            self.e.set_ct_encode(inp["ct_encode"])
        if init is None:
            self.e.init_mapping_normal(7)
        else:
            init(self.e)
        self.Ke, self.ld, self.splits, self.rparts, self.nchunks = (int(x) for x in self.e.debug("shape"))
        self.S = torch.from_numpy(self.e.debug("Sx").reshape(N, self.Ke)).to("cuda").double()
        self.G = torch.as_tensor(np.asarray(inp["G"], dtype=np.float64), device="cuda")
        self.d = torch.as_tensor(np.asarray(inp["d"], dtype=np.float64), device="cuda")

    def buf(self, name, cols=None):
        import torch
        x = self.e.debug(name)
        return torch.from_numpy(x.reshape(-1, cols) if cols else x).to("cuda").double()

    def chunk_rows(self):
        return [_round_up(c * self.N // self.nchunks, 256) for c in range(self.nchunks)] + [self.N]


def _round_up(x, m):
    return -(-x // m) * m


_INPUTS = {}


def _bench_work(name, **kw):
    import bench
    from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph
    from tangram_b200 import _lib
    N, V, K, T, _, _ = bench.WORKLOADS[name]
    if name not in _INPUTS:
        _INPUTS.clear()
        _INPUTS[name] = bench.gen_inputs(name, 0, N)
    lam, graphs = {}, None
    if name == "c5":
        lam = dict(bench.C5_LAMBDAS)
        conn, dist = grid_graph(V)
        graphs = {_lib.GRAPH_VOXEL_WEIGHTS: spatial_weights_from_graph(conn, dist, True, True),
                  _lib.GRAPH_NEIGHBORHOOD_FILTER: spatial_weights_from_graph(conn, dist, False, False),
                  _lib.GRAPH_SPATIAL_WEIGHTS: spatial_weights_from_graph(conn, dist, False, True)}
    return _Work(name, N, V, K, T, _INPUTS[name], lam, graphs, **kw)


def _need(device_gb, host_gb):
    import gc

    import torch
    from tangram_b200.engine import host_memory_available
    gc.collect()                      # handles and device tensors of the cases before this one
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    host = host_memory_available()
    if free < device_gb * GIB or (host is not None and host < host_gb * GIB):
        pytest.skip(f"needs {device_gb} GiB free on the device and {host_gb} GiB of MemAvailable; "
                    f"{free / GIB:.1f} GiB and {(host or 0) / GIB:.1f} GiB are there")
    print(f"[memory] device free {free / GIB:.1f} GiB, MemAvailable {(host or 0) / GIB:.1f} GiB")


def _assert_bench_path(r):
    """C3: 4 chunks, ld 10048, Ke 2048, a last column tile of 16 live voxels.  C5: 4 chunks, ld 5056, Ke 2048, and a
    chunk with an odd number of 128-row tiles (a phantom tile in the last pair of the 2-CTA clusters)."""
    rows = r.chunk_rows()
    tiles = [_cdiv(b - a, 128) for a, b in zip(rows, rows[1:])]
    assert r.nchunks == 4 and r.Ke == 2048 and r.rparts == _cdiv(r.V, 256), (r.nchunks, r.Ke, r.rparts)
    if r.name == "c3":
        assert r.ld == 10048 and r.V - 256 * (_cdiv(r.ld, 256) - 1) == 16, "C3: 40 column tiles, the last with 16 live voxels"
    else:
        assert r.ld == 5056 and any(x % 2 for x in tiles), f"C5: a chunk of odd row tiles, {tiles}"
    print(f"[path] {r.name}: chunks at rows {rows}, row tiles {tiles}, ld {r.ld}, Ke {r.Ke}, {r.rparts} row-dot partials")


@pytest.mark.parametrize("name", ["c3", "c5"])
def test_bf16_stages_at_benchmark_size(name):
    """bench.gen_inputs' workload with the default chunk count and TGB200_UPDATE_SMS: the row pass (step 1), the carry
    (steps 2, 3), the forward, the loss stage, dq and the row-dot, the streaming update and the P~ / z~ it leaves, at
    steps 1, 2 and 3 on every row."""
    assert "TGB200_CHUNKS" not in os.environ and "TGB200_UPDATE_SMS" not in os.environ
    _need(60, 40)
    r = _bench_work(name)
    _assert_bench_path(r)
    for step in (1, 2, 3):
        _stage_step(r, step, [(0, r.N)], M_loss64=name == "c5")
    r.e.close()


def test_c3_run_and_update_share_invariance(monkeypatch):
    """C3: run(3) leaves every buffer and the history bit-identical to three step_begin / step_end pairs, its prefetched
    third forward checked elementwise against float64 from that forward's operands; and with TGB200_UPDATE_SMS at 0, 16
    (the default) and 126 three steps give the same M, m, v and history bit for bit."""
    torch = _torch()
    _need(60, 30)
    a = _bench_work("c3")
    for step in range(3):
        a.e.step_begin()
        if step == 2:                     # the operands of the third forward: its reference, summed over row blocks
            izt = a.buf("inv_zt")
            Yref = torch.zeros((a.V, a.Ke), dtype=torch.float64, device="cuda")
            Ysc = torch.zeros_like(Yref)

            def fwd(r0, r1, x):
                P = torch.from_numpy(x[:, :a.V]).to("cuda").double()
                Ss = _bf16_round(a.S[r0:r1].float() * izt[r0:r1].float()[:, None])
                Yref.addmm_(P.t(), Ss)
                Ysc.addmm_(P.t(), Ss.abs())

            _HostRows(a.e, "Pb", a.N, a.ld, [(0, 0)], visit=fwd)
        a.e.step_end(LR)
    b = _bench_work("c3")
    b.e.run(3)
    for name in ["Y", "M", "m", "v", "Pb", "dq", "inv_zt", "lseA", "zsum", "rcenter", "rdot", "rowc", "stats"]:
        x, y = a.e.debug(name), b.e.debug(name)
        assert np.array_equal(x, y, equal_nan=True), f"{name}: run() and step_begin / step_end differ in {int((x != y).sum())} elements"
        del x, y
    assert np.array_equal(a.e.history(), b.e.history(), equal_nan=True), "history"
    _check_forward(b, b.buf("Y", b.Ke), None, *_bf16_forward_consts(b), "c3 run() prefetched", ref=(Yref, Ysc))
    b.e.close()
    del b, Yref, Ysc
    ref, _ = _pre_state(a)
    hist = a.e.history()
    a.e.close()
    del a
    torch.cuda.empty_cache()
    for share in ("0", "16", "126"):
        monkeypatch.setenv("TGB200_UPDATE_SMS", share)
        c = _bench_work("c3")
        for _ in range(3):
            c.e.step_begin()
            c.e.step_end(LR)
        _same_state(c, ref, f"TGB200_UPDATE_SMS={share}")
        assert np.array_equal(c.e.history(), hist, equal_nan=True), f"TGB200_UPDATE_SMS={share}: history"
        c.e.close()
        del c
        torch.cuda.empty_cache()


# ================================================================================================== 3. past 2^31
BIG = (224_000, 10_000, 200)
BIG_SEED = 42
CROSS = (213_700, 213_760)      # element 2^31 of an ld = 10048 operand is in row 213,722, byte 2^32 of a bf16 one too


def _big_work(state_memory="device", precision="bf16"):
    from oracle.tangram_oracle import synthetic_inputs
    N, V, K = BIG
    if "big" not in _INPUTS:
        _INPUTS.clear()
        _INPUTS["big"] = synthetic_inputs(N, V, K, seed=3)

    def init(e):
        e.init_mapping_legacy(np.random.RandomState(BIG_SEED).get_state())
    return _Work("big", N, V, K, 0, _INPUTS["big"], {}, state_memory=state_memory, init=init, precision=precision)


def _big_windows(r):
    rows = r.chunk_rows()
    wins = [(0, 64)]
    for c in rows[1:-1]:
        wins.append((c - 64, c + 64))
    wins += [CROSS, (r.N - 64, r.N)]
    return rows, wins


def test_mapping_past_2_31_elements(monkeypatch):
    """224,000 x 10,000 x 200, bf16, resident: ld 10048, so 2.25e9 elements, and Pb / dq pass 2^32 bytes inside row
    213,722.  The legacy draw equals numpy's RandomState.normal bit for bit over all of it; every stage of steps 1..3 is
    checked on the first rows, both sides of every chunk boundary, rows 213,700..213,760 and the last rows (Y in full);
    and state_memory="host" and "auto" (its host rows starting below row 213,722) reproduce the resident handle's M, m, v
    and history bit for bit after 3 steps -- their kernels index slot-relative rows, so this checks the resident
    handle's 64-bit offsets independently of any bound."""
    torch = _torch()
    N, V, K = BIG
    assert (CROSS[0] * 10048 < 2 ** 31 < CROSS[1] * 10048) and (CROSS[0] * 10048 * 2 < 2 ** 32 < CROSS[1] * 10048 * 2)
    _need(68, 48)         # estimated: the handle 32 GB, pre-step state 27 GB; host state pins 22 GB
    r = _big_work()
    rows, wins = _big_windows(r)
    assert (r.ld, r.Ke, r.nchunks) == (10048, 256, 4) and rows[1:4] == [56064, 112128, 168192], (r.ld, r.Ke, rows)
    # the legacy draw, streamed from numpy in row blocks of the same generator
    pre, t = _pre_state(r)
    assert t == 0
    rs = np.random.RandomState(BIG_SEED)
    for a in range(0, N, 2000):
        want = rs.normal(0, 1, (min(N, a + 2000) - a, V)).astype(np.float32)
        got = pre[0][a:a + 2000].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"legacy draw differs in rows {a}..{a + 2000}"
    del pre, want, got
    torch.cuda.empty_cache()
    print(f"[stage] legacy draw of {N * V} values: bit-equal to numpy")
    for step in (1, 2, 3):
        _stage_step(r, step, wins)
    ref, _ = _pre_state(r)
    hist = r.e.history()
    r.e.close()
    del r
    torch.cuda.empty_cache()
    for sm, forced in (("host", None), ("auto", "200000")):
        if forced:
            monkeypatch.setenv("TGB200_STATE_RESIDENT_ROWS", forced)
        o = _big_work(sm)
        if forced:
            assert o.e.resident_rows() == int(forced) < CROSS[0]
        for _ in range(3):
            o.e.step_begin()
            o.e.step_end(LR)
        _same_state(o, ref, f"state_memory={sm}")
        assert np.array_equal(o.e.history(), hist, equal_nan=True), f"state_memory={sm}: history"
        o.e.close()
        del o
        torch.cuda.empty_cache()
        print(f"[stage] state_memory={sm}: M, m, v and history bit-identical to the resident handle")
