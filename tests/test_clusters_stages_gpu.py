"""Each stage of the clusters-regime iteration -- tens to a few hundred mapping rows, tens of thousands of voxels -- checked
against float64 from the device's own inputs to that stage, with bounds that follow the reduction each kernel actually
runs rather than the number of voxels.

tests/test_stages_gpu.py bounds a sum over V voxels by V u.  At V = 50,000 that is 3e-3, and a kernel that drops a float4
of a row, a partial of a row-dot or a voxel of a loss sum stays inside it.  The kernels' sums are short serial runs
followed by trees, so their error is a few dozen u.  Here every bound is that structure's (u = 2^-24, fp32 round to
nearest: a serial run of n adds followed by a tree of depth d is within (n + d) u of the sum of the magnitudes):

* Row pass (k_softmax_rows, bucket table of launch_softmax_rows mirrored in row_pass_layout): each of T threads sums
  n = ceil(ld / 4 / T) float4, each float4 as a pair of pairs (2), then a block tree of log2 T levels:
      z relative:  cz = (n + 2 + log2 T + 4) u + u sum_j P_j |M_j - mx|   (expf <= 2 ulp, its rounded argument)
      log z:       cz + 2 u |log z| (logf, 1 ulp);   1 / z relative: cz + u;   P relative: cz + 6 u + u |M - mx|
      h:           sum_j P_j (cP_j |log P_j| + u |M_j - mx| + u |log P_j|) + c_logz + (4 n + log2 T + 1) u sum_j P_j |log P_j|
  Catches z off by (n + 6) u ~ 2e-6 relative; the uncached pass dropping the last float4 of a row (4 / V = 8e-5) is
  40 times that.
* Forward: checked from the device's own P (Pb / Pf), so P's row-pass error is not in it: the contraction bounds of
  test_stages_gpu (_x3_contraction_consts over the one cell chain; FFMA: (2 chain + splits + 4) u) on every column, the
  density pair hi + lo included.  In bf16 mode, at step 1 (z~ = 1), the pair also against the unsplit weights of
  d_source: hi is exact in bf16, lo is rounded once, so the sum carries 16 bits (2 u_b^2 on top of the contraction).
* Row-dot (bf16x3, TcEpiDpStoreF32 + k_rowdot_finalize): each lane chains 64 FMAs over its 256-column tile, a quad sum
  adds 2, the finalize adds the r_parts partials in a row: against sum_j P_j dP_j of the device's P and dP,
      |r - ref| <= (64 + 2 + r_parts + 1) u sum_j |P_j dP_j|      (263 u at C4: one dropped 80-column tile is ~1e-3)
  The fp32 row-dot (SIMT EpiRowDot) is a V-long FFMA chain per element of P dY_ext, so its V-scaled bound is the
  structure's (tests/test_stages_gpu.py::_check_backward_fp32).
* Loss stage (k_loss_reduce, k_col_finalize, k_loss_scalars, k_dy_assemble; loss_layout mirrors the handle's
  loss_rows / nchunk).  A per-gene column sum chains loss_rows rows, then the finalize's two interleaved chains of
  nchunk / 2 partials and one add: D_col = loss_rows + ceil(nchunk / 2) + 1 (337 at C4).  A per-voxel row sum over the
  genes: 4 columns per thread, a warp tree, 4 warps, then one partial per 512 columns: D_row = 12 + ceil(Ke / 512).  A
  cosine from such sums (dot, norm^2, sqrt, one division) is off by at most
      D u sum|a b| / (|a| |b|) + (D / 2 + 3) u |cs|,
  and its mean over n columns adds the loop's serial run and tree, (ceil(n / 1024) + 11) u mean |cs|.  G's norms are
  the device's own (debug "ngc", "ngr", "nwg", "nag": set-up constants, one of them a V-long serial chain).  The graph
  terms add their nnz-long SpMM chains twice (Z = W Y and W G).  KL: (ceil(V / 1024) + 14) u sum_j (|d log d| +
  |d log dhat| + d).  Entropy: the device's per-row h summed by k_row_scalar_reduce, (ceil(N / 1024) + 11) u sum |h_i|
  (each h_i is checked by the row pass or the bf16 carry).  L1 / L2: the row pass's run (or, in bf16 mode after step 1,
  the streaming update's 8 ceil(V / 256) + 5) plus that reduce.  Cell-type islands: (nnz + 2) u per R that can reach the
  hinge (R > -that), 256-thread block trees, then the scalar loop.  The total: the terms' bounds weighted by their lambdas plus 12 u sum |lambda term|.
  Dropping voxel 0 of the vg loop moves vg by |cs_0| / V = 250 u |cs_0| at V = 66,000, against ~100 u mean |cs|.
  dY_ext: a_k = 1 / (K |Y_k| |G_k|) is off by (D / 2 + 4) u, b_k = cs_k / (K |Y_k|^2) by (2.5 D + 8) u; the bound is
  (2.5 D + 8) u times the magnitude of each part,
  |a_k G_jk| + |b_k Y_jk| (+ the vg, neighbourhood and Getis-Ord parts), elementwise; the density columns
  -d_j / dhat_j within 4 u.  A cell-type gradient whose island indicator R sits within rounding of 0 (so that fp32
  and float64 may disagree on it) is left out and counted.

Statistics: where an elementwise bound above is a worst case, rel-Frobenius and signed mean of err / bound are held to
0.5 and 0.25 of it (0.75 / 0.1 where a bf16 rounding of dY_ext is the floor).

Steps 1 and 3 of every case, and on the C4 and tutorial shapes steps 998 and 1,000 after run(): late bias corrections
(bc2 = 0.63 instead of 0.004) and long-history m, v through the update checks, and in bf16x3 through the bit-exact
comparison with torch.optim.Adam.

Observed maxima over all cases and steps, as fractions of each bound (H100 80GB HBM3, 700 W power limit):

    stage                                elementwise   rel-Fro   bias
    row pass log z, fp32 / bf16x3 / bf16     0.22          0.29      0.13
    row pass 1 / z                           0.082         0.09      0.03
    row pass P, fp32 / bf16x3                0.26          0.1       0.011
    row pass P~, bf16                        0.99          0.57      0.016    (its own bf16 rounding: u_b is the bound)
    row pass h                               0.023         0.017     0.0052
    forward Y_ext genes / ct                 0.17          0.083     0.11
    forward density hi + lo                  0.16          0.16      0.17
    forward density vs unsplit d_source      0.12          0.046     0.029    (bf16, step 1)
    backward dP, bf16x3                      0.027         0.46      0.2      (fixed 8 u / 4 u bounds)
    row-dot, bf16x3                          0.047         0.034     0.023
    row-dot, fp32                            0.0015        0.047     0.063    (V-long FFMA chains: worst case V u)
    history columns 0, 1, 3                  0.0086        -         -
    history columns 2, 7, 9 (cosines)        0.0098        -         -
    history columns 4, 5, 6 (row terms)      0.094         -         -
    dY_ext genes, fp32 / bf16x3              0.033         0.0075    0.0003
    dY_ext genes, bf16                       0.99          0.56      0.0075   (its bf16 rounding)
    dY_ext density                           1.0           0.61      0.7      (bf16; fp32 / bf16x3: 0.25, 0.23, 0.005)
    dY_ext ct                                0.21          0.28      0.0004
    update step, fp32 / bf16x3 / bf16        -             0.41      0.14     (steps 1 .. 1,000; bf16x3 bit-exact torch Adam)

The loss's cosine and total columns sit at 1e-3 .. 1e-2 of their bounds: those are worst cases over D = 337 (C4) serial
adds whose rounding errors in practice cancel like a random walk.  The cell-type islands column (4.5e-7 of its bound,
before its bound counted only the R that can reach the hinge) has almost every R well below 0 (a voxel's filter sums six
neighbours), so its sum has few terms.  The bf16 carry (lseT, P~ / z~, h, z~) keeps the V-scaled bounds of
tests/test_stages_gpu.py.

Planted errors, each run once at its case (one step): the uncached row pass skipping the last float4 of each row's data
fails log z at 165 times its bound; k_rowdot_finalize summing nparts - 1 partials fails the row-dot at 171 times; the vg
loop of k_loss_scalars starting at voxel 1 fails history column 2 at 2.7 times.  The V-scaled elementwise bounds of
tests/test_stages_gpu.py hold for each of them (log z 0.15, row-dot 0.33 of the bound); what catches them there is a
fixed statistical bound (16 u rel-Fro of 1 / z, 4 u row-dot bias) or, for the vg loop, the zero coefficient it leaves
in dY_ext's voxel 0.
"""
import numpy as np
import pytest

from tests.test_stages_gpu import (ALL_TERMS, B1, B2, EPS, LR, U, UB, X3_BWD_BIAS, X3_BWD_FRO, Run, _bf16_forward_consts,
                                   _bf16_round, _check, _check_bf16_update_step, _check_carry, _check_update, _grad_terms,
                                   _loss_of_Y, _state, _torch, _x3_contraction_consts)



def _no_gpu():
    import torch
    return not torch.cuda.is_available()


pytestmark = [pytest.mark.gpu, pytest.mark.skipif(_no_gpu(), reason="needs an H100 GPU")]
FRO, BIAS = 0.5, 0.25
ROW_BUCKETS = ((256, 1), (256, 2), (256, 4), (512, 3), (512, 4), (512, 5), (1024, 3), (1024, 4), (1024, 6))
BLOCK = 4096            # voxel rows per block of the V x Ke checks: float64 temporaries stay near 4096 x Ke x 8 bytes


def _cdiv(a, b):
    return -(-a // b)


def row_pass_layout(ld):
    """launch_softmax_rows for rows of `ld` floats -> (threads, float4 slots cached per thread or 0 when the row is
    re-read, float4 summed per thread)"""
    nvec = ld // 4
    for threads, items in ROW_BUCKETS:
        if nvec <= threads * items:
            return threads, items, _cdiv(nvec, threads)
    return 1024, 0, _cdiv(nvec, 1024)


def loss_layout(V, Ke):
    """the handle's voxel rows per loss CTA, row chunks, and 512-column chunks of the per-voxel sums"""
    rows = 16
    while _cdiv(V, rows) > 512 and rows < 128:
        rows += 16
    return rows, _cdiv(V, rows), _cdiv(Ke, 512)


def _tight(what, got, ref, bound, fro=FRO, bias=BIAS):
    return _check(what, got, ref, bound, 1.0, fro, bias)


class _Blocks:
    """_check's statistics accumulated over row blocks of one array"""

    def __init__(self, what, c_elem, c_fro, c_bias):
        self.what, self.c_elem, self.c_fro, self.c_bias = what, c_elem, c_fro, c_bias
        self.ratio, self.e2, self.s2, self.bsum, self.n = 0.0, 0.0, 0.0, 0.0, 0

    def add(self, got, ref, scale, floor=0.0):
        torch = _torch()
        err = got - ref
        bound = self.c_elem * scale + floor
        bad0 = (bound == 0) & (err != 0)
        assert not bool(bad0.any()), f"{self.what}: nonzero where the bound is zero, first at {torch.nonzero(bad0)[0].tolist()}"
        ratio = err.abs() / torch.where(bound > 0, bound, torch.ones_like(bound))
        worst = float(ratio.max()) if err.numel() else 0.0
        assert worst <= 1.0, f"{self.what}: max err / bound {worst:.3g}, first at {torch.nonzero(ratio > 1)[0].tolist()}"
        self.ratio = max(self.ratio, worst)
        self.e2 += float((err * err).sum())
        self.s2 += float((scale * scale).sum())
        live = scale > 0
        self.bsum += float((torch.sign(ref[live]) * err[live] / scale[live]).sum())
        self.n += int(live.sum())

    def done(self):
        """assert the accumulated statistics; -> (max err / bound, rel-Fro, bias)"""
        fro = (self.e2 / self.s2) ** 0.5 if self.s2 > 0 else 0.0
        bias = self.bsum / self.n if self.n else 0.0
        print(f"[stage] {self.what}: max err/bound {self.ratio:.3g}, rel-Fro {fro:.3g} (bound {self.c_fro:.3g}), "
              f"bias {bias:.3g} (bound {self.c_bias:.3g})")
        assert fro <= self.c_fro, f"{self.what}: rel-Frobenius {fro:.3g} > {self.c_fro:.3g}"
        assert abs(bias) <= self.c_bias, f"{self.what}: bias {bias:.3g} beyond {self.c_bias:.3g}"
        return self.ratio, fro, bias


def _free():
    _torch().cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------- row pass
def _row_pass_consts(r, M):
    """float64 softmax of M and the row pass's bounds: (P, log z, cz, c_logz, cP, |M - mx|)"""
    torch = _torch()
    threads, _, per = row_pass_layout(r.ld)
    Mv = M[:, :r.V]
    mx = Mv.max(dim=1).values
    dist = (Mv - mx[:, None]).abs()
    logz = torch.logsumexp(Mv, dim=1) - mx
    P = torch.softmax(Mv, dim=1)
    cz = (per + 2 + int(np.log2(threads)) + 4) * U + U * (P * dist).sum(dim=1)
    c_logz = cz + 2 * U * logz.abs()
    cP = cz[:, None] + 6 * U + U * dist
    return P, mx, logz, cz, c_logz, cP, dist


def _check_row_pass_tight(r, M, P_dev, stats, mode, p_extra=0.0):
    """log z, 1 / z, P (elementwise, pad columns zero) and h against float64, bounded by the row pass's own sums.
    p_extra: one more relative rounding of P (bf16 mode's P~)."""
    torch = _torch()
    V = r.V
    threads, _, per = row_pass_layout(r.ld)
    P, mx, logz, cz, c_logz, cP, dist = _row_pass_consts(r, M)
    assert torch.equal(stats[:, 0], mx), "row max"
    _tight(f"{mode} log z", stats[:, 2], logz, c_logz)
    iz = torch.exp(-logz)
    _tight(f"{mode} 1 / z", stats[:, 1], iz, (cz + U) * iz)
    _tight(f"{mode} P", P_dev[:, :V], P, (cP + p_extra) * P, fro=0.75 if p_extra else FRO, bias=0.1 if p_extra else BIAS)
    assert torch.count_nonzero(P_dev[:, V:]) == 0, "pad columns of P"
    if r.lam.get("lambda_r"):
        logP = torch.log_softmax(M[:, :V], dim=1)
        _tight(f"{mode} h", stats[:, 3], (P * logP).sum(dim=1), _row_pass_h_bound(r, P, logP, cP, dist, c_logz))
    return P


def _row_pass_h_bound(r, P, logP, cP, dist, c_logz):
    """the row pass's h = sum_j P_j log P_j: each term's P and log P error, the row's serial run and block tree"""
    threads, _, per = row_pass_layout(r.ld)
    aP = logP.abs()
    return ((P * (cP * aP + U * dist + U * aP)).sum(dim=1) + c_logz
            + (4 * per + int(np.log2(threads)) + 1) * U * (P * aP).sum(dim=1))


# ----------------------------------------------------------------------------------------------------------------- forward
def _check_forward_blocks(r, Y_dev, P, consts, mode, S=None, exact_pair=None):
    """Y_ext = P^T S_ext (P: the operand the contraction read, N x V) in blocks of voxel rows: gene columns, the density
    pair's hi + lo sum, cell-type columns, zero past them.  exact_pair: (c_elem, c_fro, c_bias) of the density pair against
    the unsplit fp32 weights r.S[:, K] + r.S[:, K + 1] instead of the operand's own pair."""
    torch = _torch()
    K, T, V = r.K, r.T, r.V
    S = r.S if S is None else S
    ce, cf, cb = consts
    genes = _Blocks(f"{mode} Y genes", ce, cf, cb)
    dens = _Blocks(f"{mode} Y density (hi + lo)", ce, cf, cb)
    ct = _Blocks(f"{mode} Y ct", ce, cf, cb) if T else None
    exact = _Blocks(f"{mode} Y density vs unsplit d_source", *exact_pair) if exact_pair else None
    w = (r.S[:, K] + r.S[:, K + 1])[:, None]
    for a in range(0, V, BLOCK):
        sl = slice(a, min(V, a + BLOCK))
        Pb = P[:, sl]
        ref = Pb.t() @ S
        scale = Pb.t() @ S.abs()
        y = Y_dev[sl]
        genes.add(y[:, :K], ref[:, :K], scale[:, :K])
        dens.add(y[:, K] + y[:, K + 1], ref[:, K] + ref[:, K + 1], scale[:, K] + scale[:, K + 1])
        if ct is not None:
            ct.add(y[:, K + 2:K + 2 + T], ref[:, K + 2:K + 2 + T], scale[:, K + 2:K + 2 + T])
        if exact is not None:
            exact.add(y[:, K] + y[:, K + 1], (Pb.t() @ w)[:, 0], (Pb.t() @ w.abs())[:, 0])
        assert torch.count_nonzero(y[:, K + 2 + T:]) == 0, "Y_ext past the last used column"
        del ref, scale
    for acc in (genes, dens, ct, exact):
        if acc is not None:
            acc.done()
    _free()


def _fp32_forward_consts_own(r):
    """FFMA forward from the device's own P: one chain per split, the splits summed in fp32"""
    chain = _cdiv(r.N, r.splits)
    return (2 * chain + r.splits + 4) * U, 4 * np.sqrt(chain) * U + (r.splits + 4) * U, 16 * U


# -------------------------------------------------------------------------------------------------------------- loss stage
def _cos_parts(a, b, nb):
    """per column: the cosine <a, b> / (|a| nb) and sum |a b| / (|a| nb)"""
    torch = _torch()
    na = torch.clamp(torch.linalg.vector_norm(a, dim=0), min=1e-8)
    ab = a * b
    cs = ab.sum(dim=0) / (na * nb)
    w = ab.abs_().sum(dim=0) / (na * nb)
    return cs, w, na


def _cos_mean_bound(cs, w, depth, n):
    return float((depth * U * w + (depth / 2 + 3) * U * cs.abs()).mean() + (_cdiv(n, 1024) + 11) * U * cs.abs().mean())


def _sparse(r, which):
    torch = _torch()
    m = r.graphs[which].tocsr()
    return torch.sparse_csr_tensor(torch.as_tensor(m.indptr, dtype=torch.int64), torch.as_tensor(m.indices, dtype=torch.int64),
                                   torch.as_tensor(m.data, dtype=torch.float64), size=m.shape).cuda()


def _nnz_max(r, which):
    return int(np.diff(r.graphs[which].tocsr().indptr).max())


def _check_loss_stage_tight(r, Y_dev, dY_dev, hist, M, stats, row_depth, mode):
    """History row (every column that is on) and dY_ext against float64 autograd of the loss of the device's Y_ext, with
    the device's norms of G; row_depth: the serial run + tree of the per-row |M|, M^2 sums the tail reduced."""
    from tangram_b200 import _lib
    torch = _torch()
    V, K, Ke, N, T, lam = r.V, r.K, r.Ke, r.N, r.T, r.lam
    rows, nchunk, nred = loss_layout(V, Ke)
    d_col = rows + _cdiv(nchunk, 2) + 1
    d_row = 12 + nred
    norms = {"ngc": r.buf("ngc"), "ngr": r.buf("ngr")}
    W = A = F = None
    if lam.get("lambda_neighborhood_g1"):
        norms["nwg"] = r.buf("nwg")
        W = _sparse(r, _lib.GRAPH_VOXEL_WEIGHTS)
    if lam.get("lambda_getis_ord"):
        norms["nag"] = r.buf("nag")
        A = _sparse(r, _lib.GRAPH_SPATIAL_WEIGHTS)
    if lam.get("lambda_ct_islands"):
        F = _sparse(r, _lib.GRAPH_NEIGHBORHOOD_FILTER)
    Yx = Y_dev.clone().requires_grad_(True)
    total, terms = _loss_of_Y(r, Yx, M, sparse=True, norms=norms)
    (dref,) = torch.autograd.grad(total, Yx)
    terms = {c: float(v) for c, v in terms.items()}
    del Yx, total
    _free()

    bound, part = {}, {}          # history bounds; dY parts: (coefficient pair, depth)
    Y, G = Y_dev[:, :K], r.G
    with torch.no_grad():
        cs, w, ny = _cos_parts(Y, G, norms["ngc"])
        bound[1] = _cos_mean_bound(cs, w, d_col, K)
        part["gv"] = (1.0 / (K * ny * norms["ngc"]), cs / (K * ny * ny), d_col)
        if lam.get("lambda_g2"):
            cs, w, ny = _cos_parts(Y.t(), G.t(), norms["ngr"])
            bound[2] = _cos_mean_bound(cs, w, d_row, V)
            g2 = lam["lambda_g2"]
            part["vg"] = (g2 / (V * ny * norms["ngr"]), g2 * cs / (V * ny * ny), d_row)
        dhat = Y_dev[:, K] + Y_dev[:, K + 1]
        if not r.clusters:
            dhat = dhat / N
        d = r.d
        xl = torch.special.xlogy(d, d)
        bound[3] = (_cdiv(V, 1024) + 14) * U * float((xl.abs() + (d * torch.log(dhat)).abs() + d).sum())
        if lam.get("lambda_r"):
            hdev = stats[:, 3]
            bound[4] = (_cdiv(N, 1024) + 11) * U * float(hdev.abs().sum())
            terms[4] = -float(hdev.sum())          # checked per row by the row pass / the bf16 carry
        tail = row_depth + _cdiv(N, 1024) + 10 + 3
        if lam.get("lambda_l1"):
            bound[5] = tail * U * terms[5]
        if lam.get("lambda_l2"):
            bound[6] = tail * U * terms[6]
        for col, op, nkey, lk in ((7, W, "nwg", "lambda_neighborhood_g1"), (9, A, "nag", "lambda_getis_ord")):
            if op is None:
                continue
            nnz = _nnz_max(r, _lib.GRAPH_VOXEL_WEIGHTS if col == 7 else _lib.GRAPH_SPATIAL_WEIGHTS)
            depth = d_col + 2 * (nnz + 1)
            Z, OG = op @ Y, op @ G
            cs, w, nz = _cos_parts(Z, OG, norms[nkey])
            sgn = torch.ones_like(cs) if col == 7 else torch.sign(Y.sum(dim=0)) * torch.sign(G.sum(dim=0))
            bound[col] = _cos_mean_bound(cs, w, depth, K)
            lk_ = lam[lk]
            part["nb" if col == 7 else "go"] = (op, OG, Z, sgn * lk_ / (K * nz * norms[nkey]), sgn * lk_ * cs / (K * nz * nz),
                                                depth + nnz)
            del cs, w
        amb = None
        if F is not None:
            C = Y_dev[:, K + 2:K + 2 + T]
            FC = F @ C
            R = C - FC
            nnz = _nnz_max(r, _lib.GRAPH_NEIGHBORHOOD_FILTER)
            rerr = (nnz + 2) * U * (C.abs() + F @ C.abs())
            nblk = _cdiv(V * T, 256)
            # an R below -rerr has a hinge of exactly 0 in both
            bound[8] = float(rerr[R > -rerr].sum() + (8 + _cdiv(nblk, 1024) + 12) * U * R.clamp(min=0).sum()) / (V * T)
            # an indicator 1[R > 0] within rounding of its threshold: fp32 and float64 may disagree, and every dY_ext
            # element that reads it (its own and its filter neighbours') is left out
            flip = ((R.abs() <= rerr) & (rerr > 0)).double()
            amb = (flip + F.to_sparse_coo().t() @ flip) > 0
        lams = {0: None, 1: 1.0, 2: lam.get("lambda_g2", 0.0), 3: 1.0, 4: lam.get("lambda_r", 0.0),
                5: lam.get("lambda_l1", 0.0), 6: lam.get("lambda_l2", 0.0), 7: lam.get("lambda_neighborhood_g1", 0.0),
                8: lam.get("lambda_ct_islands", 0.0), 9: lam.get("lambda_getis_ord", 0.0)}
        sign = {1: -1, 2: -1, 7: -1, 9: -1}
        terms[0] = sum(sign.get(c, 1) * lams[c] * terms[c] for c in terms if c)
        bound[0] = sum(abs(lams[c]) * bound[c] for c in bound if c) + 12 * U * sum(abs(lams[c] * terms[c]) for c in terms if c)
        for col in sorted(terms):
            got = float(hist[col])
            err = abs(got - terms[col])
            rel = err / bound[col] if bound[col] else 0.0        # a zero bound (no island indicator can flip) wants err 0
            print(f"[stage] {mode} history column {col}: err {err:.3g}, err/bound {rel:.3g} (bound {bound[col]:.3g})")
            assert err <= bound[col], f"{mode} history column {col}: {got} vs {terms[col]} (bound {bound[col]:.3g})"

        # dY_ext, gene columns: each part's coefficients off by (2.5 D + 8) u relative, times the part's magnitude
        bf16 = r.precision == "bf16"
        fro, bias = (0.75, 0.1) if bf16 else (FRO, BIAS)
        gacc = _Blocks(f"{mode} dY_ext genes", 1.0, fro, bias)
        mag = None
        for key in ("nb", "go"):
            if key in part:
                op, OG, Z, ca, cb, depth = part[key]
                inner = (ca.abs() * OG.abs() + cb.abs() * Z.abs()) * ((2.5 * depth + 8) * U)
                spread = op.to_sparse_coo().t() @ inner
                mag = spread if mag is None else mag + spread
                del inner
        part.pop("nb", None)
        part.pop("go", None)
        for a in range(0, V, BLOCK):
            sl = slice(a, min(V, a + BLOCK))
            y, g = Y[sl], G[sl]
            ca, cb, depth = part["gv"]
            m = (ca.abs() * g.abs() + cb.abs() * y.abs()) * ((2.5 * depth + 8) * U)
            if mag is not None:
                m += mag[sl]
            if "vg" in part:
                ca, cb, depth = part["vg"]
                m += (ca[sl].abs()[:, None] * g.abs() + cb[sl].abs()[:, None] * y.abs()) * ((2.5 * depth + 8) * U)
            dr = dref[sl, :K]
            gacc.add(dY_dev[sl, :K], dr, m * (1 + UB) + UB * dr.abs() if bf16 else m)
            del m
        gacc.done()
        del mag
        # density columns: -lambda_d d_j / dhat_j, one add, one division, one product
        dr = dref[:, K:K + 2]
        _tight(f"{mode} dY_ext density", dY_dev[:, K:K + 2], dr, (4 * U + (UB if bf16 else 0.0)) * dr.abs(), fro=fro, bias=bias)
        if T:
            dr, dd = dref[:, K + 2:K + 2 + T], dY_dev[:, K + 2:K + 2 + T]
            if amb is not None:
                n_amb = int(amb.sum())
                print(f"[stage] {mode} dY_ext ct: {n_amb} of {amb.numel()} elements next to an indicator at its threshold")
                dd = torch.where(amb, dr, dd)
            # hinge indicators summed over <= nnz + 1 neighbours, one product, one division
            c = (8 + _nnz_max(r, _lib.GRAPH_NEIGHBORHOOD_FILTER)) * U if F is not None else 0.0
            _tight(f"{mode} dY_ext ct", dd, dr, c * (dr.abs() + lams[8] / (V * T)) + (UB * dr.abs() if bf16 else 0.0),
                   fro=fro, bias=bias)
        assert torch.count_nonzero(dY_dev[:, K + 2 + T:]) == 0, "dY_ext past the last used column"
    del dref
    _free()


# -------------------------------------------------------------------------------------------------------------- backward
def _check_backward_fp32_rows(r, pre, t, stats, Pf, dY, mode, late):
    """fp32: the row-dot and the fused update (tests/test_stages_gpu.py::_check_backward_fp32).  Each row-dot is a V-long
    FFMA chain of P dY_ext, so its error is sqrt(Ke + V) u-class per row, and its signed mean over only N rows is held to
    4 u + 4 sqrt((Ke + V) / N) u."""
    V = r.V
    dPref = r.S @ dY.t()
    scale = r.S.abs() @ dY.abs().t()
    rdot = r.buf("rdot")
    rref = (Pf[:, :V] * dPref).sum(dim=1)
    rscale = (Pf[:, :V] * scale).sum(dim=1)
    n = r.Ke + V
    _check(f"{mode} row-dot", rdot, rref, rscale, (2 * n + 8) * U, 4 * np.sqrt(n) * U, 4 * U + 4 * np.sqrt(n / r.N) * U)
    g = _grad_terms(r, pre[0][:, :V], Pf[:, :V], dPref - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
    dg = Pf[:, :V] * (2 * r.Ke + 8) * U * scale + 8 * U * (g.abs() + Pf[:, :V] * (dPref.abs() + rdot.abs()[:, None] + 1.0))
    _check_update(r, pre, _state(r), g, dg, t + 1, mode, late=late)


def _check_backward_x3_tight(r, pre, t, stats, P3, dY, mode, late):
    """bf16x3: dP = S_ext dY_ext^T (one chain over Ke), the row-dot against sum P dP of the device's own P and dP, the
    update's bounds from the pre-step state, and the update bit for bit against torch.optim.Adam."""
    torch = _torch()
    V = r.V
    dpf = r.nv("dpf")
    dPref = r.S @ dY.t()
    scale = r.S.abs() @ dY.abs().t()
    ce = _x3_contraction_consts(r.Ke)[0]
    _check(f"{mode} dP (Ke {r.Ke})", dpf[:, :V], dPref, scale, ce, X3_BWD_FRO, X3_BWD_BIAS)
    assert torch.count_nonzero(dpf[:, V:]) == 0, "pad columns of dP"
    del dPref, scale
    rdot = r.buf("rdot")
    pd = P3[:, :V] * dpf[:, :V]
    _tight(f"{mode} row-dot ({r.rparts} partials)", rdot, pd.sum(dim=1), (64 + 2 + r.rparts + 1) * U * pd.abs().sum(dim=1))
    del pd
    g = _grad_terms(r, pre[0][:, :V], P3[:, :V], dpf[:, :V] - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
    if r.lam:
        dg = 8 * U * (g.abs() + P3[:, :V] * (dpf[:, :V].abs() + rdot.abs()[:, None] + 1.0))
    else:
        dg = 4 * U * (g.abs() + P3[:, :V] * (dpf[:, :V].abs() + rdot.abs()[:, None]))
    post = _state(r)
    _check_update(r, pre, post, g, dg, t + 1, mode, late=late)
    del g, dg
    if r.lam:
        return
    # torch's Adam from the device's fp32 values (tests/test_stages_gpu.py::test_bf16x3_update_is_torch_adam)
    M0, m0, v0 = (x[:, :V].float().contiguous() for x in pre)
    gf = (dpf[:, :V].float() - rdot.float()[:, None]) * P3[:, :V].float()
    p = torch.nn.Parameter(M0.clone())
    opt = torch.optim.Adam([p], lr=LR, betas=(B1, B2), eps=EPS, foreach=False, fused=False)
    p.grad = gf
    opt.state[p] = {"step": torch.tensor(float(t)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    opt.step()
    for name, got, want in (("v", post[2], opt.state[p]["exp_avg_sq"]), ("m", post[1], opt.state[p]["exp_avg"]),
                            ("M", post[0], p.detach())):
        diff = got[:, :V].float() != want
        assert not bool(diff.any()), f"{mode}: {name} differs from torch's Adam in {int(diff.sum())} of {diff.numel()} elements"


# ================================================================================================================== cases
# id: (N, V, K, T, lam, precisions, late steps, expected path)
CASES = {
    "c4": (256, 50000, 5000, 0, {}, ("bf16x3", "bf16"), True),
    "c4-fp32": (256, 50000, 300, 0, {}, ("fp32",), False),
    "sub-tile": (48, 30000, 300, 0, {}, ("fp32", "bf16x3", "bf16"), False),
    "66k-all-terms": (129, 66000, 70, 8, ALL_TERMS, ("fp32", "bf16x3", "bf16"), False),
    "tutorial": (18, 9852, 248, 0, {}, ("bf16x3", "bf16"), True),
}
PARAMS = [pytest.param(cid, prec, id=f"{cid}-{prec}") for cid, c in CASES.items() for prec in c[5]]


def _assert_path(cid, r):
    """the internal path each case is there for, from debug("shape") and the mirrored launch tables"""
    threads, items, per = row_pass_layout(r.ld)
    tc = r.precision != "fp32"
    assert r.nchunks == 1, "clusters-scale N: one cell chunk"
    if tc:
        assert r.rparts == _cdiv(r.V, 256), "one row-dot partial per 256-voxel tile"
    else:
        assert r.rparts == _cdiv(r.Ke, 128), "one row-dot partial per 128-column SIMT tile"
    if cid == "c4":
        assert (r.Ke, r.rparts, r.splits) == (5056, 196, 1), "C4: Ke 5056 uncut backward chain, 196 partials, one split"
        assert items == 0 and per == 13, "C4: the uncached row pass, 13 float4 per thread"
    elif cid == "c4-fp32":
        assert items == 0 and r.rparts == 3
    elif cid == "sub-tile":
        assert r.N < 128 and items == 0 and r.splits == 1, "less than one 128-row backward tile; the uncached row pass"
    elif cid == "66k-all-terms":
        assert r.V > 65535 and r.N == 129 and items == 0, "gridDim.x past 65,535; a second row tile of one row"
        if tc:
            assert r.rparts == 258
    elif cid == "tutorial":
        assert (threads, items) == (512, 5), "the cached 512 x 5 bucket"


def _run(cid, precision):
    N, V, K, T, lam = CASES[cid][:5]
    r = Run(precision, N, V, K, seed=N + V + K, T=T, clusters=True, lam=lam)
    r.rparts = int(r.e.debug("shape")[3])
    _assert_path(cid, r)
    return r


def _steps(cid):
    late = CASES[cid][6]
    return [1, 2, 3] + ([998, 999, 1000] if late else [])


def _catch_up(r, step):
    """before `step`: run() up to step - 1 when the handle is behind"""
    t = r.e.get_state()
    if t < step - 1:
        r.e.run(step - 1 - t)


@pytest.mark.parametrize("cid,precision", [p for p in PARAMS if p.values[1] != "bf16"])
def test_clusters_stages(cid, precision):
    """fp32 / bf16x3: row pass, forward, loss stage, backward (dP and row-dot) and the update, each from the device's
    own inputs, at steps 1 and 3 (and 998, 1,000 on the C4 and tutorial shapes)."""
    r = _run(cid, precision)
    threads, _, per = row_pass_layout(r.ld)
    row_depth = per + 2 + int(np.log2(threads))
    for step in _steps(cid):
        _catch_up(r, step)
        pre = _state(r)
        t = r.e.get_state()
        assert t == step - 1
        r.e.step_begin()
        r.e.step_end(LR)
        if step in (2, 999):
            continue
        mode = f"{cid} {precision}[{step}]"
        stats = r.buf("stats", 4)
        P = r.nv("Pb" if precision == "bf16x3" else "Pf")
        _check_row_pass_tight(r, pre[0], P, stats, f"{mode} row pass")
        Yd = r.buf("Y", r.Ke)
        consts = _x3_contraction_consts(_cdiv(r.N, r.splits), r.splits) if precision == "bf16x3" else _fp32_forward_consts_own(r)
        _check_forward_blocks(r, Yd, P[:, :r.V], consts, mode)
        dY = r.buf("dY", r.Ke)
        _check_loss_stage_tight(r, Yd, dY, r.e.history()[-1], pre[0], stats, row_depth, mode)
        del Yd
        _free()
        if precision == "bf16x3":
            _check_backward_x3_tight(r, pre, t, stats, P, dY, mode, late=step > 3)
        else:
            _check_backward_fp32_rows(r, pre, t, stats, P, dY, mode, late=step > 3)
        del dY, P, pre
        _free()
    r.e.close()


@pytest.mark.parametrize("cid", [p.values[0] for p in PARAMS if p.values[1] == "bf16"])
def test_clusters_stages_bf16(cid):
    """bf16: the row pass at step 1, the carried normalisation after it, the forward from its own operands (and at step 1
    the density pair against the unsplit d_source), the loss stage and the streaming update, at steps 1 and 3 (and 998,
    1,000 on the C4 and tutorial shapes)."""
    torch = _torch()
    r = _run(cid, "bf16")
    V = r.V
    threads, _, per = row_pass_layout(r.ld)
    for step in _steps(cid):
        _catch_up(r, step)
        pre = _state(r)
        t = r.e.get_state()
        assert t == step - 1
        mode = f"{cid} bf16[{step}]"
        r.e.step_begin()
        check = step not in (2, 999)
        if step == 1:
            stats = r.buf("stats", 4)
            _check_row_pass_tight(r, pre[0], r.nv("Pb"), stats, f"{mode} row pass", p_extra=UB)
            assert bool((r.buf("inv_zt") == 1).all()), "z~ = 1 on a fresh P"
        elif check:
            _check_carry(r, pre[0], f"{mode} carry")
        stats = r.buf("stats", 4)
        lseT_now = r.buf("lseT")
        Pt = r.nv("Pb")[:, :V]
        Ss = _bf16_round(r.S.float() * r.buf("inv_zt").float()[:, None])
        r.e.step_end(LR)
        if not check:
            continue
        ce, cf, cb = _bf16_forward_consts(r)
        exact = (ce + 2 * UB * UB, cf + 2 * UB * UB, cb + 2 * UB * UB) if step == 1 else None
        Yd = r.buf("Y", r.Ke)
        _check_forward_blocks(r, Yd, Pt, (ce, cf, cb), mode, S=Ss, exact_pair=exact)
        del Ss, Pt
        # per-row |M|, M^2: the row pass at step 1, the previous streaming update (8 columns per lane) after it
        row_depth = per + 2 + int(np.log2(threads)) if step == 1 else 8 * _cdiv(V, 256) + 5
        dY = r.buf("dY", r.Ke)
        _check_loss_stage_tight(r, Yd, dY, r.e.history()[-1], pre[0], stats, row_depth, mode)
        del Yd, dY
        _free()
        _check_bf16_update_step(r, pre, t, lseT_now, mode, late=step > 3)
        assert torch.count_nonzero(r.nv("Pb")[:, V:]) == 0, "pad columns of P~"
        del pre
        _free()
    r.e.close()
