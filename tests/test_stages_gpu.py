"""Each stage of one iteration checked on what it writes, against float64 recomputed from the device's own inputs to that
stage, in all three arithmetic modes.  The end-to-end tests see these stages only through the loss, and two properties of
the algorithm hide whole classes of errors there: Adam is scale-invariant in the gradient, and the cosine terms are
scale-invariant in the columns of Y.  Here every stage gets

* an elementwise a-priori bound |err| <= c u (|A||B|) with the unit roundoff u and the chain length of its mode (wrong
  tiles, wrong columns, pad leakage, ragged-edge slips), and
* a statistical check: the rel-Frobenius error against a sqrt(k) u-class figure and the signed mean of err / (|A||B|)
  (a bias: truncation, a dropped term, a wrong rounding mode).

Unit roundoffs: fp32 u = 2^-24 (round to nearest); bf16 u_b = 2^-8 (8 significant bits, round to nearest).  A tensor-core
fp32 accumulator truncates, so one add costs up to one ulp (2u relative) instead of half of one.

Observed maxima over all shapes and steps, as fractions of each bound (H100 80GB HBM3, 700 W power limit):

    stage                         elementwise   rel-Fro   bias
    row pass log z / 1/z / P      0.31          0.09      0.02
    row pass h                    0.01          0.003     0.001
    forward Y_ext, fp32           0.017         0.075     0.22
    forward Y_ext, bf16x3         0.022         0.16      0.16
    forward Y_ext, bf16           0.56          0.56      0.56     (all-positive density column, 8250-cell chunk)
    loss stage dY_ext             0.14          0.016     0.17     (history row: 0.007)
    backward dP, bf16x3           0.022         0.26      0.12     (Ke 64 .. 5056; fixed 8 u / 4 u bounds)
    row-dot                       0.017         0.031     0.032
    update step, fp32 / bf16x3    -             0.34      0.41     (M, m, v elementwise: within)
    update step, bf16             -             0.56      0.12     (m's bf16 rounding bias: 0.055)
    bf16 carry lseT / P~/z~ / h   0.11          0.71      0.21
    bf16 z~                       0.043         0.028     0.01
"""
import numpy as np
import pytest

from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph, synthetic_inputs

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
UB = 2.0 ** -8          # bf16 unit roundoff
UM = 2.0 ** -21         # MUFU ex2 / rcp / sqrt .approx.ftz: <= 2^-22.5 .. 2^-22 relative, doubled
B1, B2, EPS, LR = 0.9, 0.999, 1e-8, 0.1
ALL_TERMS = dict(lambda_g2=0.5, lambda_r=1e-3, lambda_l1=1e-7, lambda_l2=1e-7, lambda_neighborhood_g1=0.96,
                 lambda_ct_islands=0.17, lambda_getis_ord=0.71)


def _torch():
    import torch
    return torch


def _g(x):
    """host array -> float64 tensor on the GPU"""
    torch = _torch()
    return torch.as_tensor(np.asarray(x, dtype=np.float64), device="cuda")


class Run:
    """An Engine plus the float64 copies of its inputs.  rows=(r0, r1): a cell shard holding rows [r0, r1) of the N cells'
    inputs and initial mapping (n_cells_global = N); self.N is then the shard's row count."""

    def __init__(self, precision, N, V, K, seed=0, T=0, clusters=False, lam=None, rows=None):
        from tangram_b200 import _lib
        from tangram_b200.engine import Engine
        lam = dict(lam or {})
        r0, r1 = rows or (0, N)
        rs = slice(r0, r1)
        self.precision, self.N, self.V, self.K, self.T, self.clusters, self.lam = precision, r1 - r0, V, K, T, clusters, lam
        inp = synthetic_inputs(N, V, K, seed=seed, n_types=T, clusters=clusters)
        self.e = Engine(r1 - r0, V, K, n_types=T, n_cells_global=N, precision=precision, lambda_d=1.0,
                        density_mode=_lib.DENSITY_SOURCE if clusters else _lib.DENSITY_CELLS, **lam)
        self.e.set_expression(np.ascontiguousarray(inp["S"][rs]), inp["G"])
        d_source = inp.get("d_source")
        self.e.set_density(inp["d"], None if d_source is None else np.ascontiguousarray(d_source[rs]))
        self.graphs = {}
        if lam.get("lambda_neighborhood_g1") or lam.get("lambda_ct_islands") or lam.get("lambda_getis_ord"):
            conn, dist = grid_graph(V)
            self.graphs = {_lib.GRAPH_VOXEL_WEIGHTS: spatial_weights_from_graph(conn, dist, True, True),
                           _lib.GRAPH_NEIGHBORHOOD_FILTER: spatial_weights_from_graph(conn, dist, False, False),
                           _lib.GRAPH_SPATIAL_WEIGHTS: spatial_weights_from_graph(conn, dist, False, True)}
            for which, mat in self.graphs.items():
                self.e.set_graph(which, mat)
            self.e.set_ct_encode(np.ascontiguousarray(inp["ct_encode"][rs]))
        self.e.set_mapping(np.ascontiguousarray(np.random.default_rng(seed + 1).standard_normal((N, V)).astype(np.float32)[rs]))
        self.inp = inp
        self.Ke, self.ld, self.splits, _, self.nchunks = (int(x) for x in self.e.debug("shape"))
        self.S = _g(self.e.debug("Sx").reshape(self.N, self.Ke))   # fp32 S_ext the contractions read, widened
        self.G = _g(inp["G"])
        self.d = _g(inp["d"])

    def buf(self, name, cols=None):
        x = self.e.debug(name)
        return _g(x.reshape(-1, cols) if cols else x)

    def nv(self, name):
        return self.buf(name, self.ld)


def _check(what, got, ref, scale, c_elem, c_fro, c_bias, floor=0.0):
    """err = got - ref: |err| <= c_elem * scale + floor elementwise, ||err|| <= c_fro ||scale||, and the bias
    |mean(sign(ref) err / scale)| <= c_bias over scale > 0 (negative: the result shrinks, as a truncating accumulator makes
    it).  Returns the observed ratios."""
    torch = _torch()
    err = got - ref
    bound = c_elem * scale + floor
    ratio = float((err.abs() / torch.where(bound > 0, bound, torch.ones_like(bound))).max()) if err.numel() else 0.0
    zero_bound = (bound == 0) & (err != 0)
    fro = float(err.norm() / scale.norm()) if float(scale.norm()) > 0 else 0.0
    live = scale > 0
    bias = float((torch.sign(ref[live]) * err[live] / scale[live]).mean()) if bool(live.any()) else 0.0
    print(f"[stage] {what}: max err/bound {ratio:.3g}, rel-Fro {fro:.3g} (bound {c_fro:.3g}), bias {bias:.3g} "
          f"(bound {c_bias:.3g})")
    assert not bool(zero_bound.any()), f"{what}: nonzero where the bound is zero, first at {torch.nonzero(zero_bound)[0].tolist()}"
    assert ratio <= 1.0, f"{what}: max err / bound {ratio:.3g}, first at {torch.nonzero(err.abs() > bound)[0].tolist()}"
    assert fro <= c_fro, f"{what}: rel-Frobenius {fro:.3g} > {c_fro:.3g}"
    assert abs(bias) <= c_bias, f"{what}: bias {bias:.3g} beyond {c_bias:.3g}"
    return ratio, fro, bias


def _x3_contraction_consts(chain, splits=1):
    """bf16x3 contraction over `chain` products per accumulator.  Operands are hi + mid + lo to 2^-24 (P, whose planes
    reconstruct the fp32 value exactly) or 2^-26 relative; the three dropped partial products (m,l) (l,m) (l,l) are below
    2^-26 |a||b|.  The k-loop runs once per partial product into one fp32 accumulator that truncates: 6 chain / 16 adds
    (one per wgmma) of at most one ulp each, plus the fp32 round-to-nearest sum of `splits` partial planes:
        |err| <= (4 + 2 (6 chain / 16 + 16) + splits) u (|A||B|)
    Statistically the truncation is a one-sided drift carried by the (h,h) pass: each of its chain / 16 wgmma adds
    truncates an accumulator that grows to |A| linearly, on average half of it, by up to two ulps (4u; the 16 products are
    aligned to the accumulator before they are summed), so the result shrinks by at most chain / 8 u relative:
    shrinkage bias <= (chain / 8 + 4) u, rel-Fro <= (chain / 8 + 8) u.  obs: 0.57 of it where every term has the same sign
    (the density column of a 8250-cell bf16 chunk), 0.17 for the forward's gene columns; a forward chain of 8200 cells
    that is not cut at 2048 drifts past it."""
    adds = 6 * ((chain + 15) // 16)
    return (4 + 2 * (adds + 16) + splits) * U, (chain / 8 + 8) * U, (chain / 8 + 4) * U


# The backward's single chain over Ke is not cut (DESIGN 2): dY_ext has both signs, so its partial sums do not grow with
# the chain and the truncation stays at rounding level whatever Ke is.  Pinned here at a few u, chain-independent, far below
# the (chain / 8) u a same-sign chain of 5056 terms may drift (obs at Ke = 5056: rel-Fro 2.1 u, bias 0.5 u).
X3_BWD_FRO, X3_BWD_BIAS = 8 * U, 4 * U


def _x3_forward_consts(r):
    """The forward's chains are cut at 2048 cells (DESIGN 2), summed over `splits` partial planes; the reference is the
    float64 softmax, so P's own row-pass error (below) adds (V + 16 + max |M - mx|) u elementwise and 16 u to the
    statistics."""
    ce, cf, cb = _x3_contraction_consts(min(-(-r.N // r.splits), 2048), r.splits)
    return ce + (r.V + 16 + 12) * U, cf + 16 * U, cb + 16 * U


# ---------------------------------------------------------------------------------------------------------------- row pass
def _check_row_pass(r, M, P_dev, stats, mode):
    """P = expf(M - mx) (1 / z) (IEEE expf <= 2 ulp, z summed in fp32 over V elements, one product), mx exact:
         |log z - ref| <= (V + 4) u,   |P - ref| <= (V + 12 + |M - mx|) u P   (+ u P when P is split into three planes)
    rel-Fro and bias: the row sums' error is a per-row constant, sqrt-class in practice: <= 16 u."""
    torch = _torch()
    V = r.V
    Mv = M[:, :V]
    mx = Mv.max(dim=1).values
    assert torch.equal(stats[:, 0], mx), "row max"
    lse = torch.logsumexp(Mv, dim=1)
    _check(f"{mode} log z", stats[:, 2], lse - mx, torch.ones_like(mx), (V + 4) * U, (V + 4) * U, (V + 4) * U)
    _check(f"{mode} 1 / z", stats[:, 1], torch.exp(mx - lse), torch.exp(mx - lse), (V + 4) * U, 16 * U, 16 * U)
    Pref = torch.softmax(Mv, dim=1)
    c = (V + 13 + (Mv - mx[:, None]).abs()) * U
    err_ok = (P_dev[:, :V] - Pref).abs() <= c * Pref
    assert bool(err_ok.all()), f"{mode} P: {int((~err_ok).sum())} elements off"
    _check(f"{mode} P (stat)", P_dev[:, :V], Pref, Pref, 1.0, 16 * U, 16 * U)
    assert torch.count_nonzero(P_dev[:, V:]) == 0, "pad columns of P"
    if r.lam.get("lambda_r"):
        logP = torch.log_softmax(Mv, dim=1)
        h = (Pref * logP).sum(dim=1)
        scale = (Pref * logP.abs()).sum(dim=1) + 1.0
        _check(f"{mode} h", stats[:, 3], h, scale, 2 * (V + 16) * U, 2 * (V + 16) * U, 2 * (V + 16) * U)
    return Pref


# ----------------------------------------------------------------------------------------------------------------- forward
def _check_forward(r, Y_dev, P, c_elem, c_fro, c_bias, mode, S=None):
    """Y_ext = P^T S_ext: the gene columns, the density pair (its hi + lo sum in clusters mode) and the cell-type columns,
    zero past them."""
    torch = _torch()
    K, T = r.K, r.T
    S = r.S if S is None else S
    Yref = P.t() @ S
    scale = P.t() @ S.abs()
    _check(f"{mode} Y genes", Y_dev[:, :K], Yref[:, :K], scale[:, :K], c_elem, c_fro, c_bias)
    dsum = Y_dev[:, K] + Y_dev[:, K + 1]
    _check(f"{mode} Y density", dsum, Yref[:, K] + Yref[:, K + 1], scale[:, K] + scale[:, K + 1], c_elem, c_fro, c_bias)
    if T:
        _check(f"{mode} Y ct", Y_dev[:, K + 2:K + 2 + T], Yref[:, K + 2:K + 2 + T], scale[:, K + 2:K + 2 + T], c_elem, c_fro, c_bias)
    assert torch.count_nonzero(Y_dev[:, K + 2 + T:]) == 0, "Y_ext past the last used column"
    return Yref


# -------------------------------------------------------------------------------------------------------------- loss stage
def _loss_of_Y(r, Yx, M):
    """The loss as a function of Y_ext (float64, autograd-able), plus the row terms from M; -> (total, {hist col: value})."""
    torch = _torch()
    lam, K, T, N, V = r.lam, r.K, r.T, r.N, r.V

    def cos_cols(a, b):
        na = torch.clamp(torch.linalg.vector_norm(a, dim=0), min=1e-8)
        nb = torch.clamp(torch.linalg.vector_norm(b, dim=0), min=1e-8)
        return (a * b).sum(dim=0) / (na * nb)

    def op(which):
        return _g(r.graphs[which].toarray())

    Y, G = Yx[:, :K], r.G
    terms = {}
    gv = cos_cols(Y, G).mean()
    terms[1] = gv
    total = -gv
    if lam.get("lambda_g2"):
        vg = cos_cols(Y.t(), G.t()).mean()
        terms[2] = vg
        total = total - lam["lambda_g2"] * vg
    dens = Yx[:, K] + Yx[:, K + 1]
    dhat = dens if r.clusters else dens / N
    kl = (torch.special.xlogy(r.d, r.d) - r.d * torch.log(dhat)).sum()
    terms[3] = kl
    total = total + kl
    Mv = M[:, :V]
    if lam.get("lambda_r"):
        ent = -(torch.softmax(Mv, 1) * torch.log_softmax(Mv, 1)).sum()
        terms[4] = ent
        total = total + lam["lambda_r"] * ent
    if lam.get("lambda_l1"):
        terms[5] = Mv.abs().sum()
        total = total + lam["lambda_l1"] * terms[5]
    if lam.get("lambda_l2"):
        terms[6] = (Mv * Mv).sum()
        total = total + lam["lambda_l2"] * terms[6]
    if lam.get("lambda_neighborhood_g1"):
        W = op(0)
        c = cos_cols(W @ Y, W @ G).mean()
        terms[7] = c
        total = total - lam["lambda_neighborhood_g1"] * c
    if lam.get("lambda_ct_islands"):
        C = Yx[:, K + 2:K + 2 + T]
        R = C - op(1) @ C
        ct = torch.clamp(R, min=0).mean()
        terms[8] = ct
        total = total + lam["lambda_ct_islands"] * ct
    if lam.get("lambda_getis_ord"):
        A = op(2)
        c = cos_cols((A @ Y) / Y.sum(dim=0), (A @ G) / G.sum(dim=0)).mean()
        terms[9] = c
        total = total - lam["lambda_getis_ord"] * c
    terms[0] = total
    return total, terms


def _check_loss_stage(r, Y_dev, dY_dev, hist, M, mode):
    """History row and dY_ext = dL/dY_ext against autograd of the loss written as a function of the device's Y_ext.
    Every loss quantity is a handful of fp32 reductions over V voxels or K genes (norms, dots, sums):
        |term - ref| <= 4 (V + K) u max(1, |ref|),   |dY - ref|_jk <= 4 (V + K) u max_j |ref_jk|
    (the cosine gradient a_jk - b_jk cancels; its parts are bounded by the column's largest gradient).  rel-Fro / bias:
    sqrt-class, 4 sqrt(V + K) u."""
    torch = _torch()
    Yx = Y_dev.clone().requires_grad_(True)
    total, terms = _loss_of_Y(r, Yx, M)
    (dref,) = torch.autograd.grad(total, Yx)
    n = r.V + r.K
    for col, val in terms.items():
        got, want = float(hist[col]), float(val)
        # entropy, L1, L2 and the total also sum over the N cells
        tol = 4 * (n + (r.N if col in (0, 4, 5, 6) else 0)) * U * max(1.0, abs(want))
        print(f"[stage] {mode} history column {col}: err {abs(got - want):.3g} (bound {tol:.3g})")
        assert abs(got - want) <= tol, f"{mode} history column {col}: {got} vs {want}"
    colmax = dref.abs().max(dim=0, keepdim=True).values.expand_as(dref)
    c = 4 * n * U
    if r.precision == "bf16":
        # dY_ext is kept as one bf16 plane: one round to nearest more, u_b |ref| (tests/test_loss_stage_gpu.py)
        _check(f"{mode} dY_ext (bf16)", dY_dev, dref, colmax, c * (1 + UB), 4 * np.sqrt(n) * U + UB,
               4 * np.sqrt(n) * U + UB / 16, floor=UB * dref.abs())
    else:
        _check(f"{mode} dY_ext", dY_dev, dref, colmax, c, 4 * np.sqrt(n) * U, 4 * np.sqrt(n) * U, floor=0.0)
    return dref


# -------------------------------------------------------------------------------------------------------------- the update
def _adam64(M, m, v, g, dg, t, lr=LR):
    """torch.optim.Adam's step in float64 from (M, m, v, g) with |g error| <= dg -> (M', m', v') and first-order bounds
    of the fp32 update on them (one rounding per operation, six operations: 8 u relative slack)."""
    torch = _torch()
    bc1, bc2 = 1 - B1 ** t, 1 - B2 ** t
    m1 = m + (g - m) * (1 - B1)
    v1 = v * B2 + (1 - B2) * g * g
    den = v1.sqrt() / bc2 ** 0.5 + EPS
    step = (lr / bc1) * m1 / den
    M1 = M - step
    dm = (1 - B1) * dg + 4 * U * (m.abs() + m1.abs() + g.abs())
    dv = (1 - B2) * (2 * g.abs() * dg + dg * dg) + 4 * U * (v1 + v * B2)
    dden = dv / (2 * torch.clamp(v1.sqrt(), min=1e-30) * bc2 ** 0.5) + 4 * U * den
    dM = (lr / bc1) * (dm / den + m1.abs() * dden / (den * den)) + 8 * U * (step.abs() + M1.abs())
    return M1, m1, v1, dM, dm, dv


def _grad_terms(r, M, P, base, lse, h):
    """g = P (base - lam_r (log P - h)) + lam_l1 sign(M) + 2 lam_l2 M with log P = M - lse (float64)"""
    torch = _torch()
    lam = r.lam
    g = base.clone()
    if lam.get("lambda_r"):
        g = g - lam["lambda_r"] * ((M - lse[:, None]) - h[:, None])
    g = g * P
    if lam.get("lambda_l1"):
        g = g + lam["lambda_l1"] * torch.sign(M)
    if lam.get("lambda_l2"):
        g = g + 2 * lam["lambda_l2"] * M
    return g


def _check_update(r, pre, post, g, dg, t, mode, m_bf16=False):
    """M, m, v after the step, pad columns included (they stay exactly zero)."""
    torch = _torch()
    V = r.V
    M0, m0, v0 = (x[:, :V] for x in pre)
    M1, m1, v1 = (x for x in post)
    Mr, mr, vr, dM, dm, dv = _adam64(M0, m0, v0, g, dg, t)
    for what, got, ref, bound in (("v", v1[:, :V], vr, dv), ("M", M1[:, :V], Mr, dM)):
        bad = (got - ref).abs() > bound
        assert not bool(bad.any()), f"{mode} update {what}: {int(bad.sum())} elements off, first {torch.nonzero(bad)[0].tolist()}"
    if m_bf16:
        # m is kept in bf16: one round-to-nearest of the fp32 value (half an ulp, 2^-8 relative), unbiased
        bound = UB * mr.abs() + dm * (1 + UB)
        bad = (m1[:, :V] - mr).abs() > bound
        assert not bool(bad.any()), f"{mode} update m: {int(bad.sum())} elements off"
        live = mr.abs() > 0
        bias = float(((m1[:, :V] - mr)[live] / mr[live].abs() * torch.sign(mr[live])).mean())
        print(f"[stage] {mode} update m (bf16) rounding bias {bias:.3g} (bound {UB / 16:.3g})")
        assert abs(bias) <= UB / 16, f"{mode} update m: rounding bias {bias:.3g}"
    else:
        bad = (m1[:, :V] - mr).abs() > dm
        assert not bool(bad.any()), f"{mode} update m: {int(bad.sum())} elements off"
    for x, name in ((M1, "M"), (m1, "m"), (v1, "v")):
        assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of {name}"
    # the step itself: err / (lr |m / denom|) signed mean and rel-Fro, sqrt-class
    stepref = M0 - Mr
    # rel-Fro: where m' cancels (0.9 m + 0.1 g ~ 0) the step's relative error is heavy-tailed, up to the elementwise bound
    _check(f"{mode} update step", M0 - M1[:, :V], stepref, stepref.abs() + dM, 1e30, 256 * U, 32 * U)


def _state(r):
    return r.nv("M"), r.nv("m"), r.nv("v")


# ================================================================================================================== tests
X3_SHAPES = [
    (2047, 300, 70, False),      # one forward chain just under the 2048 cut
    (2049, 257, 130, False),     # two chains, the second one 1 cell long; ragged 256-column tile, ld = 320
    (4100, 130, 63, False),      # three chains; 65 used columns of S_ext, one past the first 64-wide k-tile
    (6600, 200, 40, False),      # four chains of 1650 cells, twelve splits
    (1000, 100, 2100, False),    # Ke = 2112 > 2048: the backward's single chain
    (600, 70, 5000, False),      # Ke = 5056 (C4's gene count): the uncut backward chain
    (8200, 4224, 2000, False),   # 264 output tiles: one split fills the GPU, so only the 2048 cut splits the forward chain
    (300, 5, 60, False),         # V < 8: one ragged 8-column group of the update
    (1200, 263, 100, True),      # clusters mode (d_source hi + lo), V % 8 != 0
]


@pytest.mark.parametrize("N,V,K,clusters", X3_SHAPES)
def test_bf16x3_stages(N, V, K, clusters):
    """bf16x3: row pass, forward, loss stage, backward (fp32 dP and row-dot) and the exact update, each from the device's
    own inputs, at step 1 and step 3."""
    r = Run("bf16x3", N, V, K, seed=N + V + K, clusters=clusters)
    for step in range(1, 4):
        pre = _state(r)
        t = r.e.get_state()
        r.e.step_begin()
        r.e.step_end(LR)
        if step == 2:
            continue
        stats = r.buf("stats", 4)
        P3 = r.nv("Pb")
        Pref = _check_row_pass(r, pre[0], P3, stats, f"x3[{step}] row pass")
        Yd = r.buf("Y", r.Ke)
        _check_forward(r, Yd, Pref, *_x3_forward_consts(r), mode=f"x3[{step}]")
        dY = r.buf("dY", r.Ke)
        hist = r.e.history()[-1]
        _check_loss_stage(r, Yd, dY, hist, pre[0], f"x3[{step}]")
        _check_backward_x3(r, pre, t, stats, P3, dY, f"x3[{step}]")


def _check_backward_x3(r, pre, t, stats, P3, dY, mode):
    """bf16x3 backward from the device's dY_ext: dP = S_ext dY_ext^T over Ke (one chain), the row-dot
    r_i = sum_j P_ij dP_ij from the fp32 P, and the exact update from the pre-step state `pre` at step count t."""
    torch = _torch()
    V = r.V
    dpf = r.nv("dpf")
    dPref = r.S @ dY.t()
    scale = r.S.abs() @ dY.abs().t()
    ce, _, _ = _x3_contraction_consts(r.Ke)
    cf, cb = X3_BWD_FRO, X3_BWD_BIAS
    _check(f"{mode} dP (Ke {r.Ke})", dpf[:, :V], dPref, scale, ce, cf, cb)
    assert torch.count_nonzero(dpf[:, V:]) == 0, "pad columns of dP"
    rdot = r.buf("rdot")
    rref = (P3[:, :V] * dPref).sum(dim=1)
    rscale = (P3[:, :V] * scale).sum(dim=1)
    _check(f"{mode} row-dot", rdot, rref, rscale, ce + (V + 2) * 2 * U, cf + V * U, cb + 4 * U)
    # the exact update: g = (dP - r) P from the device's fp32 values (the bound check; bit equality in
    # test_bf16x3_update_is_torch_adam)
    g = _grad_terms(r, pre[0][:, :V], P3[:, :V], dpf[:, :V] - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
    if r.lam:       # entropy / L1 / L2 gradient terms: the bound of test_bf16x3_all_terms_clusters
        dg = 8 * U * (g.abs() + P3[:, :V] * (dpf[:, :V].abs() + rdot.abs()[:, None] + 1.0))
    else:
        dg = 4 * U * (g.abs() + P3[:, :V] * (dpf[:, :V].abs() + rdot.abs()[:, None]))
    _check_update(r, pre, _state(r), g, dg, t + 1, mode)


@pytest.mark.parametrize("N,V,K", [(2100, 300, 70), (700, 5, 64), (1500, 263, 130)])
def test_bf16x3_update_is_torch_adam(N, V, K):
    """The exact streaming update (k_adam_rows_exact) is torch.optim.Adam(foreach=False) on CUDA element for element.
    First, the row pass's three bf16 P planes reconstruct its fp32 P exactly (expf(M - mx) * inv_z, recomputed here with
    torch's fp32 ops from the device's row statistics): that is the P the update recomputes.  Then one Adam step in torch
    from the device's M, m, v, step count and g = (dP - r) P formed in fp32 from the device's dP and row-dot must give
    M, m and v bit for bit, at step 1 and at step 3."""
    torch = _torch()
    r = Run("bf16x3", N, V, K, seed=7 * N + V)
    for step in range(1, 4):
        M0, m0, v0 = (x[:, :V].float().contiguous() for x in _state(r))
        t = r.e.get_state()
        r.e.step_begin()
        r.e.step_end(LR)
        stats = r.buf("stats", 4).float()
        P = r.nv("Pb")[:, :V].float()
        Pf = torch.exp(M0 - stats[:, 0:1]) * stats[:, 1:2]
        assert float(P.abs().min()) > 2.0 ** -100, "a P this small puts the low plane below bf16's normal range"
        assert torch.equal(P, Pf), f"P planes vs fp32 P: {int((P != Pf).sum())} elements differ"
        if step == 2:
            continue
        dpf = r.nv("dpf")[:, :V].float()
        rdot = r.buf("rdot").float()
        g = (dpf - rdot[:, None]) * P
        p = torch.nn.Parameter(M0.clone())
        opt = torch.optim.Adam([p], lr=LR, betas=(B1, B2), eps=EPS, foreach=False, fused=False)
        p.grad = g
        opt.state[p] = {"step": torch.tensor(float(t)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
        opt.step()
        M1, m1, v1 = (x[:, :V].float() for x in _state(r))
        for name, got, want in (("v", v1, opt.state[p]["exp_avg_sq"]), ("m", m1, opt.state[p]["exp_avg"]), ("M", M1, p.detach())):
            diff = got != want
            assert not bool(diff.any()), (f"step {step}: {name} differs from torch's Adam in {int(diff.sum())} of {diff.numel()} "
                                          f"elements, first {torch.nonzero(diff)[0].tolist()}")


@pytest.mark.parametrize("lam", [{}, ALL_TERMS], ids=["default", "all-terms"])
def test_bf16x3_all_terms_clusters(lam):
    """Clusters mode with every loss term on (g2, entropy, L1/L2, neighbourhood, Getis-Ord, ct islands) and many voxel
    tiles of the row-dot: the loss stage's history row and dY_ext (density and ct columns included), the backward, and
    the update with every gradient term."""
    N, V, K, T = 1500, 700, 130, 8
    r = Run("bf16x3", N, V, K, seed=2, T=T, clusters=True, lam=lam)
    for step in range(1, 4):
        pre = _state(r)
        t = r.e.get_state()
        r.e.step_begin()
        r.e.step_end(LR)
        if step == 2:
            continue
        stats = r.buf("stats", 4)
        P3 = r.nv("Pb")
        Pref = _check_row_pass(r, pre[0], P3, stats, f"x3-terms[{step}] row pass")
        Yd = r.buf("Y", r.Ke)
        _check_forward(r, Yd, Pref, *_x3_forward_consts(r), mode=f"x3-terms[{step}]")
        dY = r.buf("dY", r.Ke)
        _check_loss_stage(r, Yd, dY, r.e.history()[-1], pre[0], f"x3-terms[{step}]")
        dpf = r.nv("dpf")
        rdot = r.buf("rdot")
        g = _grad_terms(r, pre[0][:, :V], P3[:, :V], dpf[:, :V] - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
        dg = 8 * U * (g.abs() + P3[:, :V] * (dpf[:, :V].abs() + rdot.abs()[:, None] + 1.0))
        _check_update(r, pre, _state(r), g, dg, t + 1, f"x3-terms[{step}]")


FP32_SHAPES = [(2049, 257, 130, False, {}), (1000, 300, 2100, False, {}), (300, 5, 60, False, {}),
               (1200, 263, 100, True, ALL_TERMS)]


@pytest.mark.parametrize("N,V,K,clusters,lam", FP32_SHAPES, ids=["ragged", "Ke2112", "V5", "clusters-all-terms"])
def test_fp32_stages(N, V, K, clusters, lam):
    """fp32 (FFMA): row pass, forward, loss stage, and the fused update (EpiAdam never stores dP: dP is recomputed in
    float64 from the device's S_ext and dY).  FFMA chains are round-to-nearest: |err| <= 2 k u (|A||B|), rel-Fro and bias
    sqrt(k)-class, 4 sqrt(k) u and 4 u."""
    T = 8 if lam else 0
    r = Run("fp32", N, V, K, seed=N + K, T=T, clusters=clusters, lam=lam)
    for step in range(1, 4):
        pre = _state(r)
        t = r.e.get_state()
        r.e.step_begin()
        r.e.step_end(LR)
        if step == 2:
            continue
        stats = r.buf("stats", 4)
        Pf = r.nv("Pf")
        Pref = _check_row_pass(r, pre[0], Pf, stats, f"fp32[{step}] row pass")
        Yd = r.buf("Y", r.Ke)
        _check_forward(r, Yd, Pref, *_fp32_forward_consts(r), f"fp32[{step}]")
        dY = r.buf("dY", r.Ke)
        _check_loss_stage(r, Yd, dY, r.e.history()[-1], pre[0], f"fp32[{step}]")
        _check_backward_fp32(r, pre, t, stats, Pf, dY, f"fp32[{step}]")


def _fp32_forward_consts(r):
    """FFMA forward over a chain of one split of the cells, the splits summed in fp32, P's row-pass error on top."""
    chain = -(-r.N // r.splits)
    return (2 * chain + r.splits + r.V + 32) * U, 4 * np.sqrt(chain) * U + (r.splits + 16) * U, 20 * U


def _check_backward_fp32(r, pre, t, stats, Pf, dY, mode):
    """fp32 backward from the device's dY_ext: the row-dot, and the fused update from the pre-step state `pre` at step
    count t (EpiAdam never stores dP: dP is recomputed in float64 from the device's S_ext and dY)."""
    V = r.V
    dPref = r.S @ dY.t()
    scale = r.S.abs() @ dY.abs().t()
    rdot = r.buf("rdot")
    rref = (Pf[:, :V] * dPref).sum(dim=1)
    rscale = (Pf[:, :V] * scale).sum(dim=1)
    _check(f"{mode} row-dot", rdot, rref, rscale, (2 * (r.Ke + V) + 8) * U, 4 * np.sqrt(r.Ke + V) * U, 4 * U)
    g = _grad_terms(r, pre[0][:, :V], Pf[:, :V], dPref - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
    dg = Pf[:, :V] * (2 * r.Ke + 8) * U * scale + 8 * U * (g.abs() + Pf[:, :V] * (dPref.abs() + rdot.abs()[:, None] + 1.0))
    _check_update(r, pre, _state(r), g, dg, t + 1, mode)


# ------------------------------------------------------------------------------------------------------------------ bf16
def _bf16_round(x):
    return x.float().to(_torch().bfloat16).double()


def _check_carry(r, M, mode):
    """After step_begin: lseT = lseA + log z~ against float64 logsumexp(M); P~ inv_zt against float64 softmax(M); h.
    z~ sums the fp32 values of P~ (before their bf16 rounding) over V, ex2.approx.ftz on an fma'd argument:
        |lseT - ref| <= (V + 8) u + UM (1 + |lse|),   |P~ inv_zt - P| <= (u_b + (V + 8) u + UM (2 + |M| + |lse|)) P
    P~ carries one bf16 rounding each: rel-Fro <= u_b, |bias| <= u_b / 16.  h = px / z~ - lseT cancels:
        |h - ref| <= ((V + 8) u + UM (2 + |lse|)) (sum_j P |M| + |lse|)."""
    torch = _torch()
    V = r.V
    Mv = M[:, :V]
    lse = torch.logsumexp(Mv, dim=1)
    lseT = r.buf("lseT")
    _check(f"{mode} lseT", lseT, lse, torch.ones_like(lse), (V + 8) * U + UM * (1 + lse.abs().max().item()),
           (V + 8) * U + UM * (1 + lse.abs().max().item()), (V + 8) * U + UM * (1 + lse.abs().max().item()))
    Pref = torch.softmax(Mv, dim=1)
    Pt = r.nv("Pb")
    izt = r.buf("inv_zt")
    P = Pt[:, :V] * izt[:, None]
    c = UB + (V + 8) * U + UM * (2 + Mv.abs() + lse.abs()[:, None])
    bad = (P - Pref).abs() > c * Pref
    assert not bool(bad.any()), f"{mode} P~ / z~: {int(bad.sum())} elements off"
    _check(f"{mode} P~ / z~ (stat)", P, Pref, Pref, 1e30, UB, UB / 16)
    assert torch.count_nonzero(Pt[:, V:]) == 0, "pad columns of P~"
    stats = r.buf("stats", 4)
    if r.lam.get("lambda_r"):
        h = (Pref * torch.log_softmax(Mv, dim=1)).sum(dim=1)
        scale = (Pref * Mv.abs()).sum(dim=1) + lse.abs()
        ce = (V + 8) * U + UM * (2 + lse.abs().max().item())
        _check(f"{mode} h", stats[:, 3], h, scale, ce, ce, ce)
    return Pref, lse, izt


BF16_SHAPES = [
    (2049, 257, 130, 0.0),       # one chunk; ragged tiles
    (9000, 300, 70, 1e-3),       # two cell chunks, the last one ragged; entropy term on
    (33000, 130, 40, 1e-3),      # four cell chunks (step_begin / step_end: the forward runs in step_begin)
    (1000, 5, 2100, 0.0),        # V < 8; Ke > 2048
]


@pytest.mark.parametrize("N,V,K,lam_r", BF16_SHAPES)
def test_bf16_stages(N, V, K, lam_r):
    """bf16: the row pass at step 1 (P fresh, c = 0, z~ = 1), the carried row normalisation at step >= 2, the forward
    from the bf16 P~ and S / z~ (two bf16 roundings per product, fp32 accumulation over a cell chunk), and the streaming
    update (g from the device's dq and rowc; MUFU ex2 / rcp / sqrt; m rounded to bf16), then P~ and z~ the update wrote."""
    torch = _torch()
    lam = {"lambda_r": lam_r} if lam_r else {}
    r = Run("bf16", N, V, K, seed=N + V, lam=lam)
    for step in range(1, 5):
        pre = _state(r)
        t = r.e.get_state()
        r.e.step_begin()
        if step == 1:
            stats = r.buf("stats", 4)
            Mv = pre[0][:, :V]
            Pref = torch.softmax(Mv, dim=1)
            assert torch.equal(stats[:, 0], Mv.max(dim=1).values), "row max"
            bad = (r.nv("Pb")[:, :V] - Pref).abs() > (UB + (V + 16 + (Mv - stats[:, 0:1]).abs()) * U) * Pref
            assert not bool(bad.any()), f"bf16 row pass P: {int(bad.sum())} elements off"
            assert bool((r.buf("inv_zt") == 1).all()), "z~ = 1 on a fresh P"
        else:
            Pref, _, _ = _check_carry(r, pre[0], f"bf16[{step}] carry")
        lseT_now = r.buf("lseT")
        Pt_fwd = r.nv("Pb")[:, :V]
        Ss = _bf16_round(r.S.float() * r.buf("inv_zt").float()[:, None])      # k_scale_rows_bf16
        r.e.step_end(LR)
        if step in (1, 3):
            # forward from its own operands P~ and bf16(S / z~): the products are exact in fp32, the accumulation runs over
            # a cell chunk (or a split) and truncates, like bf16x3's with one partial product instead of six; Y_ext holds
            # the complete sum once step_end has begun
            _check_forward(r, r.buf("Y", r.Ke), Pt_fwd, *_bf16_forward_consts(r), f"bf16[{step}]", S=Ss)
        if step not in (1, 3):
            continue
        _check_bf16_update_step(r, pre, t, lseT_now, f"bf16[{step}]")


def _check_bf16_update_step(r, pre, t, lseT_now, mode):
    """The bf16 streaming update from the device's dq, rowc = (lse, r', h) and the pre-step state `pre` at step count t
    (lseT_now: lseT after step_begin), then the P~ and z~ it left for the next forward."""
    torch = _torch()
    V = r.V
    dq = r.nv("dq")[:, :V]
    rowc = r.buf("rowc", 4)
    assert torch.equal(rowc[:, 0], lseT_now), "rowc carries the row's exact log-sum-exp"
    Mv = pre[0][:, :V]
    P = torch.exp(Mv - rowc[:, 0:1])
    g = _grad_terms(r, Mv, P, dq - rowc[:, 1:2], rowc[:, 0], rowc[:, 2])
    dg = (UM * (4 + 2 * Mv.abs() + 2 * rowc[:, 0:1].abs()) + 4 * U) * g.abs() + 4 * U * P * (dq.abs() + rowc[:, 1:2].abs())
    dg = dg + (r.lam.get("lambda_r", 0.0) * P * 8 * U * (Mv.abs() + rowc[:, 0:1].abs() + rowc[:, 2:3].abs()))
    post = _state(r)
    _check_update_bf16(r, pre, post, g, dg, t + 1, mode)
    # what the update left for the next forward: P~ = bf16(exp(Mnew - lse)), z~ = sum of the unrounded values
    Mn = post[0][:, :V]
    lseA = r.buf("lseA")
    assert torch.equal(lseA, lseT_now), "after step_end lseA is the offset the new P~ was written with"
    Pt_ref = torch.exp(Mn - lseA[:, None])
    Pt = r.nv("Pb")
    bad = (Pt[:, :V] - Pt_ref).abs() > (UB + UM * (2 + Mn.abs() + lseA.abs()[:, None])) * Pt_ref
    assert not bool(bad.any()), f"{mode} P~ after the update: {int(bad.sum())} elements off"
    assert torch.count_nonzero(Pt[:, V:]) == 0, "pad columns of P~"
    _check(f"{mode} z~", r.buf("zsum"), Pt_ref.sum(dim=1), Pt_ref.sum(dim=1),
           (V + 8) * U + UM * (2 + Mn.abs().max().item() + lseA.abs().max().item()), (V + 8) * U + 4 * UM, (V + 8) * U + 4 * UM)


def _bf16_forward_consts(r):
    """bf16 forward: bf16 x bf16 products are exact in fp32; one partial product per k-block, so the bf16x3 bounds with one
    pass instead of six, over a chain of one cell chunk or one split."""
    parts = max(r.splits, r.nchunks)
    chain = -(-r.N // parts)
    ce, cf, cb = _x3_contraction_consts(chain, parts)
    return ce - 2 * 5 * ((chain + 15) // 16) * U, cf, cb


@pytest.mark.parametrize("N,V,K,lam_r", [(9000, 300, 70, 1e-3), (33000, 130, 40, 0.0)])
def test_bf16_run_prefetches_the_same_forward(N, V, K, lam_r):
    """tgb200_run issues each next iteration's forward (k_row_norm, k_scale_rows_bf16 and the chunk contractions) on a
    third stream between the backward's chunks, each chunk behind the streaming update of its rows, with the lseT / lseA
    buffers swapped for it; step_begin / step_end never prefetch.  Three iterations of run() (the second and third
    forwards prefetched) must leave every buffer and the history bit-identical to three step_begin / step_end pairs, and
    the Y_ext of the last, prefetched forward is checked against float64 from its operands P~ and bf16(S / z~)."""
    torch = _torch()
    lam = {"lambda_r": lam_r} if lam_r else {}
    a = Run("bf16", N, V, K, seed=N, lam=lam)
    b = Run("bf16", N, V, K, seed=N, lam=lam)
    assert a.nchunks > 1, "the prefetch runs with more than one cell chunk"
    a.e.run(3)
    for step in range(3):
        b.e.step_begin()
        if step == 2:            # the operands of the third forward
            Pt_fwd = b.nv("Pb")[:, :V]
            Ss = _bf16_round(b.S.float() * b.buf("inv_zt").float()[:, None])
        b.e.step_end(LR)
    names = ["Y", "M", "m", "v", "Pb", "dq", "inv_zt", "lseA", "zsum", "rcenter", "rdot", "rowc", "stats"]
    if lam_r:
        names.append("pxsum")
    for name in names:
        x, y = a.e.debug(name), b.e.debug(name)
        assert np.array_equal(x, y, equal_nan=True), f"{name}: run() and step_begin / step_end differ in {int((x != y).sum())} elements"
    assert np.array_equal(a.e.history(), b.e.history(), equal_nan=True), "history"
    _check_forward(a, a.buf("Y", a.Ke), Pt_fwd, *_bf16_forward_consts(a), "bf16 run() prefetched", S=Ss)
    assert torch.count_nonzero(a.nv("Pb")[:, V:]) == 0, "pad columns of P~"


def _check_update_bf16(r, pre, post, g, dg, t, mode):
    """bf16 update bound: the MUFU rcp / sqrt add 2 UM relative to the step."""
    torch = _torch()
    V = r.V
    M0, m0, v0 = (x[:, :V] for x in pre)
    M1, m1, v1 = post
    Mr, mr, vr, dM, dm, dv = _adam64(M0, m0, v0, g, dg, t)
    dM = dM + 4 * UM * (M0 - Mr).abs()
    dv = dv + 4 * UM * vr
    for what, got, ref, bound in (("v", v1[:, :V], vr, dv), ("M", M1[:, :V], Mr, dM)):
        bad = (got - ref).abs() > bound
        assert not bool(bad.any()), f"{mode} update {what}: {int(bad.sum())} elements off, first {torch.nonzero(bad)[0].tolist()}"
    bound = UB * mr.abs() + dm * (1 + UB)
    bad = (m1[:, :V] - mr).abs() > bound
    assert not bool(bad.any()), f"{mode} update m: {int(bad.sum())} elements off"
    live = mr.abs() > 0
    bias = float(((m1[:, :V] - mr)[live] / mr[live].abs() * torch.sign(mr[live])).mean())
    print(f"[stage] {mode} update m (bf16 round to nearest) bias {bias:.3g} (bound {UB / 16:.3g})")
    assert abs(bias) <= UB / 16, f"{mode} update m: rounding bias {bias:.3g}"
    for x, name in ((M1, "M"), (m1, "m"), (v1, "v")):
        assert torch.count_nonzero(x[:, V:]) == 0, f"{mode}: pad columns of {name}"
    stepref = M0 - Mr
    _check(f"{mode} update step", M0 - M1[:, :V], stepref, stepref.abs() + dM, 1e30, 8 * UM, 2 * UM)


def test_bf16_carry_horizon():
    """300 bf16 steps with the entropy term on: the carried lseT, P~ / z~ and h stay within the one-step bound (no drift
    of the row normalisation), and the pad columns of M, m, v and P~ are exactly zero."""
    torch = _torch()
    N, V, K = 2100, 263, 70
    r = Run("bf16", N, V, K, seed=5, lam={"lambda_r": 1e-3})
    r.e.run(299)
    r.e.step_begin()
    r.e.step_end(LR)
    r.e.step_begin()
    M = r.nv("M")
    _check_carry(r, M, "bf16[301] carry")
    for name in ("M", "m", "v", "Pb"):
        assert torch.count_nonzero(r.nv(name)[:, V:]) == 0, f"pad columns of {name} after 300 steps"
    r.e.step_end(LR)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_get_mapping_is_softmax_of_state(precision):
    """get_mapping = fp32 softmax of get_state's M: |P - ref| <= (V + 12 + |M - mx|) u P."""
    torch = _torch()
    N, V, K = 1500, 263, 70
    r = Run(precision, N, V, K, seed=3, lam={"lambda_r": 1e-3})
    r.e.run(3)
    M = np.empty((N, V), dtype=np.float32)
    r.e.get_state(M=M)
    out = r.e.get_mapping(np.empty((N, V), dtype=np.float32))
    Mg = _g(M)
    Pref = torch.softmax(Mg, dim=1)
    c = (V + 13 + (Mg - Mg.max(dim=1, keepdim=True).values).abs()) * U
    bad = (_g(out) - Pref).abs() > c * Pref
    assert not bool(bad.any()), f"{int(bad.sum())} elements off"
    _check(f"{precision} get_mapping", _g(out), Pref, Pref, 1e30, 16 * U, 16 * U)
