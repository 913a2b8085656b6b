"""Each stage of the constrained (filter) iteration -- `MapperConstrained`, `map_cells_to_space(mode="constrained")` --
checked on what it writes against float64 recomputed from the device's own inputs to that stage, in all three arithmetic
modes, with the bounds and checkers of tests/test_stages_gpu.py.  The filter adds four stages to the plain iteration:

* k_filter_prepare: f = sigmoid(F) and S_f = f o S_ext, the operand of every contraction;
* the tail k_row_scalar_reduce writes after Y_ext: sum f and sum (f - f^2);
* the constrained branch of k_loss_scalars: dhat = colsum / sum f, the count and f-reg terms and
  fscal = (lambda_d sum d / sum f, sign(sum f - target_count));
* k_filter_update: dL/dF from the row-dot, f and fscal, then F's own Adam step.

End-to-end runs see dL/dF only through Adam, which is scale-invariant in the gradient, so the gradient is checked here
against float64 autograd of the whole loss as a function of (M, F), and F's step against torch.optim.Adam bit for bit.
A saturated filter cell (f exactly 0 or 1 in fp32) must keep its F: dL/dF = dL/df f (1 - f) is 0 there.

Observed maxima over all shapes and steps, as fractions of each bound (H100 80GB HBM3, 400 W power limit):

    stage                          elementwise   rel-Fro   bias
    f = sigmoid(F)                 0.46          0.12      0.016    (logits -87 .. 30: 0.38)
    tail sum f / sum (f - f^2)     0.003         -         -
    forward Y_ext (S_f), fp32      0.017         0.041     0.050
    forward Y_ext (S_f), bf16x3    0.031         0.17      0.18
    forward Y_ext (S_f), bf16      0.17          0.20      0.21
    loss stage dY_ext              0.076         0.029     0.018
    loss stage dY_ext, bf16 copy   0.97          0.69      0.055
    fscal[0]                       0.062         -         -
    dP = S_f dY^T, bf16x3          0.019         0.074     0.12
    row-dot, fp32 / bf16x3         0.020         0.056     0.064
    row-dot, bf16                  0.72          -         -
    dL/dF                          0.21          -         -
    M update step                  -             0.37      0.21
F, mF and vF equal torch's Adam step bit for bit in every mode; get_filter's sigmoid equals torch.sigmoid bit for bit.
"""
import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs
from tests.test_stages_gpu import (B1, B2, EPS, LR, U, UB, UM, X3_BWD_BIAS, X3_BWD_FRO, _adam64, _bf16_forward_consts,
                                   _bf16_round, _check, _check_forward, _check_row_pass, _check_update, _check_update_bf16,
                                   _g, _grad_terms, _x3_contraction_consts, _x3_forward_consts)

pytestmark = pytest.mark.gpu

REF_DEFAULTS = dict(lambda_g2=1.0, lambda_count=1.0, lambda_f_reg=1.0)     # MapperConstrained's defaults (:445-457)


def _torch():
    import torch
    return torch


class CRun:
    """A constrained-mode Engine plus the float64 copies of its inputs.  `target` is target_count as a fraction of N."""

    def __init__(self, precision, N, V, K, seed=0, lam=None, density=True, target=0.3, F0=None, F_scale=2.0):
        from tangram_b200 import _lib
        from tangram_b200.engine import Engine
        lam = dict(REF_DEFAULTS if lam is None else lam)
        self.precision, self.N, self.V, self.K, self.T, self.lam, self.density = precision, N, V, K, 0, lam, density
        self.target = float(np.float32(target * N))
        inp = synthetic_inputs(N, V, K, seed=seed)
        self.e = Engine(N, V, K, precision=precision, density_mode=_lib.DENSITY_CELLS if density else _lib.DENSITY_NONE,
                        constrained=True, target_count=self.target, **lam)
        self.e.set_expression(inp["S"], inp["G"])
        if density:
            self.e.set_density(inp["d"])
        rng = np.random.default_rng(seed + 1)
        self.e.set_mapping(rng.standard_normal((N, V)).astype(np.float32))
        if F0 is None:
            # f from ~1e-4 to 1 - 1e-4 (1 - f cancels); smaller f make M's gradient on those rows so small that its Adam
            # step drops below M's rounding (and g^2 below fp32's normal range), which the update checks do not model.
            # Far wider logits are checked on their own (test_filter_prepare_wide_logits).
            F0 = F_scale * rng.standard_normal(N)
        self.e.set_filter(np.ascontiguousarray(F0, dtype=np.float32))
        self.Ke, self.ld, self.splits, _, self.nchunks = (int(x) for x in self.e.debug("shape"))
        self.Sx = _g(self.e.debug("Sx").reshape(N, self.Ke))       # S_ext, widened (density column of ones, or zeros)
        self.S = self.Sx
        self.G = _g(inp["G"])
        self.d = _g(inp["d"]) if density else None
        self.inp = inp

    def buf(self, name, cols=None):
        x = self.e.debug(name)
        return _g(x.reshape(-1, cols) if cols else x)

    def nv(self, name):
        return self.buf(name, self.ld)

    def lam_of(self, k):
        return float(np.float32(self.lam.get(k, 0.0)))


def _cos_cols(a, b):
    torch = _torch()
    na = torch.clamp(torch.linalg.vector_norm(a, dim=0), min=1e-8)
    nb = torch.clamp(torch.linalg.vector_norm(b, dim=0), min=1e-8)
    return (a * b).sum(dim=0) / (na * nb)


def _closs(r, Yx, f, M):
    """The constrained loss (mapping_optimizer.py:506-575) as a function of Y_ext, f and M (float64, autograd-able)
    -> (total, {history column: value})."""
    torch = _torch()
    K, V = r.K, r.V
    Y = Yx[:, :K]
    terms = {}
    gv = _cos_cols(Y, r.G).mean()
    terms[1] = gv
    total = -gv
    if r.lam.get("lambda_g2"):
        vg = _cos_cols(Y.t(), r.G.t()).mean()
        terms[2] = vg
        total = total - r.lam_of("lambda_g2") * vg
    s = f.sum()
    if r.density:
        dhat = (Yx[:, K] + Yx[:, K + 1]) / s
        kl = (torch.special.xlogy(r.d, r.d) - r.d * torch.log(dhat)).sum()
        terms[3] = kl
        total = total + kl
    if r.lam.get("lambda_r"):
        Mv = M[:, :V]
        ent = -(torch.softmax(Mv, 1) * torch.log_softmax(Mv, 1)).sum()
        terms[4] = ent
        total = total + r.lam_of("lambda_r") * ent
    terms[10] = (s - r.target).abs()
    terms[11] = (f - f * f).sum()
    total = total + r.lam_of("lambda_count") * terms[10] + r.lam_of("lambda_f_reg") * terms[11]
    terms[0] = total
    return total, terms


def _filter_grad32(r, rdot, f, fscal):
    """dL/dF as k_filter_update forms it, in torch fp32 with the kernel's operation order (one rounding per op)."""
    torch = _torch()
    rdot, f, fscal = rdot.float(), f.float(), fscal.float()
    lc = torch.tensor(r.lam_of("lambda_count"), dtype=torch.float32, device="cuda")
    lf = torch.tensor(r.lam_of("lambda_f_reg"), dtype=torch.float32, device="cuda")
    omf = 1 - f
    c = (fscal[0] + lc * fscal[1]) + lf * (1 - 2 * f)
    return rdot * omf + c * (f * omf)


def _torch_adam_step(x0, m0, v0, g, t):
    """One torch.optim.Adam(foreach=False) step on CUDA from the given fp32 state and step count -> (x, m, v)."""
    torch = _torch()
    p = torch.nn.Parameter(x0.float().clone())
    opt = torch.optim.Adam([p], lr=LR, betas=(B1, B2), eps=EPS, foreach=False, fused=False)
    p.grad = g.float().clone()
    opt.state[p] = {"step": torch.tensor(float(t)), "exp_avg": m0.float().clone(), "exp_avg_sq": v0.float().clone()}
    opt.step()
    return p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]


def _check_filter_prepare(r, F0, f, Sf, mode):
    """f = 1 / (1 + expf(-F)): IEEE expf is within 2 ulp (<= 4 u relative) of e = exp(-F); 1 + e carries it scaled by
    e / (1 + e) <= 1 plus one rounding, the division one more: |f - sigmoid(F)| <= 6 u sigmoid(F) (a floor of one
    subnormal step where f drops below 2^-126).  S_f = f o S_ext is one fp32 product per element: bit for bit."""
    torch = _torch()
    ref = torch.sigmoid(F0)
    _check(f"{mode} f = sigmoid(F)", f, ref, ref, 6 * U, 6 * U, 6 * U, floor=2.0 ** -149)
    want = f.float()[:, None] * r.Sx.float()
    diff = Sf.float() != want
    assert not bool(diff.any()), f"{mode} S_f != f o S_ext in {int(diff.sum())} elements, first {torch.nonzero(diff)[0].tolist()}"


def _check_tail(r, tail, f, mode):
    """sum f and sum (f - f^2) in fp32 over N cells (per-thread chains of N / 1024, then a 1024-wide tree): <= N u of the
    sum of the magnitudes; f - f^2 adds one product and one difference per term, <= 2 u f each (f - f^2 cancels near
    f = 1, so its scale is sum f, not sum (f - f^2))."""
    N = r.N
    fs, fr = f.sum(), (f - f * f).sum()
    e0, e1 = abs(float(tail[3] - fs)), abs(float(tail[4] - fr))
    b0, b1 = N * U * float(fs), N * U * float(fr) + 2 * U * float(fs)
    print(f"[stage] {mode} tail: sum f err/bound {e0 / b0:.3g}, sum (f - f^2) err/bound {e1 / b1:.3g}")
    assert e0 <= b0, f"{mode} sum f: {float(tail[3])} vs {float(fs)}"
    assert e1 <= b1, f"{mode} sum (f - f^2): {float(tail[4])} vs {float(fr)}"


def _check_closs_stage(r, Y_dev, dY_dev, hist, fscal, f, M, mode):
    """History row, dY_ext and fscal against autograd of the constrained loss as a function of the device's Y_ext and f.
    As in test_stages_gpu: every loss quantity is a handful of fp32 reductions over V voxels or K genes,
    |term - ref| <= 4 (V + K) u max(1, |ref|), |dY - ref|_jk <= 4 (V + K) u max_j |ref_jk|; the terms summed over the N
    cells (total, entropy, count, f-reg) add N, and their scale includes sum f (the count |sum f - target| cancels).
    fscal[0] = lambda_d sum d / sum f: two tree sums ((V + N) / 1024 + 20 u), a division and a product.
    fscal[1] = sign(sum f - target) exactly."""
    torch = _torch()
    Yx = Y_dev.clone().requires_grad_(True)
    total, terms = _closs(r, Yx, f, M)
    (dref,) = torch.autograd.grad(total, Yx)
    n = r.V + r.K
    fs = float(f.sum())
    for col, val in terms.items():
        got, want = float(hist[col]), float(val)
        summed = col in (0, 3, 4, 10, 11)
        tol = 4 * (n + (r.N if summed else 0)) * U * max(1.0, abs(want), fs if col in (0, 10, 11) else 0.0)
        print(f"[stage] {mode} history column {col}: err {abs(got - want):.3g} (bound {tol:.3g})")
        assert abs(got - want) <= tol, f"{mode} history column {col}: {got} vs {want}"
    if not r.density:
        assert np.isnan(float(hist[3])), "KL column without a density"
    colmax = dref.abs().max(dim=0, keepdim=True).values.expand_as(dref)
    if r.precision == "bf16":
        # the bf16 mode keeps only dY_ext's bf16 copy (the backward's operand): one round to nearest more, unbiased
        _check(f"{mode} dY_ext (bf16)", dY_dev, dref, colmax, 4 * n * U + UB, 4 * np.sqrt(n) * U + UB, 4 * np.sqrt(n) * U + UB / 16)
    else:
        _check(f"{mode} dY_ext", dY_dev, dref, colmax, 4 * n * U, 4 * np.sqrt(n) * U, 4 * np.sqrt(n) * U)
    if r.density:
        ref0 = float(r.d.sum()) / fs                       # lambda_d = 1
        b0 = ((r.V + r.N) / 1024 + 24) * U * abs(ref0)
        print(f"[stage] {mode} fscal[0]: err/bound {abs(float(fscal[0]) - ref0) / b0:.3g}")
        assert abs(float(fscal[0]) - ref0) <= b0, f"{mode} fscal[0] = {float(fscal[0])}, want {ref0}"
    else:
        assert float(fscal[0]) == 0.0, "fscal[0] without a density"
    cnt = fs - r.target
    assert abs(cnt) > 1e-3 * fs, "sum f too close to target_count for its sign to be checked"
    assert float(fscal[1]) == float(np.sign(cnt)), f"{mode} fscal[1] = {float(fscal[1])}, sum f - target = {cnt}"
    return dref


def _full_grad_F(r, M0, F0):
    """float64 autograd of the whole loss as a function of (M, F): P = softmax(M), f = sigmoid(F), Y = P^T (f o S_ext)
    -> (dL/dF, dL/dY_ext at the float64 Y_ext, P)."""
    torch = _torch()
    F = F0.clone().requires_grad_(True)
    P = torch.softmax(M0[:, :r.V], dim=1)
    f = torch.sigmoid(F)
    Y = (P.t() @ (r.Sx * f[:, None])).detach().requires_grad_(True)
    total, _ = _closs(r, P.t() @ (r.Sx * f[:, None]), f, M0)
    (gF,) = torch.autograd.grad(total, F)
    totY, _ = _closs(r, Y, f.detach(), M0)
    (dY,) = torch.autograd.grad(totY, Y)
    return gF, dY, P


def _check_filter_grad(r, M0, F0, f, rdot, fscal, dY_dev, c_rel, mode, extra=0.0):
    """dL/dF implied by the device's row-dot, f and fscal, g = r (1 - f) + (fscal0 + lc fscal1 + lf (1 - 2 f)) f (1 - f),
    against float64 autograd of the whole loss in (M, F).  The row-dot carries its mode's relative bound c_rel of
    sum_j P_ij |S_f||dY| (the operands P and S_f included) plus `extra` per row, and what the device's dY_ext differs from
    the float64 one (measured: sum_j P_ij |S_f,i| |dY_dev - dY_ref|_j, the forward's error carried through the loss
    stage); the bracket carries fscal[0]'s bound and 2 x 6 u of f.  f's own 6 u costs up to 6 u (|r| + |bracket| f)
    absolutely, where 1 - f cancels.  A dropped 1 / sum f, a wrong sign or a wrong power of f is O(1)."""
    torch = _torch()
    gref, dYref, P = _full_grad_F(r, M0, F0)
    Sf = r.Sx * f[:, None]
    lc, lf = r.lam_of("lambda_count"), r.lam_of("lambda_f_reg")
    c = fscal[0] + lc * fscal[1] + lf * (1 - 2 * f)
    w = f * (1 - f)
    g = rdot * (1 - f) + c * w
    rscale = (P * (Sf.abs() @ dY_dev.abs().t())).sum(dim=1)
    carry = (P * (Sf.abs() @ (dY_dev - dYref).abs().t())).sum(dim=1)
    cbound = ((r.V + r.N) / 1024 + 24) * U * abs(float(fscal[0])) + lf * 16 * U * f + 4 * U * c.abs()
    bound = (1 - f) * (c_rel * rscale + carry + extra) + w * cbound + 8 * U * (g.abs() + rdot.abs() + c.abs() * f)
    _check(f"{mode} dL/dF", g, gref, bound, 1.0, 1.0, 1.0)


def _check_filter_update(r, pre, rdot, f, fscal, t, mode):
    """F, mF, vF after the step = one torch.optim.Adam(foreach=False) step on CUDA from the device's pre-step state and
    step count, with g formed in fp32 from the device's rdot, f and fscal in k_filter_update's order: bit for bit.  Then the
    float64 Adam step from the float64 g (six roundings of g: 8 u of its terms)."""
    torch = _torch()
    F0, m0, v0 = pre
    g32 = _filter_grad32(r, rdot, f, fscal)
    Fw, mw, vw = _torch_adam_step(F0, m0, v0, g32, t)
    F1, m1, v1 = r.buf("F"), r.buf("mF"), r.buf("vF")
    for name, got, want in (("F", F1, Fw), ("mF", m1, mw), ("vF", v1, vw)):
        diff = got.float() != want
        assert not bool(diff.any()), (f"{mode}: {name} differs from torch's Adam in {int(diff.sum())} of {diff.numel()} "
                                      f"elements, first {torch.nonzero(diff)[0].tolist()}")
    lc, lf = r.lam_of("lambda_count"), r.lam_of("lambda_f_reg")
    c = fscal[0] + lc * fscal[1] + lf * (1 - 2 * f)
    g = rdot * (1 - f) + c * f * (1 - f)
    dg = 8 * U * (rdot.abs() * (1 - f) + (fscal[0].abs() + lc + lf * (1 + 2 * f)) * f * (1 - f))
    Fr, mr, vr, dF, dm, dv = _adam64(F0, m0, v0, g, dg, t + 1)
    for name, got, want, b in (("F", F1, Fr, dF), ("mF", m1, mr, dm), ("vF", v1, vr, dv)):
        bad = (got - want).abs() > b
        assert not bool(bad.any()), f"{mode} {name} vs float64 Adam: {int(bad.sum())} elements off"


def _pre(r):
    return (r.nv("M"), r.nv("m"), r.nv("v")), (r.buf("F"), r.buf("mF"), r.buf("vF"))


# ================================================================================================================== tests
SHAPES = {
    # id: (N, V, K, constructor keywords)
    "2047": (2047, 300, 70, dict(target=0.3)),                                  # one forward chain just under the 2048 cut
    "2049": (2049, 257, 130, dict(target=0.7, lam=dict(REF_DEFAULTS, lambda_r=1e-3))),   # two chains, ragged tiles; sum f < target
    "Ke2112": (1000, 100, 2100, dict(target=0.3)),                             # Ke = 2112 > 2048: the backward's single chain
    "V5": (300, 5, 60, dict(target=0.7, lam=dict(lambda_count=0.5, lambda_f_reg=2.0))),  # V < 8, no g2
    "nodensity": (1500, 200, 70, dict(target=0.3, density=False)),             # density mode none: KL NaN, fscal[0] = 0
}
X3_IDS = ["2047", "2049", "Ke2112", "V5", "nodensity"]
FP32_IDS = ["2049", "Ke2112", "V5", "nodensity"]


@pytest.mark.parametrize("sid", X3_IDS)
def test_constrained_bf16x3_stages(sid):
    """bf16x3: filter prepare, tail, forward from S_f, loss stage, dP = S_f dY^T and the row-dot, dL/dF, F's Adam step
    (torch bit for bit) and M's exact update, each from the device's own inputs, at step 1 and step 3."""
    torch = _torch()
    N, V, K, kw = SHAPES[sid]
    r = CRun("bf16x3", N, V, K, seed=N + V + K, **kw)
    for step in range(1, 4):
        pre, fpre = _pre(r)
        t = r.e.get_state()
        r.e.step_begin()
        r.e.step_end(LR)
        if step == 2:
            continue
        mode = f"c-x3[{step}]"
        f, Sf = r.buf("f"), r.buf("Sf", r.Ke)
        _check_filter_prepare(r, fpre[0], f, Sf, mode)
        _check_tail(r, r.buf("tail"), f, mode)
        stats = r.buf("stats", 4)
        P3 = r.nv("Pb")
        Pref = _check_row_pass(r, pre[0], P3, stats, f"{mode} row pass")
        Yd = r.buf("Y", r.Ke)
        _check_forward(r, Yd, Pref, *_x3_forward_consts(r), mode=mode, S=Sf)
        dY = r.buf("dY", r.Ke)
        fscal = r.buf("fscal")
        _check_closs_stage(r, Yd, dY, r.e.history()[-1], fscal, f, pre[0], mode)
        dpf = r.nv("dpf")
        dPref = Sf @ dY.t()
        scale = Sf.abs() @ dY.abs().t()
        ce, _, _ = _x3_contraction_consts(r.Ke)
        _check(f"{mode} dP = S_f dY^T", dpf[:, :V], dPref, scale, ce, X3_BWD_FRO, X3_BWD_BIAS)
        assert torch.count_nonzero(dpf[:, V:]) == 0, "pad columns of dP"
        rdot = r.buf("rdot")
        rref = (P3[:, :V] * dPref).sum(dim=1)
        rscale = (P3[:, :V] * scale).sum(dim=1)
        _check(f"{mode} row-dot", rdot, rref, rscale, ce + (V + 2) * 2 * U, 8 * U + V * U, 8 * U)
        c_rel = ce + (V + 2) * 2 * U + (V + 13 + 12) * U
        _check_filter_grad(r, pre[0], fpre[0], f, rdot, fscal, dY, c_rel, mode)
        _check_filter_update(r, fpre, rdot, f, fscal, t, mode)
        g = _grad_terms(r, pre[0][:, :V], P3[:, :V], dpf[:, :V] - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
        dg = 4 * U * (g.abs() + P3[:, :V] * (dpf[:, :V].abs() + rdot.abs()[:, None]))
        # the entropy term's (M - mx) - log z - h in fp32: on rows of small f it is most of g
        lse = (stats[:, 0] + stats[:, 2])[:, None]
        dg = dg + r.lam.get("lambda_r", 0.0) * P3[:, :V] * 8 * U * (pre[0][:, :V].abs() + lse.abs() + stats[:, 3:4].abs() + 1.0)
        _check_update(r, pre, (r.nv("M"), r.nv("m"), r.nv("v")), g, dg, t + 1, mode)


@pytest.mark.parametrize("sid", FP32_IDS)
def test_constrained_fp32_stages(sid):
    """fp32 (FFMA): the same stages; the row-dot and dP are recomputed in float64 from the device's S_f, P and dY_ext
    (EpiAdam never stores dP)."""
    N, V, K, kw = SHAPES[sid]
    r = CRun("fp32", N, V, K, seed=N + K, **kw)
    for step in range(1, 4):
        pre, fpre = _pre(r)
        t = r.e.get_state()
        r.e.step_begin()
        r.e.step_end(LR)
        if step == 2:
            continue
        mode = f"c-fp32[{step}]"
        f, Sf = r.buf("f"), r.buf("Sf", r.Ke)
        _check_filter_prepare(r, fpre[0], f, Sf, mode)
        _check_tail(r, r.buf("tail"), f, mode)
        stats = r.buf("stats", 4)
        Pf = r.nv("Pf")
        Pref = _check_row_pass(r, pre[0], Pf, stats, f"{mode} row pass")
        chain = -(-N // r.splits)
        Yd = r.buf("Y", r.Ke)
        _check_forward(r, Yd, Pref, (2 * chain + r.splits + V + 32) * U, 4 * np.sqrt(chain) * U + (r.splits + 16) * U, 20 * U,
                       mode, S=Sf)
        dY = r.buf("dY", r.Ke)
        fscal = r.buf("fscal")
        _check_closs_stage(r, Yd, dY, r.e.history()[-1], fscal, f, pre[0], mode)
        dPref = Sf @ dY.t()
        scale = Sf.abs() @ dY.abs().t()
        rdot = r.buf("rdot")
        rref = (Pf[:, :V] * dPref).sum(dim=1)
        rscale = (Pf[:, :V] * scale).sum(dim=1)
        c_r = (2 * (r.Ke + V) + 8) * U
        _check(f"{mode} row-dot", rdot, rref, rscale, c_r, 4 * np.sqrt(r.Ke + V) * U, 4 * U)
        _check_filter_grad(r, pre[0], fpre[0], f, rdot, fscal, dY, c_r + (V + 13 + 12) * U, mode)
        _check_filter_update(r, fpre, rdot, f, fscal, t, mode)
        g = _grad_terms(r, pre[0][:, :V], Pf[:, :V], dPref - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
        dg = Pf[:, :V] * (2 * r.Ke + 8) * U * scale + 8 * U * (g.abs() + Pf[:, :V] * (dPref.abs() + rdot.abs()[:, None] + 1.0))
        _check_update(r, pre, (r.nv("M"), r.nv("m"), r.nv("v")), g, dg, t + 1, mode)


BF16_SHAPES = {
    "2049": (2049, 257, 130, dict(target=0.3)),
    "9000": (9000, 300, 70, dict(target=0.7, lam=dict(REF_DEFAULTS, lambda_r=1e-3))),   # constrained: one cell chunk
    "V5-Ke2112": (1000, 5, 2100, dict(target=0.3, lam=dict(lambda_count=0.5, lambda_f_reg=2.0))),
    "nodensity": (1500, 200, 70, dict(target=0.7, density=False)),
}


@pytest.mark.parametrize("sid", list(BF16_SHAPES))
def test_constrained_bf16_stages(sid):
    """bf16: the filter stages, the forward from its operands P~ and bf16(S_f / z~) (the density column carries one bf16
    rounding of f_i / z~_i), the staged row-dot r = c + r' (exact) and against float64 from the bf16 operands of the
    store-only contraction, dL/dF, F's Adam step and M's streaming update (g from dq and rowc)."""
    torch = _torch()
    N, V, K, kw = BF16_SHAPES[sid]
    r = CRun("bf16", N, V, K, seed=N + V, **kw)
    assert r.nchunks == 1, "constrained mode runs the bf16 iteration as one cell chunk (the filter update couples all rows)"
    for step in range(1, 4):
        pre, fpre = _pre(r)
        t = r.e.get_state()
        c_pre = r.buf("rcenter")
        r.e.step_begin()
        lseT_now = r.buf("lseT")
        Pt = r.nv("Pb")[:, :V]
        izt = r.buf("inv_zt")
        r.e.step_end(LR)
        if step == 2:
            continue
        mode = f"c-bf16[{step}]"
        f, Sf = r.buf("f"), r.buf("Sf", r.Ke)
        _check_filter_prepare(r, fpre[0], f, Sf, mode)
        _check_tail(r, r.buf("tail"), f, mode)
        Ss = _bf16_round(Sf.float() * izt.float()[:, None])            # k_scale_rows_bf16 of S_f
        Yd = r.buf("Y", r.Ke)
        _check_forward(r, Yd, Pt, *_bf16_forward_consts(r), mode, S=Ss)
        dY = r.buf("dY", r.Ke)
        fscal = r.buf("fscal")
        _check_closs_stage(r, Yd, dY, r.e.history()[-1], fscal, f, pre[0], mode)
        # row-dot: r = c + r' with r' = (sum_j P~_ij dq_ij) / z~_i, dq = bf16(bf16(S_f) bf16(dY)^T - c)
        rdot, rowc = r.buf("rdot"), r.buf("rowc", 4)
        want = c_pre.float() + rowc[:, 1].float()
        assert torch.equal(rdot.float(), want), f"{mode}: rdot != c + r' in {int((rdot.float() != want).sum())} rows"
        assert torch.equal(r.buf("rcenter"), rdot), "the row-dot is the next centre"
        dPref = _bf16_round(Sf) @ dY.t()
        scale = _bf16_round(Sf).abs() @ dY.abs().t()
        ce = (4 + 2 * ((r.Ke + 15) // 16 + 16) + 1) * U
        dev = (dPref - c_pre[:, None]).abs()
        rref = c_pre + (Pt * (dPref - c_pre[:, None])).sum(dim=1) * izt
        rb = izt * (Pt * (ce * scale * (1 + UB) + (UB + (V + 4) * U) * dev)).sum(dim=1) + 2 * U * (c_pre.abs() + rdot.abs())
        _check(f"{mode} row-dot", rdot, rref, rb, 1.0, 1.0, 1.0)
        # dL/dF: the row-dot against sum_j P_ij (S_f dY^T)_ij carries the bf16 rounding of P~, of S_f and of dq (the last
        # one of dP - c: the centre c adds 2 u_b |c|)
        _check_filter_grad(r, pre[0], fpre[0], f, rdot, fscal, dY, 6 * UB, mode, extra=2 * UB * c_pre.abs())
        _check_filter_update(r, fpre, rdot, f, fscal, t, mode)
        dq = r.nv("dq")[:, :V]
        assert torch.equal(rowc[:, 0], lseT_now), "rowc carries the row's exact log-sum-exp"
        Mv = pre[0][:, :V]
        P = torch.exp(Mv - rowc[:, 0:1])
        g = _grad_terms(r, Mv, P, dq - rowc[:, 1:2], rowc[:, 0], rowc[:, 2])
        dg = (UM * (4 + 2 * Mv.abs() + 2 * rowc[:, 0:1].abs()) + 4 * U) * g.abs() + 4 * U * P * (dq.abs() + rowc[:, 1:2].abs())
        dg = dg + (r.lam.get("lambda_r", 0.0) * P * 8 * U * (Mv.abs() + rowc[:, 0:1].abs() + rowc[:, 2:3].abs()))
        _check_update_bf16(r, pre, (r.nv("M"), r.nv("m"), r.nv("v")), g, dg, t + 1, mode)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_filter_prepare_wide_logits(precision):
    """f = sigmoid(F) and S_f over logits from -87 (f ~ 1.6e-38, the last normal fp32 values) to 30 (f rounds to 1):
    within 6 u (_check_filter_prepare), S_f bit for bit.  An exp whose argument is rounded first (ex2 of F log2 e) is off
    by up to |F| u there."""
    N, V, K = 4000, 64, 40
    rng = np.random.default_rng(9)
    F0 = np.concatenate([np.linspace(-87.0, 30.0, N // 2), 3 * rng.standard_normal(N - N // 2)])
    r = CRun(precision, N, V, K, seed=9, F0=F0)
    F = r.buf("F")
    r.e.step_begin()
    _check_filter_prepare(r, F, r.buf("f"), r.buf("Sf", r.Ke), f"{precision} wide logits")
    r.e.step_end(LR)


SATURATED = [-np.inf, -100.0, -89.0, -80.0, 0.0, 100.0, np.inf]


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_saturated_filter_stays_finite(precision):
    """Filter logits at -inf, -100, -89 (f = 0 in fp32: expf(89) overflows), -80 (f ~ 2e-35), 0, 100 and +inf (f = 1)
    among normal draws, ten steps of run() (MapperConstrained.train): every buffer and history value stays finite, the
    cells whose f is exactly 0 or 1 keep F bit for bit with mF = vF = 0 (dL/dF = dL/df f (1 - f) = 0, as the reference's
    autograd gives), and the mapping and the other F track OracleMapperConstrained from the same M0 / F0 at
    test_constrained.py's tolerances."""
    from oracle.tangram_oracle import OracleMapperConstrained
    from tangram_b200 import MapperConstrained
    from tests.helpers import rel_fro
    N, V, K = 600, 150, 80
    inp = synthetic_inputs(N, V, K, seed=21)
    rng = np.random.default_rng(22)
    M0 = rng.standard_normal((N, V)).astype(np.float32)
    F0 = rng.standard_normal(N).astype(np.float32)
    planted = np.arange(0, 7 * 37, 37)
    F0[planted] = SATURATED
    o = OracleMapperConstrained(inp["S"], inp["G"], inp["d"], target_count=200, M0=M0, F0=F0)
    oo, oF, _ = o.train(10, print_each=None)
    m = MapperConstrained(inp["S"], inp["G"], inp["d"], target_count=200, device="cuda:0", precision=precision, M0=M0, F0=F0)
    out, F_out, hist = m.train(10, print_each=None)
    e = m._engine
    H = e.history()
    for col in (0, 1, 2, 3, 10, 11):
        assert np.isfinite(H[:, col]).all(), f"history column {col}: {H[:, col]}"
    for name in ("M", "m", "v", "F", "f", "mF", "vF", "Y", "rdot", "fscal", "tail", "Sf", "Sx"):
        x = e.debug(name)
        if name == "F":
            x = x[~np.isinf(F0)]
        assert np.isfinite(x).all(), f"{name}: {int((~np.isfinite(x)).sum())} non-finite values"
    assert np.isfinite(out).all() and np.isfinite(F_out).all()
    f = e.debug("f")
    sat = (f == 0) | (f == 1)
    assert set(planted[[0, 1, 2, 5, 6]]) <= set(np.nonzero(sat)[0]), "f of the planted saturated logits"
    F1 = e.debug("F")
    assert np.array_equal(F1[sat], F0[sat]), "F of a saturated cell moved"
    assert not e.debug("mF")[sat].any() and not e.debug("vF")[sat].any(), "Adam state of a saturated cell"
    live = ~sat
    if precision == "bf16":
        assert rel_fro(F_out, oF) < 2e-2 and rel_fro(out, oo) < 5e-2
    else:
        assert rel_fro(F1[live], o.F.numpy()[live]) < 1e-4 and rel_fro(out, oo) < 1e-4
        assert rel_fro(F_out, oF) < 1e-4


@pytest.mark.parametrize("precision,N,V,K", [("bf16", 9000, 300, 70), ("bf16x3", 2049, 257, 130)])
def test_constrained_run_matches_steps(precision, N, V, K):
    """MapperConstrained.train drives run(), the stage checks step_begin / step_end: three iterations of each leave
    every buffer and the history bit-identical in constrained mode."""
    a = CRun(precision, N, V, K, seed=N, lam=dict(REF_DEFAULTS, lambda_r=1e-3))
    b = CRun(precision, N, V, K, seed=N, lam=dict(REF_DEFAULTS, lambda_r=1e-3))
    a.e.run(3)
    for _ in range(3):
        b.e.step_begin()
        b.e.step_end(LR)
    names = ["Y", "M", "m", "v", "Pb", "rdot", "stats", "F", "f", "mF", "vF", "Sf", "fscal", "tail"]
    names += ["dq", "inv_zt", "lseA", "zsum", "rcenter", "rowc"] if precision == "bf16" else ["dpf"]
    for name in names:
        x, y = a.e.debug(name), b.e.debug(name)
        assert np.array_equal(x, y, equal_nan=True), f"{name}: run() and step_begin / step_end differ in {int((x != y).sum())} elements"
    assert np.array_equal(a.e.history(), b.e.history(), equal_nan=True), "history"


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_reset_adam_restarts_the_filter_optimizer(precision):
    """reset_adam zeroes mF and vF and restarts F's bias correction with M's: the next step is torch's Adam at t = 1 from
    a fresh state, so a second train() is a fresh optimizer over [M, F] (:607)."""
    torch = _torch()
    r = CRun(precision, 700, 130, 60, seed=3)
    r.e.run(3)
    assert r.e.get_state() == 3 and bool(r.buf("vF").abs().max() > 0)
    r.e.reset_adam()
    assert r.e.get_state() == 0
    for name in ("mF", "vF", "m", "v"):
        assert not bool(r.buf(name).any()), f"{name} after reset_adam"
    F0 = r.buf("F")
    c_pre = r.buf("rcenter") if precision == "bf16" else None
    r.e.step_begin()
    r.e.step_end(LR)
    f, rdot, fscal = r.buf("f"), r.buf("rdot"), r.buf("fscal")
    if c_pre is not None:
        assert torch.equal(rdot.float(), c_pre.float() + r.buf("rowc", 4)[:, 1].float())
    zero = torch.zeros_like(F0)
    _check_filter_update(r, (F0, zero, zero), rdot, f, fscal, 0, f"{precision} after reset_adam")


def test_get_filter_sigmoid_is_torch_sigmoid():
    """get_filter(sigmoid=...) (k_sigmoid, 1 / (1 + expf(-F))) against torch.sigmoid on CUDA over logits from -200 to 200,
    +-inf and normal draws: bit for bit (both are 1 / (1 + expf(-F)) in fp32 with IEEE expf)."""
    torch = _torch()
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    F = np.concatenate([np.linspace(-200, 200, 40001), [-np.inf, np.inf, -88.72, -88.73, -87.0, 17.0, 16.6],
                        np.random.default_rng(0).standard_normal(20000) * 5]).astype(np.float32)
    N, V, K = F.size, 8, 16
    e = Engine(N, V, K, precision="fp32", density_mode=_lib.DENSITY_NONE, constrained=True, target_count=1.0)
    e.set_filter(F)
    s = np.empty(N, dtype=np.float32)
    e.get_filter(sigmoid=s)
    want = torch.sigmoid(torch.from_numpy(F).cuda()).cpu().numpy()
    ulps = np.abs(s.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    print(f"[stage] get_filter sigmoid vs torch.sigmoid: {int((ulps > 0).sum())} of {N} differ, max {int(ulps.max())} ulp")
    assert np.array_equal(s, want), f"{int((ulps > 0).sum())} of {N} differ, max {int(ulps.max())} ulp"
