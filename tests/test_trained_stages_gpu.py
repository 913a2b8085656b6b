"""Each stage of the cells-mode iteration checked against float64 at trained mappings, and the gradient the update applies
checked against float64 autograd of the loss.

tests/test_stages_gpu.py checks every stage at steps 1 .. 4 from M ~ N(0, 1).  A real run trains 500 to 1,000 epochs, and
within a hundred most rows are peaked: one voxel leads by tens of units of M and the other P fall to 1e-20 .. 1e-45, into
fp32's subnormal range.  There the softmax Jacobian cancels on the dominant entry (g = P (dP_j - r) with r ~ dP_j), the
bf16 mode's MUFU ex2 / rcp / sqrt (.approx.ftz) return 0 where float64 keeps a subnormal, and Adam's v is subnormal on
the off-peak entries.  Here the states are

* the c1 fixture (5000 cells x 9852 voxels x 249 genes, tests/golden/c1_reference.npz) trained 600 epochs in bf16x3 from
  a seeded draw, with lambda_r = 1e-3 and without, saved with get_state, and
* planted rows written into a copy of it, near the first and last row of every cell chunk of the 1-, 2- and 4-chunk
  bf16 layouts (the last chunk is ragged): a two-way tie, margins 8, 30, 87.3 (off-peak P at 2^-126), 95 (subnormal P)
  and 110 (P below 2^-149), a constant row, and the trained row shifted by +1e3, -1e3 and +1e4, with the spike at
  column 0, at V - 1 and inside the ragged last 8-column group of the update,

loaded with set_state at t = 600 and t = 5000 in fp32, bf16x3 and bf16 with 1, 2 and 4 cell chunks.  Two step_begin /
step_end pairs follow each load: the fresh row pass (bf16: dq uncentred, c = 0), then (bf16) the carried normalisation
with the centre in place.  Every stage gets the bound of tests/test_stages_gpu.py with the late-step constants.

Underflow.  Every fp32 rounding whose result is subnormal is off by up to 2^-150 absolute instead of u relative (IEEE
gradual underflow), and an .ftz MUFU op returns 0 where the exact value is below 2^-126.  Those are the only floors added
(`tiny=True` of the shared helpers): the row pass's P gets 3 * 2^-149; Adam's m' and v' 4 * 2^-149, g 2^-149; in bf16
mode P~ (carry and update) 2^-126 times the factor it is multiplied with (inv_zt), g 2^-126 |dq - r'| (plus the entropy
factor), m's bf16 rounding 2^-134 (half of bf16's smallest subnormal).  Relative statistics are taken over the values
above 2^-126.

The gradient the update applies.  g_dev, in float64 from the device's own buffers (fp32: Pf (dP - rdot) with dP = S_ext
dY^T from the device's dY; bf16x3: the fp32 P, dpf, rdot; bf16: exp(M - lse) (dq - r')), plus the entropy term, against
g_ref = torch.autograd.grad of the loss as a function of M (softmax, Y = P^T S_ext, _loss_of_Y), all float64.  With
E_ij a bound on the error of the dP operand the row uses (contraction: c_bwd (|S| |dY|)_ij; bf16: both operands rounded
to bf16, 2 u_b (|S| |dY|)_ij, and dq's rounding u_b |dP_ij - c_i|; every mode: |S| dY's own error, the loss stage's
4 (V + K) u plus 4 (c_fwd + c_P) for Y's error, times each column's largest |dY|), c_P the row pass's (or the carry's)
relative error of P, c_r the row-dot's chain, and w the mismatch between the weights of the row-dot and the P of the
update (bf16: the bf16 rounding of P~, u_b; otherwise 8 u):

    |g_dev - g_ref|_ij <= c_P P_ij |dP_ij - r_i|                                    P's own error
                        + P_ij ((1 - P_ij) E_ij + sum_k P_ik E_ik - P_ij E_ij)      the operand error; the row-dot
                                                                                    cancels it on a dominant entry
                        + P_ij (4 u |dP_ij - c_i| + (c_r + w) sum_k P_ik |dP_ik - c_i|)
                        + the entropy term's and the underflow floors

where c_i is the centre the bf16 backward stored dq relative to (the previous step's row-dot) and 0 in fp32 / bf16x3.  On
a dominant entry of a peaked row the last line is the whole story: the centring makes it u_b |dP - c| instead of
u_b |dP|.  The bound is checked elementwise, rel-Fro and bias at 0.5 and 0.25 of it, for dominant (P >= 0.5) and other
entries separately.

Peaked states.  The statistical bias bounds of the FFMA chains (fp32 row-dot, forward) are the elementwise ones here: the
cells (voxels) that do not peak add terms below half an ulp of the running sum, which are dropped, all on one side
(observed 20 u on the row-dot and 60 u on the density column at the entropy state, against sqrt-class 4 u and 20 u).  For
the same reason the bf16 forward's elementwise bound takes two ulps per 16-product wgmma add (observed 1.34 of one ulp).

Observed maxima over both states, both step counts and 1, 2 and 4 chunks, as fractions of each bound (H100 80GB HBM3,
700 W power limit); [1] the fresh row pass, [2] the second step (bf16: the carry, dq centred):

    stage                              mode       elementwise   rel-Fro    bias
    row pass log z / 1 / z / P / h     fp32, x3   0.0039        0.11       0.039
    forward Y_ext genes / density      fp32       0.025         0.22       0.0041
                                       bf16x3     0.025         0.47       0.0052
                                       bf16       0.91          0.73       0.32
    loss stage dY_ext                  fp32, x3   0.015         1e-5       4e-5
                                       bf16       0.61          0.0066     0.003
    backward dP                        bf16x3     0.069         0.11       0.061
    backward dq                        bf16       1.0           0.87       0.12     (its own bf16 rounding)
    row-dot                            fp32       0.091         0.47       0.0097
                                       bf16x3     0.00089       7e-5       0.33
    carry lseT / P~ / h, z~            bf16       0.14          0.46       0.01
    update step (M, m, v: within)      all        -             0.23       0.011    (bf16x3: bit-exact torch Adam)
    gradient vs autograd, dominant     fp32       0.011         0.0014     0.0013
                                       bf16x3     0.00012       1e-4       5e-5
                                       bf16 [1]   0.47          0.066      0.027
                                       bf16 [2]   0.23          0.074      0.024
    gradient vs autograd, other        fp32, x3   0.054         4e-4       4e-5
                                       bf16       0.8           0.04       0.0016

On the 2,930 peaked rows (max P >= 0.99) of the entropy state the dominant entry's error is a median 1.1 % of |g| at the
uncentred first bf16 step after set_state and above |g| in 0.10 % of the rows; at the centred second step 0.27 % and
0.99 % (fp32: 0.043 % and 0.86 %, bf16x3: 0.001 % and none).  So the first step after a state load does not apply noise to
the peaks.  The centre lags dP_j* by a median 1.3 .. 1.6 % (one step's change of dY).  Learning rates 1 and 10 keep every
bf16 buffer finite and the carry within its bound (lseT 0.11, P~ 0.52 of rel-Fro): Adam moves an entry by at most a few
lr per step; at this V the carry stays within fp32's range up to lr ~ 25 (test_bf16_large_learning_rate_carry).

The centring check asks median |dP_j* - c| / |dP_j*| < 2^-5 on the peaked entropy state (observed 1.3 .. 1.6 %), not
2^-6: the centre is the previous step's row-dot, so it lags by one step's change of dY.  On the default state, whose only
peaked rows are planted into a mapping that still moves by about lr per step, 2^-3 (observed 6 .. 9 %).

m's bf16 rounding.  At the entropy state the stored m' has a signed mean error of +0.18 u_b against float64; round to
nearest of the kernel's own fp32 m' (emulated from g rounded to fp32) has the same mean to 3e-8 and every stored value
is that rounding within g's error bound.  The mean belongs to the values rounded (m' ~ b1 m with m on the bf16 grid
where g is small), not to the kernel, so _check_update_bf16 compares the two.

Planted errors, each built once into a copy of the library and run at bf16, one chunk, entropy, t = 600:
* the centre held at 0 (k_rowdot_finalize_staged writing center[i] = 0): fails "the centre is the previous iteration's
  row-dot", and the centring median reads 1.  With both of those assertions taken out the composed gradient bound still
  holds: the dominant-entry error grows from 0.0036 to 0.087 of it (share of peaked rows above |g|: 0.89 -> 2.4 %),
  because the bound's row-dot weight term is bf16's worst case u_b per entry, while on a peaked row P~ of the dominant
  entry rounds nearly exactly.
* the update's ragged 8-column group skipped: fails the update's v (and M) bound at column 9848 = V - 4, the first of
  the ragged group, on every row.
* lse rounded once more before ex2 in k_adam_rows (times 1 + 2^-23): fails the offset rows' P~ statistic at -1.52 u |lse|
  (bound 0.5; unmutated within 0.2 at every state and step).
"""
import os

import numpy as np
import pytest

from tests.test_stages_gpu import (B1, B2, EPS, LR, SUB, TINY, U, UB, UBS, UM, Run, _bf16_forward_consts, _bf16_round,
                                   _check, _check_backward_fp32, _check_bf16_update_step, _check_carry, _check_forward,
                                   _check_loss_stage, _check_row_pass, _check_update, _fp32_forward_consts, _g, _grad_terms,
                                   _loss_of_Y, _state, _torch, _x3_contraction_consts, _x3_forward_consts)

C1 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "c1_reference.npz")
TRAIN_EPOCHS = 600
FRO, BIAS = 0.5, 0.25
LAMS = {"default": {}, "entropy": {"lambda_r": 1e-3}}
MODES = [("fp32", 1), ("bf16x3", 1), ("bf16", 1), ("bf16", 2), ("bf16", 4)]
KINDS = ["tie", "m8", "m30", "m87.3", "m95", "m110", "const", "+1e3", "-1e3", "+1e4"]


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


gpu = [pytest.mark.gpu, pytest.mark.skipif(_no_gpu(), reason="needs an H100 GPU")]


# ---------------------------------------------------------------------------------------------------- float64 reference
def _ref_grad(r, M):
    """torch.autograd.grad of the loss as a function of M: softmax, Y_ext = P^T S_ext, _loss_of_Y (float64)"""
    torch = _torch()
    Mx = M[:, :r.V].clone().requires_grad_(True)
    Yx = torch.softmax(Mx, dim=1).t() @ r.S
    total, _ = _loss_of_Y(r, Yx, Mx)
    (g,) = torch.autograd.grad(total, Mx)
    return g


class _CpuRun:
    """what _loss_of_Y reads of a Run, on the CPU: cells mode, S_ext = [S, 1, 0] (genes, the density pair)"""

    def __init__(self, S, G, d, lam):
        torch = _torch()
        self.N, self.K = S.shape
        self.V, self.T, self.clusters, self.lam, self.graphs = G.shape[0], 0, False, dict(lam), {}
        self.S = torch.as_tensor(np.hstack([S, np.ones((self.N, 1)), np.zeros((self.N, 1))]), dtype=torch.float64)
        self.G = torch.as_tensor(G, dtype=torch.float64)
        self.d = torch.as_tensor(d, dtype=torch.float64)


@pytest.mark.parametrize("N,V,K", [(40, 30, 12), (130, 77, 25)])
@pytest.mark.parametrize("lam", list(LAMS), ids=list(LAMS))
def test_reference_gradient_is_the_oracle(N, V, K, lam):
    """The float64 autograd gradient the GPU checks below compare with equals OracleMapper(dtype=float64)'s closed-form
    loss_and_grad to 1e-12 (relative to its largest entry), so the reference is pinned to the oracle.  CPU only."""
    torch = _torch()
    from oracle.tangram_oracle import OracleMapper, synthetic_inputs
    inp = synthetic_inputs(N, V, K, seed=N + K)
    S, G, d = (np.asarray(inp[k], dtype=np.float32).astype(np.float64) for k in ("S", "G", "d"))
    M0 = np.random.default_rng(N).standard_normal((N, V)).astype(np.float32) * 4
    r = _CpuRun(S, G, d, LAMS[lam])
    o = OracleMapper(S=S, G=G, d=d, lambda_g1=1.0, lambda_d=1.0, M0=M0, dtype=torch.float64, **LAMS[lam])
    _, g_oracle = o.loss_and_grad()
    g = _ref_grad(r, torch.as_tensor(M0, dtype=torch.float64))
    err = float((g - g_oracle).abs().max() / g_oracle.abs().max())
    assert err <= 1e-12, f"autograd vs oracle: {err:.3g}"


# ------------------------------------------------------------------------------------------------------------- states
def _c1_data():
    import scipy.sparse as sp
    z = np.load(C1)
    S = sp.csr_matrix((z["S_data"], z["S_indices"], z["S_indptr"]), shape=tuple(z["S_shape"])).toarray().astype(np.float32)
    return S, np.ascontiguousarray(z["G"], dtype=np.float32), np.ascontiguousarray(z["d"], dtype=np.float32)


def _chunk_rows(N, nc):
    """the handle's cell chunks (tgb200_create: chunk c starts at round_up(c N / nc, 256))"""
    return [0] + [-(-(c * N // nc) // 256) * 256 for c in range(1, nc)] + [N]


def _plant(M, seed=11):
    """A copy of M with the planted rows near the first and last row of every chunk of the 1-, 2- and 4-chunk layouts
    -> (M, {row: kind})."""
    N, V = M.shape
    rng = np.random.default_rng(seed)
    M = M.copy()
    spikes = [0, V - 1, (V // 8) * 8 + (V % 8) // 2 if V % 8 else V - 5]
    rows = {}
    for nc in (1, 2, 4):
        b = _chunk_rows(N, nc)
        for c in range(nc):
            for k, kind in enumerate(KINDS):
                for i in (b[c] + k, b[c + 1] - 1 - k):
                    rows.setdefault(i, kind)
    for n, (i, kind) in enumerate(sorted(rows.items())):
        j = spikes[n % len(spikes)]
        if kind.startswith("m") or kind == "tie":
            margin = 30.0 if kind == "tie" else float(kind[1:])
            row = -margin - 3.0 * rng.random(V)
            row[j] = 0.0
            if kind == "tie":
                row[(j + V // 2) % V] = 0.0
        elif kind == "const":
            row = np.full(V, 0.37)
        else:
            row = M[i].astype(np.float64) + float(kind)
        M[i] = row.astype(np.float32)
    return M, rows


def _peakedness(what, M):
    torch = _torch()
    P = torch.softmax(_g(M), dim=1)
    q = torch.tensor([0.01, 0.1, 0.5, 0.9, 0.99], dtype=torch.float64, device=P.device)
    pmax = P.max(dim=1).values
    pmin = -torch.log10(torch.clamp(P.min(dim=1).values, min=1e-300))
    print(f"[state] {what}: quantiles 1/10/50/90/99 % of max_j P: {[round(float(x), 4) for x in torch.quantile(pmax, q)]}; "
          f"of -log10 min_j P: {[round(float(x), 1) for x in torch.quantile(pmin, q)]}")


@pytest.fixture(scope="module")
def c1_states():
    """{lam id: (planted M, m, v, {row: kind})}, the c1 fixture trained 600 bf16x3 epochs from a seeded draw"""
    from tangram_b200.engine import Engine
    S, G, d = _c1_data()
    N, K = S.shape
    V = G.shape[0]
    out = {}
    for lid, lam in LAMS.items():
        e = Engine(N, V, K, precision="bf16x3", lambda_d=1.0, **lam)
        e.set_expression(S, G)
        e.set_density(d)
        e.set_mapping(np.random.default_rng(42).standard_normal((N, V)).astype(np.float32))
        e.run(TRAIN_EPOCHS, LR)
        M, m, v = (np.empty((N, V), dtype=np.float32) for _ in range(3))
        assert e.get_state(M, m, v) == TRAIN_EPOCHS
        e.close()
        _peakedness(f"c1 {lid}, {TRAIN_EPOCHS} epochs", M)
        Mp, rows = _plant(M)
        _peakedness(f"c1 {lid}, planted", Mp)
        out[lid] = (Mp, m, v, rows)
    return out, (S, G, d)


class TrainedRun(Run):
    """Run on the c1 data from a saved state (M, m, v, t) instead of a seeded draw"""

    def __init__(self, precision, data, lam, state, t):
        from tangram_b200 import _lib
        from tangram_b200.engine import Engine
        S, G, d = data
        self.N, self.K = S.shape
        self.V, self.T, self.clusters, self.lam, self.precision, self.graphs = G.shape[0], 0, False, dict(lam), precision, {}
        self.e = Engine(self.N, self.V, self.K, precision=precision, lambda_d=1.0, density_mode=_lib.DENSITY_CELLS, **lam)
        self.e.set_expression(S, G)
        self.e.set_density(d)
        M, m, v = state
        self.e.set_state(M, m, v, t)
        self.Ke, self.ld, self.splits, self.rparts, self.nchunks = (int(x) for x in self.e.debug("shape"))
        self.S = _g(self.e.debug("Sx").reshape(self.N, self.Ke))
        self.G = _g(G)
        self.d = _g(d)


# ------------------------------------------------------------------------------------------------- the composed gradient
def _check_gradient(r, mode, M, g_dev, P, dPop, rdot_row, E, cP, c_r, w, centre, peaked, tiny_floor):
    """g_dev against autograd (module docstring): elementwise, rel-Fro and bias, dominant and other entries apart.
    dPop: the dP operand of the row (float64 of the device's values), rdot_row: sum_k P dPop, E: bound on dPop's error,
    centre: c_i (N), peaked: rows whose largest P >= 0.99.  Returns (g_ref, bound)."""
    torch = _torch()
    V = r.V
    g_ref = _ref_grad(r, M)
    Mv = M[:, :V]
    d = (dPop - centre[:, None]).abs()
    PE = (P * E).sum(dim=1, keepdim=True)
    bound = (cP * P * (dPop - rdot_row[:, None]).abs()
             + P * ((1 - P) * E + PE - P * E)
             + P * (4 * U * d + (c_r + w) * (P * d).sum(dim=1, keepdim=True))
             + tiny_floor)
    lam_r = r.lam.get("lambda_r", 0.0)
    if lam_r:
        lse = torch.logsumexp(Mv, dim=1, keepdim=True)
        # log P = M - lse and h: absolute errors of cP times the magnitudes they are formed from
        bound = bound + lam_r * P * (cP + 8 * U) * (1.0 + Mv.abs() + lse.abs() + (P * Mv.abs()).sum(dim=1, keepdim=True))
    dom = P >= 0.5
    for what, sel in (("dominant", dom), ("other", ~dom)):
        _check(f"{mode} gradient vs autograd, {what} entries", g_dev[sel], g_ref[sel], bound[sel], 1.0, FRO, BIAS)
    # the dominant entry of each peaked row, as a fraction of |g|
    if bool(peaked.any()):
        j = P.argmax(dim=1)
        rows = torch.nonzero(peaked & (g_ref.gather(1, j[:, None])[:, 0] != 0))[:, 0]
        err = (g_dev[rows, j[rows]] - g_ref[rows, j[rows]]).abs()
        gabs = g_ref[rows, j[rows]].abs()
        frac = err / torch.clamp(gabs, min=1e-300)
        above = float((frac > 1).double().mean())
        print(f"[stage] {mode} dominant entry of {rows.numel()} peaked rows: |err| / |g| median {float(frac.median()):.3g}, "
              f"above 1 in {above * 100:.3g} % of them")
        if rows.numel() >= 1000:        # a peaked state, not only the planted rows
            assert above <= 0.03, f"{mode}: the update applies noise to the peak of {above * 100:.3g} % of the peaked rows"
    return g_ref, bound


def _dY_err(r, dY, c_fwd, cPmax):
    """the bound on dY's error: the loss stage's 4 (V + K) u plus Y's error through the cosine's gradient (4 (c_fwd + c_P)),
    times each column's largest |dY|"""
    colmax = dY.abs().max(dim=0, keepdim=True).values
    return (4 * (r.V + r.K) * U + 4 * (c_fwd + cPmax) + UB * (r.precision == "bf16")) * colmax


# ------------------------------------------------------------------------------------------------------------ the tests
def _cases():
    out = []
    for prec, nc in MODES:
        for lid in LAMS:
            for t in (TRAIN_EPOCHS, 5000):
                out.append(pytest.param(prec, nc, lid, t, id=f"{prec}-{nc}chunk-{lid}-t{t}", marks=gpu))
    return out


@pytest.mark.parametrize("precision,chunks,lid,t", _cases())
def test_trained_stages(c1_states, monkeypatch, precision, chunks, lid, t):
    """Two iterations from a trained, planted state: every stage against float64 with the late-step constants, and the
    gradient the update applies against autograd."""
    torch = _torch()
    states, data = c1_states
    Mp, m, v, rows = states[lid]
    monkeypatch.setenv("TGB200_CHUNKS", str(chunks))
    r = TrainedRun(precision, data, LAMS[lid], (Mp, m, v), t)
    assert r.nchunks == chunks
    V = r.V
    for step in (1, 2):
        mode = f"{precision}/{chunks} {lid} t{t}[{step}]"
        pre = _state(r)
        t0 = r.e.get_state()
        assert t0 == t + step - 1
        Mv = pre[0][:, :V]
        Pref = torch.softmax(Mv, dim=1)
        peaked = Pref.max(dim=1).values >= 0.99
        if precision == "bf16":
            centre = r.buf("rcenter")
            if step == 1:
                assert torch.count_nonzero(centre) == 0, "set_state leaves the centre at 0"
            else:
                assert torch.equal(centre, prev_rdot), "the centre is the previous iteration's row-dot"
        r.e.step_begin()
        if precision == "bf16":
            if step == 1:
                stats = r.buf("stats", 4)
                assert torch.equal(stats[:, 0], Mv.max(dim=1).values), "row max"
                c = (UB + (V + 16 + (Mv - stats[:, 0:1]).abs()) * U) * Pref + UBS + 3 * SUB
                bad = (r.nv("Pb")[:, :V] - Pref).abs() > c
                assert not bool(bad.any()), f"{mode} row pass P: {int(bad.sum())} elements off"
                assert bool((r.buf("inv_zt") == 1).all()), "z~ = 1 on a fresh P"
            else:
                _check_carry(r, pre[0], f"{mode} carry", tiny=True)
            lseT_now = r.buf("lseT")
            Pt_fwd = r.nv("Pb")[:, :V]
            Ss = _bf16_round(r.S.float() * r.buf("inv_zt").float()[:, None])
        r.e.step_end(LR)
        Yd = r.buf("Y", r.Ke)
        dY = r.buf("dY", r.Ke)
        hist = r.e.history()[-1]
        if precision == "bf16":
            _check_forward(r, Yd, Pt_fwd, *_bf16_forward_consts_peaked(r), f"{mode}", S=Ss)
            del Pt_fwd, Ss
        else:
            stats = r.buf("stats", 4)
            Pdev = r.nv("Pf" if precision == "fp32" else "Pb")
            _check_row_pass(r, pre[0], Pdev, stats, f"{mode} row pass", floor=3 * SUB + (UBS if precision == "bf16x3" else 0.0))
            ce, cf, _ = _fp32_forward_consts(r) if precision == "fp32" else _x3_forward_consts(r)
            # peaked: the cells that do not peak on a voxel add terms below half an ulp of its running sum, dropped on one
            # side, so the bias is held to the elementwise bound
            _check_forward(r, Yd, Pref, ce, cf, ce, mode=mode)
        _check_loss_stage(r, Yd, dY, hist, pre[0], mode)
        lam_r = r.lam.get("lambda_r", 0.0)
        cPmax = (V + 16 + float((Mv - Mv.max(dim=1, keepdim=True).values).abs().max())) * U
        if precision == "fp32":
            _check_backward_fp32(r, pre, t0, stats, Pdev, dY, mode, late=True, tiny=True)
            P = Pdev[:, :V]
            dPop = r.S @ dY.t()
            rdot = r.buf("rdot")
            g_dev = _grad_terms(r, Mv, P, dPop - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
            # EpiAdam never stores dP: the operand here is S_ext dY^T from the device's dY, its fp32 chain is in the update's dg
            E = r.S.abs() @ _dY_err(r, dY, _fp32_forward_consts(r)[0], cPmax).t()
            cP, c_r, w = (V + 13 + (Mv - Mv.max(dim=1, keepdim=True).values).abs()) * U, (2 * (r.Ke + V) + 8) * U, 8 * U
            centre = torch.zeros_like(rdot)
            floor = SUB * (1 + lam_r)
        elif precision == "bf16x3":
            P, rdot, dPop = _check_backward_x3_trained(r, pre, t0, stats, dY, mode)
            g_dev = _grad_terms(r, Mv, P, dPop - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
            ce = _x3_contraction_consts(r.Ke)[0]
            E = ce * (r.S.abs() @ dY.abs().t()) + r.S.abs() @ _dY_err(r, dY, _x3_forward_consts(r)[0], cPmax).t()
            cP, c_r, w = (V + 13 + (Mv - Mv.max(dim=1, keepdim=True).values).abs()) * U, (V + 2) * 2 * U + ce, 8 * U
            centre = torch.zeros_like(rdot)
            floor = SUB * (1 + lam_r)
        else:
            _check_bf16_update_step(r, pre, t0, lseT_now, mode, late=True, tiny=True)
            dq = r.nv("dq")[:, :V]
            rowc = r.buf("rowc", 4)
            lse = rowc[:, 0]
            P = torch.exp(Mv - lse[:, None])
            g_dev = _grad_terms(r, Mv, P, dq - rowc[:, 1:2], lse, rowc[:, 2])
            _check_dq(r, dq, dY, centre, mode)
            _check_offset_rows(r, rows, lseT_now, mode)
            # the operand the kernel used is dq + its own centre; the bound is written with the centre it should have
            # used (0 after set_state, then the previous row-dot), so a centre that stays 0 fails it
            c_dev = centre
            dPop = dq + c_dev[:, None]
            centre = torch.zeros_like(c_dev) if step == 1 else prev_rdot
            Sb = _bf16_round(r.S)
            ce = _x3_contraction_consts(r.Ke)[0]
            prod = Sb.abs() @ dY.abs().t()
            E = (ce + 2 * UB) * prod + UB * (dPop - centre[:, None]).abs() + Sb.abs() @ _dY_err(r, dY, _bf16_forward_consts(r)[0], cPmax).t()
            del prod
            lse_abs = lse.abs()[:, None]
            cP = (V + 16) * U + UM * (3 + Mv.abs() + 2 * lse_abs)
            c_r = (64 + 2 + r.rparts + 1) * U
            w = UB + UM * (2 + Mv.abs().max(dim=1, keepdim=True).values + lse_abs)
            floor = TINY * ((dq - rowc[:, 1:2]).abs() + lam_r * ((Mv - lse[:, None]) - rowc[:, 2:3]).abs()) + SUB
            prev_rdot = r.buf("rdot")
            if step == 2:
                # centring: on the peaked rows the stored dq of the dominant entry is small against dP itself
                j = P.argmax(dim=1)
                rr = torch.nonzero(peaked)[:, 0]
                dPj = (r.S[rr] * dY[j[rr]]).sum(dim=1)
                ratio = ((dPj - c_dev[rr]).abs() / dPj.abs()).median()
                # the centre is the previous step's row-dot, so it lags dP_j* by one step's change of dY: 1.3 .. 1.6 % on
                # the peaked entropy state; the default state's only peaked rows are the planted ones, in a mapping that
                # still moves by about lr per entry and step (6 .. 9 %).  A centre held at 0 gives 1.
                lim = 2.0 ** -5 if lid == "entropy" else 2.0 ** -3
                print(f"[stage] {mode} centring: median |dP_j* - c| / |dP_j*| over {rr.numel()} peaked rows {float(ratio):.3g} "
                      f"(bound {lim:.3g})")
                assert float(ratio) < lim, f"{mode}: the centre does not track the dominant dP ({float(ratio):.3g})"
        rdot_row = (P * dPop).sum(dim=1)
        _check_gradient(r, mode, pre[0], g_dev, P, dPop, rdot_row, E, cP, c_r, w, centre, peaked, floor)
        del g_dev, E, P, dPop, Yd, dY, pre
        torch.cuda.empty_cache()
    r.e.close()


def _check_offset_rows(r, rows, lseA, mode):
    """The P~ the bf16 update wrote on the planted rows shifted by +-1e3 and +1e4, row by row.  The kernel forms
    exp(M' - lse) as ex2(fma(M', log2 e, -fl(lse log2 e))): the rounding of lse log2 e shifts a row's log P~ by at most
    u |lse| (one constant per row, of either sign), ex2's own error is ~2^-22 and bf16's rounding of P~ averages out over
    the row.  So s_i = mean_j (P~ - exp(M' - lse)) / exp(M' - lse) / (u |lse_i|) lies within [-1, 1] plus noise, and the
    mean of sign(lse_i) s_i over the ~24 offset rows is near 0 (their roundings have no common sign): held to 1/2.  An
    error of u |lse| on one side (one more rounding of lse) moves it by 1 or more."""
    torch = _torch()
    V = r.V
    idx = torch.as_tensor([i for i, k in sorted(rows.items()) if k in ("+1e3", "-1e3", "+1e4")], device="cuda")
    Mn = r.nv("M")[idx, :V]
    Pt = r.nv("Pb")[idx, :V]
    lse = lseA[idx]
    ref = torch.exp(Mn - lse[:, None])
    keep = ref >= 2.0 ** -100                # far from flush to zero and from bf16's subnormals
    rel = torch.where(keep, (Pt - ref) / ref, torch.zeros_like(ref))
    s = rel.sum(dim=1) / keep.sum(dim=1) / (U * lse.abs())
    stat = float((torch.sign(lse) * s).mean())
    print(f"[stage] {mode} P~ on {idx.numel()} offset rows: per-row mean error / (u |lse|) in [{float(s.min()):.3g}, "
          f"{float(s.max()):.3g}], signed mean {stat:.3g} (bound 0.5)")
    assert abs(stat) <= 0.5, f"{mode}: P~ on the offset rows is off by {stat:.3g} u |lse| on one side"


def _bf16_forward_consts_peaked(r):
    """_bf16_forward_consts with two ulps (4 u) per 16-product wgmma add elementwise instead of one: at a peaked state a
    voxel's running sum is set by the few cells that peak on it, and the tiny products of every other block of 16 cells
    are truncated against it (the two ulps _x3_contraction_consts's statistics already take); bias as elementwise"""
    ce, cf, _ = _bf16_forward_consts(r)
    parts = max(r.splits, r.nchunks)
    ce = ce + 2 * ((-(-r.N // parts) + 15) // 16) * U
    return ce, cf, ce


def _check_dq(r, dq, dY, centre, mode):
    """bf16 store-only backward: dq = bf16(bf16(S_ext) dY^T - c), the fp32 accumulation over Ke then one rounding"""
    Sb = _bf16_round(r.S)
    ref = Sb @ dY.t() - centre[:, None]
    chain = _x3_contraction_consts(r.Ke)[0] * (Sb.abs() @ dY.abs().t())
    _check(f"{mode} dq", dq, ref, UB * ref.abs() + chain * (1 + UB), 1.0, FRO, BIAS, floor=UBS)


def _check_backward_x3_trained(r, pre, t, stats, dY, mode):
    """bf16x3 backward at a trained state: dP, the row-dot from the three P planes, the update's bounds and the update bit
    for bit against torch.optim.Adam from the device's g.  The update recomputes P in fp32 (expf(M - mx) * 1 / z); below
    2^-100 the planes lose the low bits of a subnormal, so the bit comparison takes P from that fp32 recomputation
    (torch's expf on the device) and checks the planes against it only where P > 2^-100.  -> (P, rdot, dP)"""
    torch = _torch()
    V = r.V
    M0, m0, v0 = (x[:, :V].float().contiguous() for x in pre)
    st = stats.float()
    Pf = torch.exp(M0 - st[:, 0:1]) * st[:, 1:2]
    P3 = r.nv("Pb")[:, :V].float()
    big = Pf > 2.0 ** -100
    assert torch.equal(P3[big], Pf[big]), f"P planes vs fp32 P: {int((P3[big] != Pf[big]).sum())} elements differ"
    del P3
    dpf = r.nv("dpf")
    dPref = r.S @ dY.t()
    scale = r.S.abs() @ dY.abs().t()
    ce = _x3_contraction_consts(r.Ke)[0]
    _check(f"{mode} dP (Ke {r.Ke})", dpf[:, :V], dPref, scale, ce, 8 * U, 4 * U)
    assert torch.count_nonzero(dpf[:, V:]) == 0, "pad columns of dP"
    del dPref
    P = Pf.double()
    rdot = r.buf("rdot")
    pd = P * dpf[:, :V]
    _check(f"{mode} row-dot", rdot, pd.sum(dim=1), pd.abs().sum(dim=1), (V + 2) * 2 * U + ce + 4 * U, 4 * U * V, 4 * U)
    g = _grad_terms(r, pre[0][:, :V], P, dpf[:, :V] - rdot[:, None], stats[:, 0] + stats[:, 2], stats[:, 3])
    dg = 8 * U * (g.abs() + P * (dpf[:, :V].abs() + rdot.abs()[:, None] + 1.0)) + SUB
    post = _state(r)
    _check_update(r, pre, post, g, dg, t + 1, mode, late=True, tiny=True)
    if not r.lam:
        gf = (dpf[:, :V].float() - rdot.float()[:, None]) * Pf
        p = torch.nn.Parameter(M0.clone())
        opt = torch.optim.Adam([p], lr=LR, betas=(B1, B2), eps=EPS, foreach=False, fused=False)
        p.grad = gf
        opt.state[p] = {"step": torch.tensor(float(t)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
        opt.step()
        for name, got, want in (("v", post[2], opt.state[p]["exp_avg_sq"]), ("m", post[1], opt.state[p]["exp_avg"]),
                                ("M", post[0], p.detach())):
            diff = got[:, :V].float() != want
            assert not bool(diff.any()), f"{mode}: {name} differs from torch's Adam in {int(diff.sum())} of {diff.numel()} elements"
    return P, rdot, dpf[:, :V]


@pytest.mark.parametrize("lr", [1.0, 10.0])
@pytest.mark.gpu
@pytest.mark.skipif(_no_gpu(), reason="needs an H100 GPU")
def test_bf16_large_learning_rate_carry(c1_states, lr):
    """bf16 at the trained state with learning rates 1 and 10.  Adam moves an entry by at most lr (1 - b1) / sqrt(1 - b2)
    = 3.16 lr per step (a gradient after a long quiet stretch), so the carry P~ = exp(M_new - lseA) takes arguments up to
    3.16 lr, and its row sum z~ up to V exp(3.16 lr): within fp32's range (e^88.7) for lr < (88.7 - ln V) / 3.16, about
    25 at this V.  Nothing checks larger rates, at which the carry can overflow; at lr 1 and 10 three steps keep every
    buffer finite and the carry within _check_carry."""
    torch = _torch()
    states, data = c1_states
    Mp, m, v, _ = states["entropy"]
    r = TrainedRun("bf16", data, LAMS["entropy"], (Mp, m, v), TRAIN_EPOCHS)
    for step in range(3):
        pre = _state(r)
        r.e.step_begin()
        if step:
            _check_carry(r, pre[0], f"bf16 lr {lr}[{step + 1}] carry", tiny=True)
        r.e.step_end(lr)
        for name in ("M", "m", "v", "Pb", "dq"):
            assert bool(torch.isfinite(r.nv(name)).all()), f"lr {lr}: {name} not finite after step {step + 1}"
        for name in ("zsum", "lseA", "lseT", "inv_zt", "rcenter", "rdot"):
            assert bool(torch.isfinite(r.buf(name)).all()), f"lr {lr}: {name} not finite after step {step + 1}"
    r.e.close()
