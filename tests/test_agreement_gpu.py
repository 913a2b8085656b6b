"""tgb200_agreement (mapping_parameter_tuning.agreement) on the H100 against a float64 evaluation of the tuner's three
metrics from their definitions: every run count R = 1..8, each with Pearson only and with both per-row entropies, at row
counts that make the warps stride over the grid, with large common offsets, a shift sample that misses the mean,
degenerate runs, ties, zeros, NaN and infinities, in every layout the entry point takes, and once at C3 (3 x 100k x 10k).

The reference (`_reference`) runs in float64 on the GPU, in chunks of rows, so that no float64 copy of a whole mapping is
made at C3.  The small cubes also check it against numpy itself.
  pearson    np.corrcoef of the flattened runs: two passes, cross products taken about the means, at
             np.tril_indices(R, -1).  With R = 1 there is no pair and the kernel returns an empty array; the reference's
             pearson_corr raises IndexError there (np.corrcoef of one row is a 0-d array).
  vote       np.argmax per run and row (a NaN beats every number, the first NaN wins, an all -inf row votes for column
             0), the votes counted exactly, the entropy of the shares c / R over log(cols).
  consensus  p = numpy's float32 mean over the runs (sequential fp32 adds, then / R: the array the reference hands
             scipy.stats.entropy, and the value the kernel forms), then scipy's entropy of p / sum(p) in float64, over
             log(cols).  With cols == 1 both entropies are 0 / log(1): NaN.

Bounds, u = 2^-53 (the fp64 unit roundoff):
  Pearson.  The kernel takes its sums about a shift c_r, the mean of 4096 evenly strided elements (recomputed here):
    S_rs = sum d_r d_s and T_r = sum d_r with d_r = x_r - c_r.  Every term passes through at most h additions: one lane's
    chain (ceil(rows / 8g) rows of at most ceil(cols / 32) + 5 elements), the warp butterfly (5), the eight warps of the
    block (8) and the g block partials, maximised over every grid g the entry point can pick (from min(rows / 8, #SM) to
    min(rows / 8, 8 #SM) blocks).  Forming d costs u and the product two of them, so
        |dS_rs| <= (h + 3) u sum|d_r d_s|,   |dT_r| <= (h + 2) u sum|d_r|.
    The numerator N_rs = S_rs - T_r T_s / n adds (|T_r| |dT_s| + |T_s| |dT_r| + |dT_r dT_s|) / n and its own four
    roundings, 4 u (sum|d_r d_s| + |T_r T_s| / n).  The reference's N_rs has at most h_ref = cols + 2048 + chunks
    additions on any path, so it is within (h_ref + 3) u sum|(x_r - m_r)(x_s - m_s)| plus n dm_r dm_s from its means.
    With e_rs the sum of both, the correlation N_rs / sqrt(N_rr N_ss) moves by at most
        1.02 (e_rs / sqrt(N_rr N_ss) + |rho| (e_rr / N_rr + e_ss / N_ss) / 2) + 10 u |rho|
    (first order, with e_rr / N_rr < 1 % asserted, and the roundings of the divisions and square roots).  On the offset
    cases this bound is broken by the unshifted one-pass sum(xy) - sum(x) sum(y) / n in float64 on the host.
  Vote.  The counts are exact: within one float32 ulp.
  Consensus.  logf is within 1 ulp and the fp32 product p logf(p) adds half of one: 2^-22 sum|p log p| / s / log(cols),
    plus (2 cols + 64) u (1 + |log s| + 2 sum|p log p| / s) / log(cols) for the fp64 sums on both sides, plus half a
    float32 ulp for the output.

Observed maxima over all cases, as fractions of each bound (H100 80GB HBM3, 700 W power limit): Pearson 0.012 (the bound
is a worst case linear in the chain lengths), vote 0.48, consensus 0.41.  The unshifted one-pass formula misses the
reference by 2e4 to 3e5 times the Pearson bound on the offset case.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from tangram_b200 import _lib
from tangram_b200 import mapping_parameter_tuning as mpt

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
SAMPLE = 4096           # elements per run behind the kernel's shift (kAgrSample)
CHUNK = 2048            # rows per chunk of the reference
NAN = float("nan")


def _argmax(x):
    """np.argmax along the rows of a float32 CUDA tensor: the first NaN if there is one, else the first maximum (the tie
    rule torch.argmax documents)."""
    nan = torch.isnan(x)
    return torch.where(nan.any(1), nan.float().argmax(1), torch.argmax(x, 1))


def _entr(x):
    """scipy.special.entr: -x log x, 0 at 0, -inf below 0, NaN at NaN."""
    lx = torch.log(torch.where(x > 0, x, torch.ones_like(x)))
    return torch.where(x > 0, -x * lx, torch.where(x == 0, torch.zeros_like(x),
                                                   torch.where(x < 0, torch.full_like(x, -math.inf), x)))


def _shift(runs):
    """The kernel's per-run shift: the float64 mean of min(n, 4096) elements at floor(n k / ns)."""
    N, V = runs[0].shape
    total = N * V
    ns = min(total, SAMPLE)
    k = torch.arange(ns, device=runs[0].device, dtype=torch.int64)
    e = total // ns * k + (total % ns) * k // ns
    return torch.stack([r[e // V, e % V] for r in runs]).double().mean(1)


def _kernel_depth(N, V):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_row = -(-V // 32) + 5
    need = -(-N // 8)
    return max(-(-N // (8 * g)) * per_row + g for g in range(min(need, sms), min(need, 8 * sms) + 1)) + 13


def _reference(runs):
    """float64 evaluation of the three metrics of R equally shaped float32 CUDA tensors, with the sums behind the bounds.
    -> dict of numpy arrays: pearson and pearson_bound (tril order), vote and vote_bound, cons and cons_bound (rows)."""
    R = len(runs)
    N, V = runs[0].shape
    n = N * V
    dev = runs[0].device
    f64 = dict(dtype=torch.float64, device=dev)
    c = _shift(runs)
    sum_x, sum_abs = torch.zeros(R, **f64), torch.zeros(R, **f64)
    for i0 in range(0, N, CHUNK):
        x = torch.stack([r[i0:i0 + CHUNK] for r in runs]).double()
        sum_x += x.sum(2).sum(1)
        sum_abs += x.abs().sum(2).sum(1)
    m = sum_x / n
    Nc, Ac, A = torch.zeros((R, R), **f64), torch.zeros((R, R), **f64), torch.zeros((R, R), **f64)
    B = torch.zeros(R, **f64)
    vote, cons, scale, logs = [], [], [], []
    for i0 in range(0, N, CHUNK):
        xf = torch.stack([r[i0:i0 + CHUNK] for r in runs])
        x = xf.double()
        y, d = x - m[:, None, None], x - c[:, None, None]
        ya, da = y.abs(), d.abs()
        B += da.sum(2).sum(1)
        for r in range(R):
            for s in range(r + 1):
                Nc[r, s] += (y[r] * y[s]).sum(1).sum()
                Ac[r, s] += (ya[r] * ya[s]).sum(1).sum()
                A[r, s] += (da[r] * da[s]).sum(1).sum()
        del x, y, d, ya, da
        votes = torch.stack([_argmax(xf[r]) for r in range(R)])
        count = (votes[:, None] == votes[None]).sum(1).double()          # count[r] = runs voting as run r does
        vote.append(-torch.log(count / R).mean(0) / math.log(V))
        p = xf[0].clone()
        for r in range(1, R):
            p += xf[r]
        p = (p / torch.full_like(p, R)).double()                   # a true division, as numpy's (not p * (1 / R))
        s = p.sum(1)
        cons.append(_entr(p / s[:, None]).sum(1) / math.log(V))
        plogp = torch.where(p > 0, p * torch.log(torch.where(p > 0, p, torch.ones_like(p))), torch.zeros_like(p))
        scale.append(plogp.abs().sum(1) / s.abs())
        logs.append(torch.log(s.abs()).abs())
    for M in (Nc, Ac, A):
        M.copy_(torch.tril(M) + torch.tril(M, -1).T)
    Nc, Ac, A, B, sum_abs = (t.cpu().numpy() for t in (Nc, Ac, A, B, sum_abs))
    T = np.abs((sum_x - n * c).cpu().numpy())
    out = {}

    # Pearson and its bound
    h, h_ref = _kernel_depth(N, V), V + min(N, CHUNK) + -(-N // CHUNK)
    T = T + (h_ref + 1) * U * sum_abs                          # |T_r|, with the reference's own error in it
    eT = (h + 2) * U * B
    e = ((h + 3) * U * A + (T[:, None] * eT[None] + eT[:, None] * T[None] + np.outer(eT, eT)) / n
         + 4 * U * (A + np.outer(T, T) / n))
    dm = (h_ref + 1) * U * sum_abs / n
    e += (h_ref + 3) * U * Ac + n * np.outer(dm, dm)
    ii, jj = np.tril_indices(R, -1)
    with np.errstate(divide="ignore", invalid="ignore"):
        dg = np.diag(Nc)
        rho = np.clip(Nc / np.sqrt(dg)[:, None] / np.sqrt(dg)[None], -1.0, 1.0)
        rel = np.diag(e) / dg
        assert np.all(rel[np.isfinite(rel)] < 0.01), "bound outside its first-order range"
        bound = 1.02 * (e / np.sqrt(np.outer(dg, dg)) + np.abs(rho) * (rel[:, None] + rel[None]) / 2) + 10 * U * np.abs(rho)
    out["pearson"], out["pearson_bound"] = rho[ii, jj], bound[ii, jj]

    # the per-row entropies and their bounds
    out["vote"] = torch.cat(vote).cpu().numpy()
    out["cons"] = torch.cat(cons).cpu().numpy()
    scale, logs = torch.cat(scale).cpu().numpy(), torch.cat(logs).cpu().numpy()
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        out["vote_bound"] = np.spacing(np.abs(out["vote"]).astype(np.float32)).astype(np.float64)
        b = (2.0 ** -22 * scale + (2 * V + 64) * U * (1 + logs + 2 * scale)) / math.log(V)
        out["cons_bound"] = b + 0.5 * np.spacing((np.abs(out["cons"]) + b).astype(np.float32)).astype(np.float64)
    return out


def _close(what, got, exp, bound):
    """NaN where exp is NaN, equal where exp is infinite, within bound elsewhere -> max err / bound."""
    got = np.asarray(got, dtype=np.float64)
    nan = np.isnan(exp)
    bad = np.flatnonzero(nan != np.isnan(got))
    assert bad.size == 0, f"{what}: NaN pattern differs at {bad[:8]}: got {got[bad[:8]]}, reference {exp[bad[:8]]}"
    inf = np.isinf(exp)
    assert np.array_equal(got[inf], exp[inf]), what
    fin = ~nan & ~inf
    err = np.abs(got - exp)[fin]
    b = bound[fin]
    worst = np.argsort(-(err - b))[:8]
    assert np.all(err <= b), (f"{what}: {int((err > b).sum())} of {err.size} beyond the bound, e.g. at "
                              f"{np.flatnonzero(fin)[worst]}: got {got[fin][worst]}, reference {exp[fin][worst]}")
    return float(np.max(err / np.where(b > 0, b, 1.0), initial=0.0))


def _check(what, got, ref, rows):
    p, v, c = got
    R2 = ref["pearson"].shape[0]
    assert p.shape == (R2,) and p.dtype == np.float64, what
    assert np.all(np.abs(p[~np.isnan(p)]) <= 1), what
    r = {"pearson": _close(what + " pearson", p, ref["pearson"], ref["pearson_bound"])}
    if rows:
        assert v.dtype == np.float32 and c.dtype == np.float32 and v.shape == c.shape == ref["vote"].shape, what
        r["vote"] = _close(what + " vote", v, ref["vote"], ref["vote_bound"])
        r["cons"] = _close(what + " consensus", c, ref["cons"], ref["cons_bound"])
    else:
        assert v is None and c is None
    print(f"{what}: max err / bound " + ", ".join(f"{k} {x:.3g}" for k, x in r.items()))
    return r


def _both(what, cube, ref):
    """k_agreement<R, false> and <R, true> on the same data."""
    for rows in (False, True):
        _check(f"{what} rows={rows}", mpt.agreement(cube, vote=rows, consensus=rows), ref, rows)


def _softmax_cube(R, N, V, seed, ld=None):
    """R correlated softmax mappings drawn on the device; ld pads every row with NaN, which must never be read."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn((N, V), device="cuda", generator=g) * 3
    buf = torch.full((R, N, ld or V), NAN, device="cuda")
    for r in range(R):
        buf[r, :, :V] = torch.softmax(base + torch.randn((N, V), device="cuda", generator=g), dim=1)
    return buf[:, :, :V]


def _check_reference_against_numpy(cube, ref):
    """The reference's Pearson and votes against np.corrcoef and np.argmax on the host (small cubes only)."""
    x = cube.cpu().numpy()
    R = x.shape[0]
    if R == 1:
        with pytest.raises(IndexError):
            np.corrcoef(x.reshape(1, -1).astype(np.float64))[np.tril_indices(1, -1)]
    else:
        with np.errstate(divide="ignore", invalid="ignore"):
            want = np.corrcoef(x.reshape(R, -1).astype(np.float64))[np.tril_indices(R, -1)]
        np.testing.assert_allclose(ref["pearson"], want, rtol=0, atol=1e-12)
    votes = x.argmax(axis=2)
    np.testing.assert_array_equal(torch.stack([_argmax(r) for r in cube.unbind(0)]).cpu().numpy(), votes)
    with np.errstate(divide="ignore", invalid="ignore"):
        vote = -np.log((votes[:, None] == votes[None]).sum(1) / R).mean(axis=0) / np.log(x.shape[2])
    np.testing.assert_allclose(ref["vote"], vote, rtol=1e-14, atol=0)


# (R, rows, cols, padded ld): every R, every row count and every column count at least once; 20011 rows are more than
# 8 warps x 132 SMs x 8 blocks, so warps stride over the grid at any occupancy.  A padded ld (a multiple of 4) takes the
# float4 body with a scalar tail; an unpadded cols that is not a multiple of 4 takes the scalar path.
SWEEP = [
    (1, 7, 5, False),
    (1, 20011, 4, False),
    (2, 1, 1001, True),
    (2, 8, 1, False),
    (3, 9, 3, False),
    (3, 20011, 5, True),
    (4, 20011, 128, False),
    (5, 7, 129, True),
    (6, 8, 127, True),
    (7, 9, 1001, False),
    (7, 1, 4100, False),
    (8, 20011, 4100, False),
]


@pytest.mark.parametrize("R,N,V,padded", SWEEP)
def test_every_run_count_against_float64(R, N, V, padded):
    cube = _softmax_cube(R, N, V, seed=R * 1000 + V, ld=(V + 3) // 4 * 4 + 4 if padded else None)
    ref = _reference(list(cube.unbind(0)))
    if R * N * V <= 1 << 24:
        _check_reference_against_numpy(cube, ref)
    _both(f"R={R} {N}x{V}{' padded' if padded else ''}", cube, ref)


def test_one_column_gives_nan_entropies():
    """log(1) = 0: the reference divides by it, so both entropies are NaN on every row; Pearson is unaffected."""
    g = torch.Generator(device="cuda").manual_seed(5)
    cube = torch.rand((3, 20011, 1), device="cuda", generator=g) + 0.1
    cube[:, :3] = 1.0
    ref = _reference(list(cube.unbind(0)))
    assert np.all(np.isnan(ref["vote"])) and np.all(np.isnan(ref["cons"]))
    _both("one column", cube, ref)


def _unshifted_pearson(x):
    """sum(xy) - sum(x) sum(y) / n in float64, without a shift: the one-pass formula the kernel's shift protects."""
    R, n = x.shape
    S = np.array([[np.dot(x[r], x[s]) for s in range(R)] for r in range(R)])
    T = x.sum(axis=1)
    Nu = S - np.outer(T, T) / n
    return (Nu / np.sqrt(np.diag(Nu))[:, None] / np.sqrt(np.diag(Nu))[None])[np.tril_indices(R, -1)]


@pytest.mark.parametrize("case", ["offsets", "decades"])
def test_pearson_with_large_common_offsets(case):
    """offsets: runs of offset_r + unit noise, offsets 1e3 .. 1e4, one run negatively correlated with the others.
    decades: gene-cube-like values from 1e-3 to 1e3 with run-to-run noise."""
    rng = np.random.default_rng(11)
    R, N, V = 4, 2000, 1000
    z = rng.standard_normal((N, V))
    if case == "offsets":
        off, a, b = [1e3, 2.5e3, 5e3, 1e4], [1.0, 0.8, -0.9, 0.3], [0.5, 1.0, 0.4, 1.0]
        x = np.stack([off[r] + a[r] * z + b[r] * rng.standard_normal((N, V)) for r in range(R)]).astype(np.float32)
    else:
        x = np.stack([10.0 ** (z * 1.0) * np.exp(0.3 * rng.standard_normal((N, V))) for r in range(R)]).astype(np.float32)
        assert x.min() < 1e-3 and x.max() > 1e3
    cube = torch.from_numpy(x).cuda()
    ref = _reference(list(cube.unbind(0)))
    _check_reference_against_numpy(cube, ref)
    _both(case, cube, ref)
    if case == "offsets":
        assert np.any(ref["pearson"] < -0.5) and np.any(ref["pearson"] > 0.5)
        # the bound is tight enough to see an unshifted one-pass formula
        miss = np.abs(_unshifted_pearson(x.reshape(R, -1).astype(np.float64)) - ref["pearson"]) / ref["pearson_bound"]
        print(f"unshifted one-pass: err / bound {miss.min():.3g} .. {miss.max():.3g}")
        assert np.all(miss > 1), miss


def test_pearson_when_the_shift_sample_misses_the_mean():
    """rows = cols = 4096: the shift samples exactly column 0 of every row.  Column 0 holds 1, the rest small positive
    values, so every shift is 1 while the means are below 1e-3."""
    N = V = 4096
    g = torch.Generator(device="cuda").manual_seed(3)
    base = torch.rand((N, V), device="cuda", generator=g) * 1e-3
    cube = torch.stack([base + torch.rand((N, V), device="cuda", generator=g) * 3e-4 * (r + 1) for r in range(3)])
    cube[:, :, 0] = 1.0
    runs = list(cube.unbind(0))
    c = _shift(runs)
    assert torch.all(c == 1.0)
    assert torch.all(torch.stack([r.double().mean() for r in runs]) < 2e-3)
    _both("shift far from the mean", cube, _reference(runs))


def test_degenerate_runs():
    """A constant run gives NaN for its pairs (0 / 0, as np.corrcoef); an identical run gives 1 and a negated one -1,
    within the bound and the clip."""
    x = _softmax_cube(1, 777, 129, seed=4)[0]
    cube = torch.stack([x, torch.full_like(x, 1.0 / 129), x, -x])
    ref = _reference(list(cube.unbind(0)))
    _check_reference_against_numpy(cube, ref)
    for rows in (False, True):
        p = mpt.agreement(cube, vote=rows, consensus=rows)[0]
        # tril order: (1,0) (2,0) (2,1) (3,0) (3,1) (3,2)
        assert np.all(np.isnan(p[[0, 2, 4]])), p
        want, b = np.array([1.0, -1.0, -1.0]), ref["pearson_bound"][[1, 3, 5]]
        assert np.all(np.abs(p[[1, 3, 5]] - want) <= b) and np.all(np.abs(p[[1, 3, 5]]) <= 1), (p, b)
    _both("degenerate runs", cube, ref)


# The special cube: R = 3, 40 rows of 1001 columns (a padded ld that is a multiple of 4 gives a float4 body of 1000
# columns and a scalar tail of one).  Run 0 holds the pattern; run 1 votes for the column np.argmax picks in run 0 and
# run 2 for column 600, so a wrong vote in run 0 changes the vote entropy.  Lanes of the float4 body: column c is in lane
# (c // 4) % 32; in the scalar path, lane c % 32.
V_SP, OTHER = 1001, 600
PATTERNS = [
    ("tie in one float4", {1: 0.9, 2: 0.9}, 1),
    ("tie in one lane, two iterations", {5: 0.9, 133: 0.9}, 5),
    ("tie across lanes", {9: 0.9, 6: 0.9}, 6),
    ("tie, the lower column in the higher lane", {300: 0.9, 200: 0.9}, 200),
    ("tie across the body / tail boundary", {996: 0.9, 1000: 0.9}, 996),
    ("tie of the tail with column 0", {0: 0.9, 1000: 0.9}, 0),
    ("NaN in column 0", {0: NAN, 500: 5.0}, 0),
    ("NaN in the body", {517: NAN, 3: 5.0}, 517),
    ("NaN in the tail", {1000: NAN, 2: 5.0}, 1000),
    ("two NaNs", {300: NAN, 200: NAN}, 200),
    ("two NaNs in one lane", {130: NAN, 2: NAN}, 2),
    ("NaN in the tail and the body", {1000: NAN, 999: NAN}, 999),
    ("+inf twice", {700: math.inf, 40: math.inf}, 40),
    ("+inf and NaN", {10: math.inf, 800: NAN}, 800),
    ("-inf entries beside a finite maximum", {7: -math.inf, 11: 0.9}, 11),
]
ALL_NEG_INF, ZERO_ROW, N_SP = len(PATTERNS), len(PATTERNS) + 1, 40


def _special_cube():
    rng = np.random.default_rng(8)
    x = rng.standard_normal((3, N_SP, V_SP)).astype(np.float32)
    x = np.exp(x - x.max(axis=2, keepdims=True))
    x /= x.sum(axis=2, keepdims=True) * 20                       # every value below 0.05
    for i, (_, pat, want) in enumerate(PATTERNS):
        for col, val in pat.items():
            x[0, i, col] = val
        x[1, i, want] = 0.5
        x[2, i, OTHER] = 0.5
    x[0, ALL_NEG_INF] = -np.inf
    x[1, ALL_NEG_INF, 0] = 0.5
    x[2, ALL_NEG_INF, OTHER] = 0.5
    x[:, ZERO_ROW] = 0.0
    for i, (what, _, want) in enumerate(PATTERNS):
        assert x[0, i].argmax() == want, what
    assert x[0, ALL_NEG_INF].argmax() == 0
    return x


def _raw(runs, ld, rows):
    """tgb200_agreement on raw per-run device pointers."""
    lib = _lib.load()
    R = len(runs)
    N, V = runs[0].shape
    p = np.empty(R * (R - 1) // 2)
    v, c = (np.empty(N, dtype=np.float32), np.empty(N, dtype=np.float32)) if rows else (None, None)
    dev = torch.cuda.current_device()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    ptrs = (_lib._P * R)(*[r.data_ptr() for r in runs])
    assert lib.tgb200_agreement(ptrs, R, N, V, ld, _lib.ptr(p), _lib.ptr(v), _lib.ptr(c), dev, stream) == 0
    return p, v, c


def _padded(x, ld):
    buf = torch.full((x.shape[0], x.shape[1], ld), NAN, device="cuda")
    buf[:, :, :x.shape[2]] = torch.from_numpy(x)
    return buf[:, :, :x.shape[2]]


@pytest.mark.parametrize("layout", ["contiguous", "ld multiple of 4", "ld not a multiple of 4", "misaligned base",
                                    "separate tensors"])
def test_ties_zeros_and_non_finite(layout):
    """np.argmax's order in every layout: ties go to the first column within a lane, across lanes and across the
    float4-body / scalar-tail boundary; a NaN beats every number and the first NaN wins; an all -inf row votes for
    column 0; +inf wins.  A row of zeros votes 0 with a NaN consensus; non-finite rows give NaN consensus.  Padding
    holds NaN and must never be read."""
    x = _special_cube()
    R, N, V = x.shape
    ref = _reference(list(torch.from_numpy(x).cuda().unbind(0)))
    if layout == "contiguous":
        cube = torch.from_numpy(x).cuda()
        _check_reference_against_numpy(cube, ref)
        assert ref["vote"][ZERO_ROW] == 0 and np.isnan(ref["cons"][ZERO_ROW])
    elif layout == "ld multiple of 4":
        cube = _padded(x, 1008)
    elif layout == "ld not a multiple of 4":
        cube = _padded(x, 1003)
    elif layout == "separate tensors":
        cube = [_padded(x[r:r + 1], 1004)[0] for r in range(R)]
    if layout != "misaligned base":
        _both(layout, cube, ref)
        return
    ld = 1008
    buf = torch.full((R, N * ld + 4), NAN, device="cuda")
    runs = [buf[r, 1:1 + N * ld].view(N, ld)[:, :V] for r in range(R)]
    for r in range(R):
        runs[r].copy_(torch.from_numpy(x[r]))
        assert runs[r].data_ptr() % 16 == 4
    for rows in (False, True):
        _check(f"{layout} rows={rows}", _raw(runs, ld, rows), ref, rows)


def test_c3_every_row_against_float64():
    """R = 3 mappings of 100k x 10k drawn on the device: Pearson and both entropies on every row against the float64
    reference, chunked by rows on the GPU."""
    N, V, R = 100_000, 10_000, 3
    g = torch.Generator(device="cuda").manual_seed(17)
    cube = torch.empty((R, N, V), device="cuda")
    for r in range(R):
        cube[r] = torch.softmax(torch.randn((N, V), device="cuda", generator=g) * 4, dim=1)
    ref = _reference(list(cube.unbind(0)))
    _both("C3", cube, ref)
    del cube
    torch.cuda.empty_cache()
