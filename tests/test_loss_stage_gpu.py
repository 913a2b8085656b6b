"""The loss stage (k_loss_reduce, k_col_finalize, k_spatial_colstats, k_ct_islands, k_loss_scalars, k_dy_assemble) checked
on what it writes -- the history row and dY_ext -- against float64 autograd of the loss written from the reference
formulas as a function of the device's own Y_ext, in fp32, bf16x3 and bf16, where tests/test_stages_gpu.py does not reach:

* a training-gene mask (tgb200_set_loss_genes): every cosine term over Y[:, a], G[:, a] and their graph products,
  averaged over the Kact active genes; lambda_g2's row cosine over the active genes.  Inactive genes sit at 0, K - 1, the
  last gene of a float4 group and on both sides of the 128- and 512-column boundaries of the loss kernels; K = 1100 gives
  three 512-column reduction chunks;
* one active gene; masks switched between steps (stale per-voxel norms or coefficients would show);
* irregular graphs: a grid with ~2 % of its voxels cut loose (empty rows and columns in W, A and F) and a hub voxel with
  300 outgoing edges, with and without self-inclusion, passed as scipy CSR, as a dense ndarray and as a CSR with
  duplicate and unsorted entries (its reference is toarray());
* signed expression (as sc.pp.scale leaves it), with a per-gene offset that puts genes in all four sign cases of
  sign(colsum Y) x sign(colsum G): Getis-Ord is computed literally, cos((A Y) / colsum Y, (A G) / colsum G);
* V = 9001 (32 voxel rows per loss CTA, a ragged last row chunk) and V = 66000 (voxels past gridDim.y's 65535);
* 37 cell types (ct columns across a float4 boundary, not a multiple of 4), F with empty rows;
* the order of the set_* calls, which must not change a bit; malformed CSR graphs, which are refused.

Bounds, as in test_stages_gpu: every loss quantity is a handful of fp32 reductions over V voxels, K genes and, where a
sparse product enters, the longest row or column D_max of a graph, n = V + K + D_max:
    |term - ref| <= 4 n u max(1, |ref|)   (+ N for the terms summed over cells),
    |dY - ref|_jk <= 4 n u max_j |ref_jk|,   rel-Fro and bias <= 4 sqrt(n) u.
bf16 mode keeps dY_ext as one bf16 plane: one round to nearest more, u_b |ref| elementwise (half an ulp is up to 2^-8
relative), rel-Fro + u_b and bias + u_b / 16.  Exactly: dY is 0 on inactive gene columns and on the pad columns past
ct_off + T, and the history column of a term that is off is NaN.

bf16 runs drive step_begin / step_end; tgb200_run's prefetched forward leaves the same Y_ext bit for bit
(test_stages_gpu.test_bf16_run_prefetches_the_same_forward).

Observed maxima over steps 1 and 3 and every parameter set, as fractions of each bound (one H100, 80 GB); fp32 and
bf16x3 agree to two digits and share a row:

    case                          dY_ext fp32 / bf16x3          dY_ext bf16                   history
                                  elem     rel-Fro   bias       elem     rel-Fro   bias
    gene mask, all terms          0.0047   0.0093    0.018      0.95     0.47      0.011      0.0033
    one active gene               0.0066   0.051     0.015      0.90     0.21      0.18       0.0070
    mask switching                0.0066   0.012     0.014      0.96     0.36      0.032      0.0039
    irregular graphs              0.0037   0.0079    0.016      0.88     0.35      0.009      0.0026
    signed data                   0.0062   0.025     0.0015     0.93     0.20      0.0071     0.0003
    V = 9001                      0.0021   0.023     0.039      0.61     0.25      0.010      0.0034
    V = 66000                     0.0063   0.12      0.18       0.17     0.23      0.033      0.0072
    T = 37                        0.0048   0.0073    0.024      0.92     0.38      0.031      0.0025
    call order (step 3)           0.0038   0.0087    0.015      0.91     0.36      0.0072     0.0024
    after refused graphs          0.0088   0.010     0.023      -        -         -          0.0039

The bf16 elementwise figures sit near 1: there the bound is the round to nearest of dY itself, which is up to u_b |ref|.
"""
import numpy as np
import pytest

from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph, synthetic_inputs
from tests.test_constrained_stages_gpu import REF_DEFAULTS, CRun
from tests.test_stages_gpu import ALL_TERMS, LR, U, UB, _check, _g

pytestmark = pytest.mark.gpu
PRECISIONS = ["fp32", "bf16x3", "bf16"]
SPATIAL = dict(lambda_g2=0.5, lambda_neighborhood_g1=0.96, lambda_getis_ord=0.71)


def _torch():
    import torch
    return torch


# ------------------------------------------------------------------------------------------------------------- graphs
def _op64(mat, V):
    """The operator as the caller passed it -> float64 sparse tensor on the GPU (duplicates summed in float32, as
    toarray() sums them), and the longest row or column of what the device is given (duplicates counted)."""
    import scipy.sparse as sp
    torch = _torch()
    coo = sp.coo_matrix(mat, dtype=np.float32, copy=True)
    coo.sum_duplicates()
    idx = torch.as_tensor(np.vstack([coo.row, coo.col]).astype(np.int64), device="cuda")
    op = torch.sparse_coo_tensor(idx, torch.as_tensor(coo.data.astype(np.float64), device="cuda"), (V, V),
                                 check_invariants=True).coalesce()
    raw = sp.csr_matrix(mat)
    dmax = max(int(np.diff(raw.indptr).max()), int(np.bincount(raw.indices, minlength=V).max()))
    return op, dmax


def _grid_ops(V):
    conn, dist = grid_graph(V)
    return {0: spatial_weights_from_graph(conn, dist, True, True), 1: spatial_weights_from_graph(conn, dist, False, False),
            2: spatial_weights_from_graph(conn, dist, False, True)}


def _irregular_graph(V, seed, hub_degree=300):
    """grid_graph(V) with every edge of ~2 % of the voxels cut, plus one hub voxel with `hub_degree` outgoing edges only
    -> (connectivities, distances, cut voxels, hub)."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    conn, dist = grid_graph(V)
    c = conn.tocoo()
    rows, cols = c.row, c.col
    dv = np.asarray(dist.tocsr()[rows, cols]).ravel()
    cut = rng.choice(V, max(1, V // 50), replace=False)
    keep = ~(np.isin(rows, cut) | np.isin(cols, cut))
    rows, cols, dv = rows[keep], cols[keep], dv[keep]
    hub = int(rng.choice(np.setdiff1d(np.arange(V), cut)))
    taken = np.concatenate([cut, [hub], cols[rows == hub]])
    tgt = rng.choice(np.setdiff1d(np.arange(V), taken), hub_degree, replace=False)
    rows = np.concatenate([rows, np.full(hub_degree, hub)])
    cols = np.concatenate([cols, tgt])
    dv = np.concatenate([dv, rng.uniform(1.0, 4.0, hub_degree)])
    conn = sp.csr_matrix((np.ones_like(dv), (rows, cols)), shape=(V, V))
    dmat = sp.csr_matrix((dv, (rows, cols)), shape=(V, V))
    return conn, dmat, cut, hub


def _noncanonical(mat):
    """The same operator as a CSR with every third entry split into two duplicates (1/4 and 3/4 of it) and each row's
    entries in descending column order."""
    import scipy.sparse as sp
    c = sp.coo_matrix(mat)
    r, k, v = c.row, c.col, c.data.astype(np.float32)
    dup = np.arange(v.size) % 3 == 0
    r2 = np.concatenate([r, r[dup]])
    k2 = np.concatenate([k, k[dup]])
    v2 = np.concatenate([np.where(dup, v * np.float32(0.25), v), v[dup] * np.float32(0.75)]).astype(np.float32)
    order = np.lexsort((-k2, r2))
    V = mat.shape[0]
    indptr = np.concatenate([[0], np.cumsum(np.bincount(r2, minlength=V))]).astype(np.int32)
    out = sp.csr_matrix((v2[order], k2[order].astype(np.int32), indptr), shape=mat.shape)
    assert not out.has_sorted_indices and out.nnz > mat.nnz
    return out


def _irregular_ops(V, seed, self_inclusion, fmt):
    """W (standardised), F (binary, no self) and A (binary) of an irregular graph in the format the caller passes."""
    conn, dist, cut, hub = _irregular_graph(V, seed)
    ops = {0: spatial_weights_from_graph(conn, dist, True, self_inclusion),
           1: spatial_weights_from_graph(conn, dist, False, False),
           2: spatial_weights_from_graph(conn, dist, False, self_inclusion)}
    if fmt == "dense":
        ops = {w: m.toarray() for w, m in ops.items()}
    elif fmt == "noncanonical":
        ops = {w: _noncanonical(m) for w, m in ops.items()}
    return ops, cut, hub


# ---------------------------------------------------------------------------------------------------------------- runs
class LRun:
    """An Engine on given inputs, graphs (which -> operator in any form Engine.set_graph takes) and gene mask, plus the
    float64 copies the reference loss needs.  `order` lists the set_* calls in the order they are made."""

    DEFAULT_ORDER = ("expr", "density", "graphs", "ct", "mask")

    def __init__(self, precision, S, G, d, *, d_source=None, ct_encode=None, graphs=None, mask=None, lam=None, seed=0,
                 order=DEFAULT_ORDER, first_expression=None):
        from tangram_b200 import _lib
        from tangram_b200.engine import Engine
        torch = _torch()
        self.precision = precision
        self.N, self.K = S.shape
        self.V = G.shape[0]
        self.T = 0 if ct_encode is None else ct_encode.shape[1]
        self.lam = dict(lam or {})
        self.clusters = d_source is not None
        self.constrained = False
        self.e = Engine(self.N, self.V, self.K, n_types=self.T, precision=precision, lambda_d=1.0,
                        density_mode=_lib.DENSITY_SOURCE if self.clusters else _lib.DENSITY_CELLS, **self.lam)
        graphs = dict(graphs or {})
        self.ops, self.dmax = {}, 0
        for which, mat in graphs.items():             # before set_graph: Engine sorts a CSR's indices in place
            self.ops[which], dm = _op64(mat, self.V)
            self.dmax = max(self.dmax, dm)
        calls = {
            "expr": lambda: self.e.set_expression(S, G),
            "density": lambda: self.e.set_density(d, d_source),
            "graphs": lambda: [self.e.set_graph(w, m.copy()) for w, m in graphs.items()],
            "ct": lambda: self.e.set_ct_encode(ct_encode) if ct_encode is not None else None,
            "mask": lambda: self.e.set_loss_genes(mask) if mask is not None else None,
        }
        if first_expression is not None:
            self.e.set_expression(*first_expression)
        for c in order:
            calls[c]()
        self.e.set_mapping(np.random.default_rng(seed + 1).standard_normal((self.N, self.V)).astype(np.float32))
        self.Ke = int(self.e.debug("shape")[0])
        self.ld = int(self.e.debug("shape")[1])
        self.G = _g(G)
        self.d = _g(d)
        self.act = None if mask is None else torch.as_tensor(np.asarray(mask, dtype=bool), device="cuda")

    def set_mask(self, mask):
        self.e.set_loss_genes(mask)
        self.act = None if mask is None else _torch().as_tensor(np.asarray(mask, dtype=bool), device="cuda")

    def buf(self, name, cols=None):
        x = self.e.debug(name)
        return _g(x.reshape(-1, cols) if cols else x)

    def nv(self, name):
        return self.buf(name, self.ld)


def _crun(precision, N, V, K, seed, mask):
    """A constrained-mode CRun (MapperConstrained's defaults) with a gene mask, dressed with what _ref_loss reads."""
    r = CRun(precision, N, V, K, seed=seed, lam=REF_DEFAULTS, target=0.3)
    r.e.set_loss_genes(mask)
    r.act = _torch().as_tensor(np.asarray(mask, dtype=bool), device="cuda")
    r.ops, r.dmax, r.clusters, r.constrained = {}, 0, False, True
    return r


# ------------------------------------------------------------------------------------------------- the float64 loss
def _cos_cols(a, b):
    torch = _torch()
    na = torch.clamp(torch.linalg.vector_norm(a, dim=0), min=1e-8)
    nb = torch.clamp(torch.linalg.vector_norm(b, dim=0), min=1e-8)
    return (a * b).sum(dim=0) / (na * nb)


def _ref_loss(r, Yx, M, f=None):
    """The loss (mapping_optimizer.py's formulas) as a function of Y_ext, float64 and autograd-able; with a gene mask
    every gene term runs on Y[:, a] and G[:, a].  Constrained mode: dhat = colsum / sum f, the count and f-reg terms.
    -> (total, {history column: value})."""
    torch = _torch()
    K, T, N, V = r.K, r.T, r.N, r.V
    lam = {k: float(np.float32(v)) for k, v in r.lam.items()}
    Y, G = Yx[:, :K], r.G
    if r.act is not None:
        Y, G = Y[:, r.act], G[:, r.act]
    mm = torch.sparse.mm
    terms = {1: _cos_cols(Y, G).mean()}
    total = -terms[1]
    if lam.get("lambda_g2"):
        terms[2] = _cos_cols(Y.t(), G.t()).mean()
        total = total - lam["lambda_g2"] * terms[2]
    dens = Yx[:, K] + Yx[:, K + 1]
    dhat = dens / f.sum() if f is not None else (dens if r.clusters else dens / N)
    terms[3] = (torch.special.xlogy(r.d, r.d) - r.d * torch.log(dhat)).sum()
    total = total + terms[3]
    Mv = M[:, :V]
    if lam.get("lambda_r"):
        terms[4] = -(torch.softmax(Mv, 1) * torch.log_softmax(Mv, 1)).sum()
        total = total + lam["lambda_r"] * terms[4]
    if lam.get("lambda_l1"):
        terms[5] = Mv.abs().sum()
        total = total + lam["lambda_l1"] * terms[5]
    if lam.get("lambda_l2"):
        terms[6] = (Mv * Mv).sum()
        total = total + lam["lambda_l2"] * terms[6]
    if lam.get("lambda_neighborhood_g1"):
        W = r.ops[0]
        terms[7] = _cos_cols(mm(W, Y), mm(W, G)).mean()
        total = total - lam["lambda_neighborhood_g1"] * terms[7]
    if lam.get("lambda_ct_islands"):
        C = Yx[:, K + 2:K + 2 + T]
        terms[8] = torch.clamp(C - mm(r.ops[1], C), min=0).mean()
        total = total + lam["lambda_ct_islands"] * terms[8]
    if lam.get("lambda_getis_ord"):
        A = r.ops[2]
        terms[9] = _cos_cols(mm(A, Y) / Y.sum(dim=0), mm(A, G) / G.sum(dim=0)).mean()
        total = total - lam["lambda_getis_ord"] * terms[9]
    if f is not None:
        terms[10] = (f.sum() - r.target).abs()
        terms[11] = (f - f * f).sum()
        total = total + lam.get("lambda_count", 0.0) * terms[10] + lam.get("lambda_f_reg", 0.0) * terms[11]
    terms[0] = total
    return total, terms


def _check_loss(r, M, mode, f=None):
    """History row and dY_ext of the last step against autograd of _ref_loss at the device's Y_ext; the exact zeros and
    NaNs.  M: the mapping logits before the step (entropy, L1, L2); f: sigmoid(F) of the step (constrained mode)."""
    torch = _torch()
    K, T, V = r.K, r.T, r.V
    Y_dev, dY_dev = r.buf("Y", r.Ke), r.buf("dY", r.Ke)
    hist = r.e.history()[-1]
    Yx = Y_dev.clone().requires_grad_(True)
    total, terms = _ref_loss(r, Yx, M, f)
    (dref,) = torch.autograd.grad(total, Yx)
    n = V + K + r.dmax
    summed = {0, 4, 5, 6} | ({3, 10, 11} if f is not None else set())
    fs = float(f.sum()) if f is not None else 0.0
    worst = 0.0
    for col, val in sorted(terms.items()):
        got, want = float(hist[col]), float(val.detach())
        tol = 4 * (n + (r.N if col in summed else 0)) * U * max(1.0, abs(want), fs if col in (0, 10, 11) else 0.0)
        worst = max(worst, abs(got - want) / tol)
        assert abs(got - want) <= tol, f"{mode} history column {col}: {got} vs {want} (bound {tol:.3g})"
    print(f"[stage] {mode} history: max err/bound {worst:.3g} over columns {sorted(terms)}")
    for col in range(1, 12):
        if col not in terms:
            assert np.isnan(hist[col]), f"{mode} history column {col} of a term that is off: {hist[col]}"
    colmax = dref.abs().max(dim=0, keepdim=True).values.expand_as(dref)
    if r.precision == "bf16":
        _check(f"{mode} dY_ext (bf16)", dY_dev, dref, colmax, 4 * n * U * (1 + UB), 4 * np.sqrt(n) * U + UB,
               4 * np.sqrt(n) * U + UB / 16, floor=UB * dref.abs())
    else:
        _check(f"{mode} dY_ext", dY_dev, dref, colmax, 4 * n * U, 4 * np.sqrt(n) * U, 4 * np.sqrt(n) * U)
    if r.act is not None:
        off = torch.nonzero(~r.act).ravel()
        assert torch.count_nonzero(dY_dev[:, off]) == 0, f"{mode}: dY on inactive gene columns"
        assert torch.count_nonzero(dY_dev[:, torch.nonzero(r.act).ravel()]) > 0
    assert torch.count_nonzero(dY_dev[:, K + 2 + T:]) == 0, f"{mode}: dY past ct_off + T"
    return terms


def _run_and_check(r, mode, steps=(1, 3), f=False):
    for step in range(1, max(steps) + 1):
        M = r.nv("M")
        r.e.step_begin()
        r.e.step_end(LR)
        if step in steps:
            _check_loss(r, M, f"{mode}[{step}]", f=r.buf("f") if f else None)


def _inactive(K, rng):
    """Inactive genes at 0, K - 1, the last gene of a float4 group, both sides of the 128- and 512-column boundaries,
    and ~10 % of the rest."""
    off = {0, 3, K - 1} | {b + s for b in (128, 512, 1024) if b < K - 1 for s in (-1, 0)}
    off |= set(rng.choice(K, max(1, K // 10), replace=False).tolist())
    a = np.ones(K, dtype=bool)
    a[sorted(off)] = False
    return a


# ================================================================================================================ tests
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("K", [130, 1100])
@pytest.mark.parametrize("clusters", [False, True], ids=["cells", "clusters"])
def test_mask_all_terms(precision, K, clusters, monkeypatch):
    """A gene mask with every loss term on and T = 8; bf16 with two cell chunks."""
    if precision == "bf16":
        monkeypatch.setenv("TGB200_CHUNKS", "2")
    N, V, T = 2100, 700, 8
    inp = synthetic_inputs(N, V, K, seed=K + clusters, n_types=T, clusters=clusters)
    a = _inactive(K, np.random.default_rng(K))
    r = LRun(precision, inp["S"], inp["G"], inp["d"], d_source=inp.get("d_source"), ct_encode=inp["ct_encode"],
             graphs=_grid_ops(V), mask=a, lam=ALL_TERMS, seed=K)
    _run_and_check(r, f"mask K{K} {'clusters' if clusters else 'cells'} {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mask_constrained(precision):
    """Constrained mode (MapperConstrained's defaults: lambda_g2, count, f-reg) under a gene mask."""
    N, V, K = 2049, 257, 130
    r = _crun(precision, N, V, K, seed=11, mask=_inactive(K, np.random.default_rng(5)))
    _run_and_check(r, f"mask constrained {precision}", f=True)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_single_active_gene(precision):
    """Kact = 1 with lambda_g2 on: the 1 / Kact divisor and the per-voxel norms of G over one gene."""
    N, V, K, T = 1500, 300, 130, 8
    inp = synthetic_inputs(N, V, K, seed=3, n_types=T)
    a = np.zeros(K, dtype=bool)
    a[77] = True
    r = LRun(precision, inp["S"], inp["G"], inp["d"], ct_encode=inp["ct_encode"], graphs=_grid_ops(V), mask=a,
             lam=ALL_TERMS, seed=3)
    _run_and_check(r, f"one gene {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mask_switching(precision):
    """Mask A, step, mask B, step, no mask, step: each step against the mask in force."""
    N, V, K, T = 1500, 300, 130, 8
    inp = synthetic_inputs(N, V, K, seed=4, n_types=T)
    rng = np.random.default_rng(4)
    a = _inactive(K, rng)
    b = np.ones(K, dtype=bool)
    b[rng.choice(K, K // 2, replace=False)] = False
    r = LRun(precision, inp["S"], inp["G"], inp["d"], ct_encode=inp["ct_encode"], graphs=_grid_ops(V), mask=a,
             lam=ALL_TERMS, seed=4)
    for i, mask in enumerate((a, b, None)):
        if i:
            r.set_mask(mask)
        M = r.nv("M")
        r.e.step_begin()
        r.e.step_end(LR)
        _check_loss(r, M, f"switch {('A', 'B', 'none')[i]} {precision}")


IRREGULAR = [(True, "csr"), (False, "csr"), (False, "dense"), (False, "noncanonical")]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("self_inclusion,fmt", IRREGULAR, ids=["csr-self", "csr", "dense", "noncanonical"])
def test_irregular_graphs(precision, self_inclusion, fmt):
    """Isolated voxels (empty rows and columns) and a 300-edge hub row, every spatial term on."""
    N, V, K, T = 1500, 700, 130, 8
    inp = synthetic_inputs(N, V, K, seed=6, n_types=T)
    ops, cut, hub = _irregular_ops(V, 6, self_inclusion, fmt)
    r = LRun(precision, inp["S"], inp["G"], inp["d"], ct_encode=inp["ct_encode"], graphs=ops, lam=ALL_TERMS, seed=6)
    rows = (r.ops[0].to_dense() != 0).sum(dim=1)
    assert int(rows[hub]) >= 300 and r.dmax >= 300
    if not self_inclusion:
        for w in (0, 2):
            dense = r.ops[w].to_dense() != 0
            assert not bool(dense[cut].any()) and not bool(dense[:, cut].any()), "cut voxels have no edges"
    assert not bool((r.ops[1].to_dense() != 0)[cut].any())
    _run_and_check(r, f"irregular {fmt}{' +I' if self_inclusion else ''} {precision}")


def _signed_inputs(N, V, K, seed):
    """Expression as sc.pp.scale leaves it (per-gene zero mean, unit variance, both signs) plus a per-gene offset that
    puts the genes in the four cases of sign(colsum S) x sign(colsum G); a positive density with exact zeros."""
    rng = np.random.default_rng(seed)

    def scaled(n):
        X = np.log1p(rng.poisson(0.8, (n, K))).astype(np.float64)
        return (X - X.mean(axis=0)) / np.maximum(X.std(axis=0), 1e-3)

    case = np.arange(K) % 4
    sS, sG = np.where(case & 1, -1.0, 1.0), np.where(case & 2, -1.0, 1.0)
    S = (scaled(N) + sS * rng.uniform(0.05, 0.3, K)).astype(np.float32)
    G = (scaled(V) + sG * rng.uniform(0.05, 0.3, K)).astype(np.float32)
    for X, s in ((S, sS), (G, sG)):
        X64 = X.astype(np.float64)
        cs = X64.sum(axis=0)
        assert (np.abs(cs) >= 1e-3 * np.abs(X64).sum(axis=0)).all(), "a column sum near rounding level"
        assert (np.sign(cs) == s).all()
    d = rng.random(V)
    d[rng.random(V) < 0.1] = 0.0
    d = (d / d.sum()).astype(np.float32)
    assert (d == 0).any()
    return S, G, d, sS, sG


@pytest.mark.parametrize("precision", PRECISIONS)
def test_signed_data(precision):
    """Signed S and G: all four sign cases of the Getis-Ord shortcut sgn = sign(colsum Y) sign(colsum G)."""
    N, V, K = 1500, 500, 130
    S, G, d, sS, sG = _signed_inputs(N, V, K, seed=8)
    conn, dist, _, _ = _irregular_graph(V, 8)
    ops = {0: spatial_weights_from_graph(conn, dist, True, True), 2: spatial_weights_from_graph(conn, dist, False, True)}
    r = LRun(precision, S, G, d, graphs=ops, lam=SPATIAL, seed=8)
    for step in range(1, 4):
        M = r.nv("M")
        r.e.step_begin()
        r.e.step_end(LR)
        if step in (1, 3):
            ys = r.buf("Y", r.Ke)[:, :K].sum(dim=0).cpu().numpy()
            # rows of P sum to 1: colsum Y = colsum S, whatever the mapping
            assert (np.sign(ys) == sS).all() and (np.abs(ys) > 1e-3 * np.abs(S).sum(axis=0)).all()
            assert {(a, b) for a, b in zip(np.sign(ys), sG)} == {(1, 1), (1, -1), (-1, 1), (-1, -1)}
            _check_loss(r, M, f"signed {precision}[{step}]")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_scale_v9001(precision):
    """V = 9001: 32 voxel rows per loss CTA and a last row chunk of 9; every term on."""
    N, V, K, T = 600, 9001, 70, 8
    inp = synthetic_inputs(N, V, K, seed=9, n_types=T)
    r = LRun(precision, inp["S"], inp["G"], inp["d"], ct_encode=inp["ct_encode"], graphs=_grid_ops(V), lam=ALL_TERMS,
             seed=9)
    _run_and_check(r, f"V9001 {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_scale_v66000(precision):
    """V = 66000 > 65535: voxels on gridDim.x; neighbourhood, Getis-Ord and lambda_g2."""
    N, V, K = 64, 66000, 70
    inp = synthetic_inputs(N, V, K, seed=10)
    ops = _grid_ops(V)
    r = LRun(precision, inp["S"], inp["G"], inp["d"], graphs={0: ops[0], 2: ops[2]}, lam=SPATIAL, seed=10)
    _run_and_check(r, f"V66000 {precision}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_cell_types_37(precision):
    """T = 37 (ct columns K + 2 .. K + 38: across a float4 boundary, not a multiple of 4) and F with empty rows."""
    N, V, K, T = 1500, 700, 130, 37
    inp = synthetic_inputs(N, V, K, seed=12, n_types=T)
    ops, cut, _ = _irregular_ops(V, 12, False, "csr")
    r = LRun(precision, inp["S"], inp["G"], inp["d"], ct_encode=inp["ct_encode"], graphs=ops,
             lam=dict(lambda_ct_islands=0.9), seed=12)
    assert r.Ke - (K + 2 + T) > 0 and T % 4 != 0
    _run_and_check(r, f"T37 {precision}")


ORDERS = {
    "graphs-first": ("graphs", "expr", "density", "ct", "mask"),
    "mask-first": ("mask", "expr", "density", "graphs", "ct"),
    "expression-twice": ("expr", "density", "graphs", "ct", "mask", "expr", "ct"),
}


@pytest.mark.parametrize("precision", PRECISIONS)
def test_call_order_does_not_matter(precision):
    """Handles that differ only in the order of set_graph, set_loss_genes and set_expression (once with an unrelated
    signed expression set first) give the same history, Y_ext and dY_ext bit for bit after two steps."""
    N, V, K, T = 1500, 700, 130, 8
    inp = synthetic_inputs(N, V, K, seed=13, n_types=T)
    a = _inactive(K, np.random.default_rng(13))
    ops, _, _ = _irregular_ops(V, 13, False, "csr")
    kw = dict(ct_encode=inp["ct_encode"], graphs=ops, mask=a, lam=ALL_TERMS, seed=13)
    base = LRun(precision, inp["S"], inp["G"], inp["d"], **kw)
    S2, G2, _, _, _ = _signed_inputs(N, V, K, seed=14)
    others = {name: LRun(precision, inp["S"], inp["G"], inp["d"], order=order, **kw) for name, order in ORDERS.items()}
    others["other-expression-first"] = LRun(precision, inp["S"], inp["G"], inp["d"], first_expression=(S2, G2), **kw)
    for r in [base, *others.values()]:
        r.e.run(2)
    for name, r in others.items():
        assert np.array_equal(r.e.history(), base.e.history(), equal_nan=True), f"{name}: history"
        for buf in ("Y", "dY"):
            x, y = r.e.debug(buf), base.e.debug(buf)
            assert np.array_equal(x, y), f"{name}: {buf} differs in {int((x != y).sum())} elements"
    M = base.nv("M")
    base.e.step_begin()
    base.e.step_end(LR)
    _check_loss(base, M, f"call order {precision}[3]")


def test_malformed_graph_is_refused():
    """tgb200_set_graph refuses an indptr that decreases between ends 0 and nnz, and one with a negative entry (either
    would make the host transpose write past its buffers); a valid graph and a step work afterwards."""
    from tangram_b200 import _lib
    from tangram_b200.engine import _csr
    N, V, K = 600, 300, 70
    inp = synthetic_inputs(N, V, K, seed=15)
    ops = _grid_ops(V)
    r = LRun("fp32", inp["S"], inp["G"], inp["d"], graphs={0: ops[0]}, lam=dict(lambda_neighborhood_g1=0.9), seed=15)
    lib = _lib.load()
    ip, ix, vv = _csr(ops[0], V)
    nnz = len(vv)
    decreasing = ip.copy()
    decreasing[1] = nnz                               # row 0 spans every entry, row 1 runs backwards
    negative = ip.copy()
    negative[V // 2] = -3
    for bad in (decreasing, negative):
        assert bad[0] == 0 and bad[V] == nnz
        rc = lib.tgb200_set_graph(r.e._h, _lib.GRAPH_VOXEL_WEIGHTS, _lib.ptr(bad), _lib.ptr(ix), _lib.ptr(vv), nnz, None)
        assert rc == -1, f"malformed indptr accepted (status {rc})"             # TGB200_ERR_INVALID
        assert b"indptr" in lib.tgb200_last_error()
    r.e.set_graph(_lib.GRAPH_VOXEL_WEIGHTS, ops[0])
    _run_and_check(r, "after refused graphs fp32", steps=(1,))
