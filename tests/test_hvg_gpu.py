"""tgb200_group_stats_expm1 and highly_variable_genes on the H100.

* the per-label sums and sums of squares of expm1(scale * x) within 1e-12 of float64 numpy, the nonzero counts (of x)
  exact, for scale 1 and ln 2: rows not a multiple of 2048, genes not a multiple of 4 or 1024, a row stride beyond the
  genes, empty rows, explicit CSR zeros, NaN, and a strided CUDA tensor;
* identical bits for dense and CSR, host and device data, block_rows 2048, 6144 and the default, and a re-run;
* highly_variable_genes on dense, CSR and CUDA-tensor X equals the float64 host stand-in run (the same genes but for
  those within 1e-9 of the cut, means and dispersions within 1e-12, dispersions_norm within one float32 rounding), and one
  run at 100k cells x 20k genes x 6 batches (CSR) equals the restatement.
"""
import ctypes

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import tangram_b200 as tg  # noqa: E402
from tangram_b200 import MiniAnnData, _lib, gene_selection  # noqa: E402
from tests.test_hvg import combine, group_stats_f64  # noqa: E402
from tests.test_rank_genes_gpu import bits, check, f64_stats, sample  # noqa: E402

DEV = torch.cuda.current_device()
SCALES = [1.0, float(np.log(2.0))]


def want_stats(X, lab, T, scale):
    """float64 sums and sums of squares of expm1(scale * x) per label, and the counts of x != 0."""
    X = X.toarray() if sp.issparse(X) else np.asarray(X)
    Y = np.expm1(scale * X.astype(np.float64))
    s, q, _ = f64_stats(Y, lab, T)
    return s, q, f64_stats(X, lab, T)[2]


def raw_call(labels, T, scale, *, X=None, x_ld=0, csr=None, n_genes=None, block=0, out=None):
    """tgb200_group_stats_expm1 on numpy arrays or torch tensors (host or device) -> (status, (sum, sumsq, nnz))."""
    lab = np.ascontiguousarray(labels, dtype=np.int32)
    G = n_genes
    s, q, n = out if out is not None else (np.zeros((T, G)), np.zeros((T, G)), np.zeros((T, G), np.int64))
    if csr is not None:
        ip, ix, dv = csr
        x = (None, 0, _lib.ptr(ip), _lib.ptr(ix), _lib.ptr(dv), int(ix.shape[0]))
    else:
        x = (_lib.ptr(X), x_ld, None, None, None, 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    st = _lib.load().tgb200_group_stats_expm1(*x, len(lab), G, _lib.ptr(lab), T, _lib.ptr(s), _lib.ptr(q), _lib.ptr(n),
                                              block, DEV, stream, scale)
    if out is not None:
        torch.cuda.synchronize()
        s, q, n = (a.cpu().numpy() for a in out)
    return st, (s, q, n)


def logged(N, G, T, seed, density=0.3):
    X, lab = sample(N, G, T, seed, density=density)
    return np.log1p(X).astype(np.float32), lab


@pytest.mark.parametrize("scale", SCALES)
def test_expm1_against_float64_awkward_shapes(scale):
    X, lab = logged(5000, 1030, 7, seed=1)
    X[17] = 0.0                                              # an empty row
    lab[lab == 5] = 2                                        # label 5 without rows
    want = want_stats(X, lab, 7, scale)
    check(gene_selection.group_stats(X, lab, 7, expm1_scale=scale), want)
    check(gene_selection.group_stats(sp.csr_matrix(X), lab, 7, expm1_scale=scale), want)
    Xw = np.zeros((5000, 1035), np.float32)                  # host rows with a stride beyond the genes
    Xw[:, :1030] = X
    st, got = raw_call(lab, 7, scale, X=Xw, x_ld=1035, n_genes=1030)
    assert st == 0
    check(got, want)
    assert np.all(got[0][5] == 0) and np.all(got[2][5] == 0)


@pytest.mark.parametrize("scale", SCALES)
def test_explicit_zeros_and_nan(scale):
    X, lab = logged(3000, 70, 4, seed=2)
    csr = sp.csr_matrix(X)
    csr.data[::9] = 0.0                                      # explicit zeros, kept as stored entries
    dense = csr.toarray()
    got = gene_selection.group_stats(csr, lab, 4, expm1_scale=scale)
    check(got, want_stats(dense, lab, 4, scale))
    assert bits(got) == bits(gene_selection.group_stats(dense, lab, 4, expm1_scale=scale))
    dense[100, 3] = np.nan
    lab[100] = 0
    s, q, n = gene_selection.group_stats(dense, lab, 4, expm1_scale=scale)
    assert np.isnan(s[0, 3]) and np.isnan(q[0, 3]) and not np.isnan(s[1:]).any()
    assert n[0, 3] == (dense[lab == 0, 3] != 0).sum()        # NaN counts as nonzero
    ok = np.ones(70, bool)
    ok[3] = False
    check(tuple(a[:, ok] for a in (s, q, n)), tuple(a[:, ok] for a in want_stats(dense, lab, 4, scale)))


def test_strided_cuda_tensor():
    X, lab = logged(4100, 300, 5, seed=3)
    big = torch.zeros((4100, 333), dtype=torch.float32, device=DEV)
    big[:, 10:310] = torch.from_numpy(X).to(DEV)
    view = big[:, 10:310]                                     # row stride 333, not 16-byte aligned
    got = gene_selection.group_stats(view, lab, 5, expm1_scale=SCALES[1])
    check(got, want_stats(X, lab, 5, SCALES[1]))
    assert bits(got) == bits(gene_selection.group_stats(X, lab, 5, expm1_scale=SCALES[1]))


def test_bits_identical_however_staged():
    X, lab = logged(9000, 1100, 9, seed=4, density=0.2)
    csr = sp.csr_matrix(X)
    ip, ix, dv = csr.indptr.astype(np.int64), csr.indices.astype(np.int32), csr.data.astype(np.float32)
    dip, dix, ddv = (torch.from_numpy(a).to(DEV) for a in (ip, ix, dv))
    dX = torch.from_numpy(X).to(DEV)
    sc = SCALES[1]
    ref = None
    for block in (2048, 6144, 0):
        runs = [raw_call(lab, 9, sc, X=X, x_ld=1100, n_genes=1100, block=block),
                raw_call(lab, 9, sc, X=dX, x_ld=1100, n_genes=1100, block=block),
                raw_call(lab, 9, sc, csr=(ip, ix, dv), n_genes=1100, block=block),
                raw_call(lab, 9, sc, csr=(dip, dix, ddv), n_genes=1100, block=block)]
        dev_out = tuple(torch.empty((9, 1100), dtype=d, device=DEV) for d in (torch.float64, torch.float64, torch.int64))
        runs.append(raw_call(lab, 9, sc, csr=(ip, ix, dv), n_genes=1100, block=block, out=dev_out))
        for st, got in runs:
            assert st == 0, _lib.load().tgb200_last_error()
            ref = ref or bits(got)
            assert bits(got) == ref
    st, got = raw_call(lab, 9, sc, X=X, x_ld=1100, n_genes=1100)
    assert st == 0 and bits(got) == ref                      # a re-run
    check(got, want_stats(X, lab, 9, sc))


def same_selection(var, hv_want, norm_want, nb_want=None):
    """The selected genes agree, except genes whose dispersions_norm is within 1e-9 relative of the cut (the last
    selected gene's, in its nbatches tier)."""
    got = var["highly_variable"].to_numpy()
    diff = np.nonzero(got != hv_want)[0]
    if diff.size == 0:
        return
    nb = np.zeros(len(got), np.int64) if nb_want is None else nb_want
    sel = np.nonzero(hv_want)[0]
    edge = sel[np.lexsort((norm_want[sel], nb[sel]))[0]]       # the weakest selected gene
    for j in diff:
        assert nb[j] == nb[edge] and abs(norm_want[j] - norm_want[edge]) <= 1e-9 * abs(norm_want[edge]), j


@pytest.mark.parametrize("kind", ["dense", "csr", "cuda"])
def test_highly_variable_genes_matches_host_stand_in(kind, monkeypatch):
    X, _ = logged(6000, 900, 1, seed=5, density=0.35)
    rng = np.random.default_rng(6)
    X *= rng.uniform(0.3, 2.0, 900).astype(np.float32)       # spread the genes' means and dispersions
    batches = np.array(["x", "y", "z"], dtype=object)[rng.integers(0, 3, 6000)]
    batches[::11] = None
    X[batches == "y", 8] = 0.0                               # a gene absent from one batch
    Xin = {"dense": X, "csr": sp.csr_matrix(X), "cuda": torch.from_numpy(X).to(DEV)}[kind]
    obs = pd.DataFrame({"batch": batches}, index=[f"c{i}" for i in range(6000)])
    var = pd.DataFrame(index=[f"G{k}" for k in range(900)])
    runs = [dict(n_top_genes=120), dict(n_top_genes=150, batch_key="batch"), dict(flavor="cell_ranger"),
            dict(flavor="cell_ranger", n_top_genes=100, batch_key="batch")]
    for kw in runs:
        ad = MiniAnnData(X=Xin, obs=obs, var=var.copy(), uns={"log1p": {"base": 2.0}})
        tg.highly_variable_genes(ad, **kw)
        with monkeypatch.context() as m:
            m.setattr(gene_selection, "group_stats", group_stats_f64)
            ad_h = MiniAnnData(X=X, obs=obs, var=var.copy(), uns={"log1p": {"base": 2.0}})
            tg.highly_variable_genes(ad_h, **kw)
        g, h = ad.var, ad_h.var
        nb = h["highly_variable_nbatches"].to_numpy() if "batch_key" in kw else None
        same_selection(g, h["highly_variable"].to_numpy(), h["dispersions_norm"].to_numpy().astype(np.float64), nb)
        for c in ("means", "dispersions"):
            np.testing.assert_allclose(g[c].to_numpy(), h[c].to_numpy(), rtol=1e-12, atol=1e-12, equal_nan=True)
        # float32 of float64 values that differ in the last bits: equal, or one float32 rounding apart
        np.testing.assert_allclose(g["dispersions_norm"].to_numpy(), h["dispersions_norm"].to_numpy(), rtol=1.2e-7,
                                   atol=1e-12, equal_nan=True)
        if nb is not None:
            np.testing.assert_array_equal(g["highly_variable_nbatches"].to_numpy(), nb)


def test_atlas_sample_against_restatement():
    """100k cells x 20k genes (CSR, ~600 entries a cell) x 6 batches, seurat with n_top_genes=2000."""
    rng = np.random.default_rng(9)
    N, G, B, k = 100_000, 20_000, 6, 600
    cols = np.cumsum(rng.integers(1, 2 * G // k, size=(N, k), dtype=np.int32), axis=1, dtype=np.int32) - 1
    keep = cols < G
    indptr = np.r_[0, np.cumsum(keep.sum(axis=1))].astype(np.int64)
    indices = cols[keep]
    gene_scale = rng.uniform(0.2, 2.5, G)
    data = np.log1p(rng.gamma(1.5, 1.0, indices.shape[0]) * gene_scale[indices]).astype(np.float32)
    X = sp.csr_matrix((data, indices, indptr), shape=(N, G))
    bat = rng.integers(0, B, N)
    names = [f"batch{b}" for b in range(B)]
    obs = pd.DataFrame({"batch": pd.Categorical.from_codes(bat, names)}, index=np.arange(N).astype(str))
    ad = MiniAnnData(X=X, obs=obs, var=pd.DataFrame(index=[f"g{j}" for j in range(G)]))
    tg.highly_variable_genes(ad, n_top_genes=2000, batch_key="batch")
    stats = []
    for b in range(B):                                        # two-pass float64 moments of expm1(x) from the CSR
        Xb = X[bat == b].astype(np.float64)
        n = Xb.shape[0]
        Yb = Xb.copy()
        Yb.data = np.expm1(Yb.data)
        mean = np.asarray(Yb.sum(axis=0)).ravel() / n
        dev = Yb.copy().tocoo()
        dev.data = (dev.data - mean[dev.col]) ** 2
        nnz = np.bincount(Yb.indices, minlength=G)
        var = (np.asarray(dev.tocsr().sum(axis=0)).ravel() + (n - nnz) * mean ** 2) / (n - 1)
        stats.append((mean, var, np.bincount(Xb.indices, weights=Xb.data != 0, minlength=G) > 0))
    want = combine(stats, "seurat", 20, 2000, None)
    assert (want["highly_variable_nbatches"] < B).any()     # some genes are absent from a batch or not chosen there
    same_selection(ad.var, want["highly_variable"], want["dispersions_norm"], want["highly_variable_nbatches"])
    for c in ("means", "dispersions"):
        np.testing.assert_allclose(ad.var[c].to_numpy(), want[c], rtol=1e-10, atol=1e-12, equal_nan=True)
    np.testing.assert_allclose(ad.var["dispersions_norm"].to_numpy(), want["dispersions_norm"].astype(np.float32),
                               rtol=1e-5, atol=1e-6, equal_nan=True)
    np.testing.assert_array_equal(ad.var["highly_variable_nbatches"].to_numpy(), want["highly_variable_nbatches"])
    assert ad.var["highly_variable"].sum() == 2000
