"""highly_variable_genes and hvg without a GPU: the Python layer runs with a float64 numpy stand-in for `group_stats` (the
device pass, tgb200_group_stats / tgb200_group_stats_expm1) and is compared with an independent restatement of scanpy
1.10's seurat and cell_ranger selection -- numpy means and variances over each batch's rows of expm1(x) (or x), bin
edges written out (pandas' rule for integer bins: linspace over [min, max] with the lowest edge lowered by 0.1 % of the
range, right-closed; np.percentile edges for cell_ranger) and per-bin mean / std / median / MAD in loops, no pd.cut and no
groupby.

* both flavors on dense, sparse and layer input, uns["log1p"]["base"], n_top_genes below the gene count, above it and
  above the non-NaN count (the warning), the default and custom cutoffs, a bin of one gene, an all-zero gene;
* batch_key as categorical, strings and with missing values, a gene absent from one batch, a one-cell batch;
* subset and inplace=False, every refusal, hvg and the tutorial flow into pp_adatas;
* tgb200_group_stats_expm1's argument checks, and the refusal of the device pass without a GPU.
"""
import ctypes
import warnings

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import tangram_b200 as tg
from tangram_b200 import MiniAnnData, _lib, gene_selection

CALLS = []


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def group_stats_f64(X, labels, n_labels, *, device=None, expm1_scale=None, _block_rows=0):
    """gene_selection.group_stats in float64 numpy over the float32 values of X (of expm1(scale * x) with expm1_scale)."""
    CALLS.append(expm1_scale)
    X = (X.toarray() if sp.issparse(X) else np.asarray(X)).astype(np.float32).astype(np.float64)
    Y = np.expm1(expm1_scale * X) if expm1_scale is not None else X
    lab = np.asarray(labels).reshape(-1)
    S = np.stack([Y[lab == t].sum(axis=0) for t in range(n_labels)])
    Q = np.stack([(Y[lab == t] ** 2).sum(axis=0) for t in range(n_labels)])
    NZ = np.stack([(X[lab == t] != 0).sum(axis=0) for t in range(n_labels)]).astype(np.int64)
    return S, Q, NZ


@pytest.fixture(autouse=True)
def host_stats(monkeypatch):
    monkeypatch.setattr(gene_selection, "group_stats", group_stats_f64)
    CALLS.clear()


def expression(N=400, G=160, seed=0):
    """log1p-like expression: gene-dependent depth and sparsity, so means and dispersions spread over every bin."""
    rng = np.random.default_rng(seed)
    depth = rng.gamma(0.8, 1.5, G)
    X = rng.gamma(1.2, 1.0, (N, G)) * depth * (rng.random((N, G)) < rng.uniform(0.2, 0.9, G))
    return np.log1p(X).astype(np.float32)


def adata_of(X, batches=None, categorical=False):
    obs = pd.DataFrame(index=[f"c{i}" for i in range(X.shape[0])])
    if batches is not None:
        obs["batch"] = pd.Categorical(batches) if categorical else batches
    return MiniAnnData(X=X, obs=obs, var=pd.DataFrame(index=[f"G{k}" for k in range(X.shape[1])]))


# ---- the restatement ---------------------------------------------------------------------------------------------------

def bin_edges(mean, flavor, n_bins):
    if flavor == "cell_ranger":
        return np.r_[-np.inf, np.percentile(mean, np.arange(10, 105, 5)), np.inf]
    mn, mx = np.nanmin(mean), np.nanmax(mean)
    if mn == mx:
        pad = 0.001 * abs(mn) if mn != 0 else 0.001
        return np.linspace(mn - pad, mx + pad, n_bins + 1)
    edges = np.linspace(mn, mx, n_bins + 1)
    edges[0] -= 0.001 * (mx - mn)
    return edges


def moments(Y):
    """Per-gene mean and variance of the (cells, genes) float64 matrix (ddof=1, or 0 for one cell)."""
    return Y.mean(axis=0), Y.var(axis=0, ddof=1) if Y.shape[0] > 1 else Y.var(axis=0)


def one_batch(mean, var, flavor, n_bins, n_top, cut):
    """scanpy's single-batch steps on one batch's per-gene mean and variance of expm1(x) (seurat) or x (cell_ranger)."""
    mean = mean.copy()
    mean[mean == 0] = 1e-12
    disp = var / mean
    if flavor == "seurat":
        disp[disp == 0] = np.nan
        with np.errstate(divide="ignore", invalid="ignore"):
            disp = np.log(disp)
        mean = np.log1p(mean)
    edges = bin_edges(mean, flavor, n_bins)
    code = np.full(len(mean), -1)
    for j, m in enumerate(mean):
        for b in range(len(edges) - 1):
            if edges[b] < m <= edges[b + 1]:
                code[j] = b
                break
    norm = np.full(len(mean), np.nan)
    for b in set(code.tolist()) - {-1}:
        members = [j for j in range(len(mean)) if code[j] == b]
        d = [disp[j] for j in members if not np.isnan(disp[j])]
        if flavor == "seurat":
            avg = sum(d) / len(d) if d else np.nan
            dev = np.sqrt(sum((v - avg) ** 2 for v in d) / (len(d) - 1)) if len(d) > 1 else np.nan
            if np.isnan(dev):
                avg, dev = 0.0, avg
        else:
            avg = np.median(d) if d else np.nan
            allv = np.array([disp[j] for j in members])
            dev = np.median(np.abs(allv - np.median(allv))) / 0.6744897501960817
        with np.errstate(divide="ignore", invalid="ignore"):
            for j in members:
                norm[j] = (disp[j] - avg) / dev
    if n_top is None:
        d0 = np.where(np.isnan(norm), 0.0, norm)
        hv = (mean > cut[0]) & (mean < cut[1]) & (d0 > cut[2]) & (d0 < cut[3])
    else:
        finite = sorted((v for v in norm if not np.isnan(v)), reverse=True)
        k = min(n_top, len(norm), len(finite))
        hv = np.array([not np.isnan(v) and k > 0 and v >= finite[k - 1] for v in norm])
    return mean, disp, norm, hv


def restate(X, batches=None, flavor="seurat", n_bins=20, n_top=None, cut=(0.0125, 3, 0.5, np.inf), base=None):
    """-> dict of the expected var columns."""
    X = (X.toarray() if sp.issparse(X) else np.asarray(X)).astype(np.float32).astype(np.float64)
    Y = np.expm1(X * (np.log(base) if base is not None else 1.0)) if flavor == "seurat" else X
    G = X.shape[1]
    if batches is None:
        mean, disp, norm, hv = one_batch(*moments(Y), flavor, n_bins, n_top, cut)
        return {"highly_variable": hv, "means": mean, "dispersions": disp, "dispersions_norm": norm}
    col = pd.Series(batches)
    names = list(col.cat.categories) if isinstance(col.dtype, pd.CategoricalDtype) else sorted(set(col.dropna()))
    stats = []
    for name in names:
        rows = np.array([v == name for v in col])
        stats.append((*moments(Y[rows]), (X[rows] != 0).sum(axis=0) > 0))
    return combine(stats, flavor, n_bins, n_top, cut)


def combine(stats, flavor, n_bins, n_top, cut):
    """The batched steps over each batch's (mean, var, gene present) -> dict of the expected var columns."""
    G = len(stats[0][0])
    per = np.zeros((4, len(stats), G))
    for b, (mean_b, var_b, present) in enumerate(stats):
        out = one_batch(mean_b[present], var_b[present], flavor, n_bins, n_top, cut)
        for k in range(4):
            per[k, b, present] = out[k]
    agg = []
    for k in range(3):
        agg.append(np.array([np.mean([v for v in per[k, :, j] if not np.isnan(v)]) if (~np.isnan(per[k, :, j])).any()
                             else np.nan for j in range(G)]))
    mean, disp, norm = agg
    nb = per[3].sum(axis=0).astype(np.int64)
    if n_top is None:
        norm = np.where(np.isnan(norm), 0.0, norm)
        hv = (mean > cut[0]) & (mean < cut[1]) & (norm > cut[2]) & (norm < cut[3])
    else:
        order = sorted(range(G), key=lambda j: (-nb[j], bool(np.isnan(norm[j])), 0.0 if np.isnan(norm[j]) else -norm[j], j))
        hv = np.zeros(G, bool)
        hv[order[:n_top]] = True
    return {"highly_variable": hv, "means": mean, "dispersions": disp, "dispersions_norm": norm,
            "highly_variable_nbatches": nb, "highly_variable_intersection": nb == len(stats)}


def check(var, want):
    assert list(var["highly_variable"].to_numpy()) == list(want["highly_variable"])
    assert var["highly_variable"].dtype == bool
    for c in ("means", "dispersions"):
        assert var[c].dtype == np.float64
        np.testing.assert_allclose(var[c].to_numpy(), want[c], rtol=1e-10, atol=1e-12, equal_nan=True)
    assert var["dispersions_norm"].dtype == np.float32
    np.testing.assert_allclose(var["dispersions_norm"].to_numpy(), want["dispersions_norm"].astype(np.float32),
                               rtol=1e-5, atol=1e-6, equal_nan=True)
    if "highly_variable_nbatches" in want:
        assert var["highly_variable_nbatches"].dtype == np.int64
        np.testing.assert_array_equal(var["highly_variable_nbatches"].to_numpy(), want["highly_variable_nbatches"])
        assert var["highly_variable_intersection"].dtype == bool
        np.testing.assert_array_equal(var["highly_variable_intersection"].to_numpy(),
                                      want["highly_variable_intersection"])


# ---- tests ---------------------------------------------------------------------------------------------------------------

def test_public_names():
    assert tg.highly_variable_genes is gene_selection.highly_variable_genes
    assert tg.hvg is gene_selection.hvg


@pytest.mark.parametrize("flavor", ["seurat", "cell_ranger"])
@pytest.mark.parametrize("kind", ["dense", "sparse", "layer"])
def test_single_batch_against_restatement(flavor, kind):
    X = expression(seed=1)
    if kind == "layer":
        ad = adata_of(np.zeros_like(X))
        ad.layers = {"logged": sp.csc_matrix(X)}
    else:
        ad = adata_of(sp.csr_matrix(X) if kind == "sparse" else X)
    layer = "logged" if kind == "layer" else None
    tg.highly_variable_genes(ad, flavor=flavor, n_top_genes=40, layer=layer)
    assert CALLS == [1.0 if flavor == "seurat" else None]           # one pass; expm1 only for seurat
    assert ad.uns["hvg"] == {"flavor": flavor}
    assert list(ad.var.columns) == ["highly_variable", "means", "dispersions", "dispersions_norm"]
    assert ad.var["highly_variable"].sum() == 40
    check(ad.var, restate(X, flavor=flavor, n_top=40))
    tg.highly_variable_genes(ad, flavor=flavor, layer=layer)          # the default cutoffs
    want = restate(X, flavor=flavor)
    assert 0 < want["highly_variable"].sum() < X.shape[1]
    check(ad.var, want)


def test_log1p_base_scales_expm1():
    X = expression(seed=2)
    ad = adata_of(X)
    ad.uns["log1p"] = {"base": 2}
    tg.highly_variable_genes(ad, n_top_genes=30)
    assert CALLS == [pytest.approx(np.log(2), rel=1e-15)]
    check(ad.var, restate(X, n_top=30, base=2))
    tg.highly_variable_genes(ad, flavor="cell_ranger", n_top_genes=30)   # cell_ranger reads x itself
    check(ad.var, restate(X, flavor="cell_ranger", n_top=30))


def test_n_top_genes_beyond_the_genes_and_the_non_nan():
    X = expression(G=60, seed=3)
    ad = adata_of(X)
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        tg.highly_variable_genes(ad, n_top_genes=500)                # no NaN: every gene, silently
    assert ad.var["highly_variable"].all()
    X[:, 7] = 0.0                                                     # an all-zero gene: dispersion NaN
    ad = adata_of(X)
    with pytest.warns(UserWarning, match="n_top_genes"):
        tg.highly_variable_genes(ad, n_top_genes=60)
    assert np.isnan(ad.var["dispersions"].iloc[7]) and np.isnan(ad.var["dispersions_norm"].iloc[7])
    assert not ad.var["highly_variable"].iloc[7] and ad.var["highly_variable"].sum() == 59
    check(ad.var, restate(X, n_top=60))


def test_custom_cutoffs_and_an_all_zero_gene():
    X = expression(seed=4)
    X[:, 3] = 0.0
    ad = adata_of(sp.csr_matrix(X))
    cut = dict(min_mean=0.2, max_mean=2.5, min_disp=-0.3, max_disp=1.5)
    tg.highly_variable_genes(ad, n_bins=8, **cut)
    want = restate(X, n_bins=8, cut=(0.2, 2.5, -0.3, 1.5))
    assert 0 < want["highly_variable"].sum() < X.shape[1]
    check(ad.var, want)
    assert not ad.var["highly_variable"].iloc[3] and np.isnan(ad.var["dispersions_norm"].iloc[3])
    tg.highly_variable_genes(ad, flavor="cell_ranger", **cut)
    check(ad.var, restate(X, flavor="cell_ranger", cut=(0.2, 2.5, -0.3, 1.5)))


def test_a_bin_of_one_gene_is_normalised_to_one():
    X = expression(seed=5)
    X[:, 11] = np.log1p(np.expm1(X[:, 11]) * 400.0)                  # far above every other mean: alone in its bin
    ad = adata_of(X)
    tg.highly_variable_genes(ad, n_top_genes=20)
    want = restate(X, n_top=20)
    assert want["dispersions_norm"][11] == pytest.approx(1.0, rel=1e-12)
    check(ad.var, want)


@pytest.mark.parametrize("kind", ["categorical", "strings", "missing"])
@pytest.mark.parametrize("flavor", ["seurat", "cell_ranger"])
def test_batches_against_restatement(kind, flavor):
    X = expression(N=420, seed=6)
    rng = np.random.default_rng(7)
    batches = np.array(["b1", "b0", "b2"], dtype=object)[rng.integers(0, 3, X.shape[0])]
    X[batches == "b1", 5] = 0.0                                       # gene 5 absent from batch b1
    if kind == "missing":
        batches[::9] = None
    ad = adata_of(X, batches, categorical=kind == "categorical")
    tg.highly_variable_genes(ad, flavor=flavor, n_top_genes=35, batch_key="batch")
    assert len(CALLS) == 1
    assert list(ad.var.columns) == ["highly_variable", "means", "dispersions", "dispersions_norm",
                                    "highly_variable_nbatches", "highly_variable_intersection"]
    want = restate(X, batches, flavor=flavor, n_top=35)
    check(ad.var, want)
    assert ad.var["highly_variable"].sum() == 35 and ad.var["highly_variable_nbatches"].max() == 3
    assert ad.var["highly_variable_nbatches"].iloc[5] <= 2
    tg.highly_variable_genes(ad, flavor=flavor, batch_key="batch")
    check(ad.var, restate(X, batches, flavor=flavor))


def test_one_cell_batch_and_a_gene_only_in_one_batch():
    X = expression(N=300, seed=8)
    batches = np.where(np.arange(300) < 150, "early", "late").astype(object)
    batches[42] = "solo"                                              # one cell: variance without the correction
    X[batches != "late", 9] = 0.0                                     # gene 9 only in "late"
    ad = adata_of(X, batches)
    with pytest.warns(UserWarning, match="n_top_genes"):            # "solo": every dispersion 0, so NaN
        tg.highly_variable_genes(ad, n_top_genes=25, batch_key="batch")
    want = restate(X, batches, n_top=25)
    check(ad.var, want)
    tg.highly_variable_genes(ad, flavor="cell_ranger", min_disp=-5.0, batch_key="batch")
    check(ad.var, restate(X, batches, flavor="cell_ranger", cut=(0.0125, 3, -5.0, np.inf)))


def test_subset_and_not_inplace():
    X = expression(seed=9)
    ad = adata_of(X)
    df = tg.highly_variable_genes(ad, n_top_genes=30, inplace=False)
    assert ad.uns == {} and list(ad.var.columns) == []                 # untouched
    assert list(df.index) == list(ad.var_names) and df["dispersions_norm"].dtype == np.float32
    check(df, restate(X, n_top=30))
    top = tg.highly_variable_genes(ad, n_top_genes=30, inplace=False, subset=True)
    pd.testing.assert_frame_equal(top, df[df["highly_variable"]])
    assert tg.highly_variable_genes(ad, n_top_genes=30, subset=True) is None
    assert ad.shape == (X.shape[0], 30) and list(ad.var_names) == list(top.index)
    np.testing.assert_array_equal(ad.X, X[:, df["highly_variable"].to_numpy()])
    assert ad.var["highly_variable"].all()


def test_refusals():
    X = expression(G=40, seed=10)
    ad = adata_of(X, np.array(["a", "b"] * 200, dtype=object))
    for f in ("seurat_v3", "seurat_v3_paper"):
        with pytest.raises(NotImplementedError, match="loess"):
            tg.highly_variable_genes(ad, flavor=f)
    with pytest.raises(ValueError, match="flavor='pearson'"):
        tg.highly_variable_genes(ad, flavor="pearson")
    with pytest.raises(ValueError, match="batch_key='nope'"):
        tg.highly_variable_genes(ad, batch_key="nope")
    with pytest.raises(ValueError, match="not in adata.layers"):
        tg.highly_variable_genes(ad, layer="counts")
    with pytest.raises(ValueError, match="n_bins=0"):
        tg.highly_variable_genes(ad, n_bins=0)
    with pytest.raises(ValueError, match="n_top_genes=0"):
        tg.highly_variable_genes(ad, n_top_genes=0)
    assert CALLS == [] and ad.uns == {} and list(ad.var.columns) == []


def test_hvg_is_the_selected_names():
    X = expression(G=300, seed=11)
    ad = adata_of(sp.csr_matrix(X))
    got = tg.hvg(ad, n_top_genes=50)
    want = restate(X, n_top=50)["highly_variable"]
    assert got == [f"G{k}" for k in np.nonzero(want)[0]] and len(got) == 50
    assert tg.hvg(ad) == list(ad.var_names)                          # 4000 > 300 genes: all of them (none is NaN)


def test_tutorial_flow_into_pp_adatas():
    """pp_adatas(ad_sc, ad_sp, genes=hvg(ad_sc)), the reference's hvg alternative to ctg."""
    X = expression(N=300, G=200, seed=12)
    ad_sc = adata_of(sp.csr_matrix(X))
    ad_sc.var.index = [f"Gene{k}" for k in range(X.shape[1])]
    rng = np.random.default_rng(13)
    sp_genes = [f"Gene{k}" for k in range(0, 200, 2)] + ["Other"]
    ad_sp = MiniAnnData(X=rng.random((20, len(sp_genes))).astype(np.float32), var=pd.DataFrame(index=sp_genes))
    genes = tg.hvg(ad_sc, n_top_genes=60)
    tg.pp_adatas(ad_sc, ad_sp, genes=genes)
    expect = {g.lower() for g in genes} & {g.lower() for g in sp_genes}
    assert sorted(ad_sc.uns["training_genes"]) == sorted(expect) and len(expect) > 0


def test_expm1_entry_point_checks_arguments():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    lab = np.array([0, 1, -1, 2], dtype=np.int32)
    s, q, n = np.empty((3, 4)), np.empty((3, 4)), np.empty((3, 4), np.int64)
    out = (_lib.ptr(s), _lib.ptr(q), _lib.ptr(n))

    def call(X=fake, x_ld=4, indptr=None, rows=4, labels=lab, T=3, outs=out, block=0, scale=1.0):
        return lib.tgb200_group_stats_expm1(X, x_ld, indptr, None, None, 0, rows, 4, _lib.ptr(labels), T, *outs, block,
                                            0, None, scale)
    assert call(X=None) == -1 and b"exactly one of X" in lib.tgb200_last_error()
    assert call(x_ld=3) == -1 and b"bad shape" in lib.tgb200_last_error()
    assert call(outs=(None, _lib.ptr(q), None)) == -1 and b"null argument" in lib.tgb200_last_error()
    assert call(T=0) == -1 and b"n_labels=0" in lib.tgb200_last_error()
    assert call(block=1024) == -1 and b"block_rows=1024 is not a multiple of 2048" in lib.tgb200_last_error()
    assert call(T=2) == -1 and b"label 2 of row 3 is outside [-1, 2)" in lib.tgb200_last_error()
    for bad in (np.nan, np.inf):
        assert call(scale=bad) == -1 and b"is not finite" in lib.tgb200_last_error()
    if not _has_gpu():
        assert call() == -5 and b"no CPU fallback" in lib.tgb200_last_error()


def test_expm1_pass_refuses_without_gpu(monkeypatch):
    monkeypatch.undo()
    gs = gene_selection.group_stats
    assert gs is not group_stats_f64
    with pytest.raises(ValueError, match=r"labels must lie in \[-1, 1\)"):
        gs(np.ones((3, 2), np.float32), [0, 1, 0], 1, expm1_scale=1.0)
    if not _has_gpu():
        with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
            gs(np.ones((3, 2), np.float32), [0, 0, -1], 1, expm1_scale=np.log(2))
        with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
            tg.highly_variable_genes(adata_of(np.ones((3, 2), np.float32)))
