"""rank_genes_groups and ctg without a GPU: the Python layer runs with a float64 numpy stand-in for `group_stats` (the
device pass, tgb200_group_stats) and is compared with an independent scipy restatement -- numpy float64 means and ddof=1
variances over X[group] and X[rest], scipy's ttest_ind_from_stats, false_discovery_control and Bonferroni.

* categorical, string and numeric labels, missing labels (in every group's rest), dense and sparse X;
* a groups subset, a reference group, rankby_abs, n_genes truncation, exact ties (the lower gene index first), pts /
  pts_rest, uns["log1p"]["base"], t-test_overestim_var, use_raw and layers;
* the np.rec layout read back through pd.DataFrame, every refusal, ctg, and the tutorial's flow into pp_adatas;
* the C entry point's argument checks, and the refusal of the device pass without a GPU.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
from scipy import stats

import tangram_b200 as tg
from tangram_b200 import MiniAnnData, _lib, gene_selection


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def group_stats_f64(X, labels, n_labels, *, device=None, _block_rows=0):
    """gene_selection.group_stats in float64 numpy over the float32 values of X."""
    X = (X.toarray() if sp.issparse(X) else np.asarray(X)).astype(np.float32).astype(np.float64)
    lab = np.asarray(labels).reshape(-1)
    S = np.stack([X[lab == t].sum(axis=0) for t in range(n_labels)])
    Q = np.stack([(X[lab == t] ** 2).sum(axis=0) for t in range(n_labels)])
    NZ = np.stack([(X[lab == t] != 0).sum(axis=0) for t in range(n_labels)]).astype(np.int64)
    return S, Q, NZ


@pytest.fixture(autouse=True)
def host_stats(monkeypatch):
    monkeypatch.setattr(gene_selection, "group_stats", group_stats_f64)


def expression(N=240, G=30, seed=0, groups="abcd"):
    """log1p-like nonnegative expression with zeros, each group raising its own block of genes."""
    rng = np.random.default_rng(seed)
    lab = np.array(list(groups))[rng.integers(0, len(groups), N)]
    X = rng.gamma(1.5, 1.0, (N, G)) * (rng.random((N, G)) < 0.6)
    for k, g in enumerate(groups):
        X[lab == g, 3 * k:3 * k + 3] += 2.0 + k
    return np.log1p(X).astype(np.float32), lab


def restate(X, labels, group, reference="rest", method="t-test", corr="benjamini-hochberg", base=None):
    X = (X.toarray() if sp.issparse(X) else np.asarray(X)).astype(np.float64)
    labels = np.asarray(labels, dtype=object)
    in_g = labels == group
    rest = labels == reference if reference != "rest" else ~in_g
    mg, vg, ng = X[in_g].mean(axis=0), X[in_g].var(axis=0, ddof=1), in_g.sum()
    mr, vr, nr = X[rest].mean(axis=0), X[rest].var(axis=0, ddof=1), rest.sum()
    sc, p = stats.ttest_ind_from_stats(mg, np.sqrt(vg), ng, mr, np.sqrt(vr), ng if method.endswith("var") else nr,
                                       equal_var=False)
    sc, p = np.nan_to_num(sc, nan=0.0), np.nan_to_num(p, nan=1.0)
    adj = stats.false_discovery_control(p, method="bh") if corr == "benjamini-hochberg" else np.minimum(p * X.shape[1], 1)
    e = (lambda m: np.expm1(m * np.log(base))) if base is not None else np.expm1
    return sc, p, adj, np.log2((e(mg) + 1e-9) / (e(mr) + 1e-9))


def check_group(uns, X, labels, genes, group, *, n_genes=None, rankby_abs=False, **kw):
    """uns's output for `group` (a label value; its field is str(group)) against the restatement."""
    sc, p, adj, lfc = restate(X, labels, group, **kw)
    order = np.argsort(-(np.abs(sc) if rankby_abs else sc), kind="stable")[:n_genes]
    f = str(group)
    assert list(uns["names"][f]) == list(np.asarray(genes)[order])
    np.testing.assert_allclose(uns["scores"][f], sc[order].astype(np.float32), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(uns["pvals"][f], p[order], rtol=1e-7, atol=1e-300)
    np.testing.assert_allclose(uns["pvals_adj"][f], adj[order], rtol=1e-7, atol=1e-300)
    np.testing.assert_allclose(uns["logfoldchanges"][f], lfc[order].astype(np.float32), rtol=1e-5, atol=1e-5)


def adata_of(X, labels, categorical=False):
    obs = pd.DataFrame({"ct": pd.Categorical(labels) if categorical else labels},
                       index=[f"c{i}" for i in range(len(labels))])
    var = pd.DataFrame(index=[f"G{k}" for k in range(X.shape[1])])
    return MiniAnnData(X=X, obs=obs, var=var)


def test_public_names():
    assert tg.rank_genes_groups is gene_selection.rank_genes_groups
    assert tg.ctg is gene_selection.ctg


@pytest.mark.parametrize("kind", ["categorical", "strings", "numeric", "missing", "sparse"])
def test_every_group_against_restatement(kind):
    X, lab = expression(seed=1)
    labels = lab.astype(object)
    if kind == "numeric":
        labels = np.array([{"a": 10, "b": 2, "c": 7, "d": 1}[g] for g in lab])
    if kind == "missing":
        labels[::7] = None                                   # no group, but in every group's rest
    Xin = sp.csr_matrix(X) if kind == "sparse" else X
    ad = adata_of(Xin, labels, categorical=kind == "categorical")
    tg.rank_genes_groups(ad, "ct")
    uns = ad.uns["rank_genes_groups"]
    expect = ["1", "2", "7", "10"] if kind == "numeric" else list("abcd")
    assert list(uns["names"].dtype.names) == expect
    assert uns["params"] == {"groupby": "ct", "reference": "rest", "method": "t-test", "use_raw": False, "layer": None,
                             "corr_method": "benjamini-hochberg"}
    for g in expect:
        check_group(uns, X, labels, ad.var_names, int(g) if kind == "numeric" else g)


def test_numeric_names_follow_numeric_order():
    X, lab = expression(seed=2)
    labels = np.array([{"a": 10.0, "b": 2.0, "c": 7.5, "d": 1.0}[g] for g in lab])
    ad = adata_of(X, labels)
    tg.rank_genes_groups(ad, "ct")
    assert list(ad.uns["rank_genes_groups"]["names"].dtype.names) == ["1.0", "2.0", "7.5", "10.0"]
    check_group(ad.uns["rank_genes_groups"], X, labels, ad.var_names, 7.5)


def test_subset_reference_rankby_abs_and_truncation():
    X, lab = expression(seed=3)
    ad = adata_of(sp.csr_matrix(X), lab, categorical=True)
    tg.rank_genes_groups(ad, "ct", groups=["c", "a"], n_genes=7)
    uns = ad.uns["rank_genes_groups"]
    assert list(uns["names"].dtype.names) == ["c", "a"] and len(uns["names"]) == 7
    for g in ("c", "a"):                                     # the rest includes the unselected groups b and d
        check_group(uns, X, lab, ad.var_names, g, n_genes=7)
    tg.rank_genes_groups(ad, "ct", groups=["a", "b", "d"], reference="b", rankby_abs=True, key_added="vs_b")
    uns = ad.uns["vs_b"]
    assert list(uns["names"].dtype.names) == ["a", "d"] and uns["params"]["reference"] == "b"
    for g in ("a", "d"):
        check_group(uns, X, lab, ad.var_names, g, reference="b", rankby_abs=True)
    tg.rank_genes_groups(ad, "ct", groups=["a"], reference="d", n_genes=100, key_added="a_vs_d")
    assert len(ad.uns["a_vs_d"]["names"]) == X.shape[1]       # n_genes beyond the genes keeps them all
    check_group(ad.uns["a_vs_d"], X, lab, ad.var_names, "a", reference="d")


def test_exact_ties_keep_gene_order():
    X, lab = expression(seed=4, G=12)
    X = np.concatenate([X[:, [5]], X, X[:, [5, 0, 0]]], axis=1)   # genes 0, 6, 13 equal; 1, 14, 15 equal
    ad = adata_of(X, lab)
    tg.rank_genes_groups(ad, "ct", groups=["b"])
    names = list(ad.uns["rank_genes_groups"]["names"]["b"])
    pos = {g: names.index(g) for g in ad.var_names}
    assert pos["G0"] < pos["G6"] < pos["G13"] and pos["G1"] < pos["G14"] < pos["G15"]
    for trio in (["G0", "G6", "G13"], ["G1", "G14", "G15"]):
        assert [pos[g] for g in trio] == list(range(pos[trio[0]], pos[trio[0]] + 3))
    check_group(ad.uns["rank_genes_groups"], X, lab, ad.var_names, "b")


def test_pts_log1p_base_and_overestim_var():
    X, lab = expression(seed=5)
    ad = adata_of(X, lab)
    ad.uns["log1p"] = {"base": 2.0}
    tg.rank_genes_groups(ad, "ct", method="t-test_overestim_var", corr_method="bonferroni", pts=True)
    uns = ad.uns["rank_genes_groups"]
    for g in "abcd":
        check_group(uns, X, lab, ad.var_names, g, method="t-test_overestim_var", corr="bonferroni", base=2.0)
        np.testing.assert_allclose(uns["pts"][g].to_numpy(), (X[lab == g] != 0).mean(axis=0), rtol=1e-15)
        np.testing.assert_allclose(uns["pts_rest"][g].to_numpy(), (X[lab != g] != 0).mean(axis=0), rtol=1e-15)
    assert list(uns["pts"].index) == list(ad.var_names) and list(uns["pts"].columns) == list("abcd")
    tg.rank_genes_groups(ad, "ct", groups=["a"], reference="c", pts=True, key_added="ref")
    assert list(ad.uns["ref"]["pts"].columns) == ["a", "c"] and "pts_rest" not in ad.uns["ref"]


def test_rec_layout_through_dataframe():
    X, lab = expression(seed=6)
    ad = adata_of(X, lab, categorical=True)
    tg.rank_genes_groups(ad, "ct", n_genes=5)
    uns = ad.uns["rank_genes_groups"]
    for field, dt in (("names", object), ("scores", np.float32), ("logfoldchanges", np.float32),
                      ("pvals", np.float64), ("pvals_adj", np.float64)):
        assert isinstance(uns[field], np.recarray)
        df = pd.DataFrame(uns[field])
        assert list(df.columns) == list("abcd") and df.shape == (5, 4)
        assert all(uns[field].dtype[g] == dt for g in "abcd")
    assert pd.DataFrame(uns["names"]).iloc[0, 0] == uns["names"]["a"][0]


def test_raw_and_layers():
    X, lab = expression(seed=7)
    ad = adata_of(np.zeros_like(X[:, :4]), lab)
    raw_genes = pd.Index([f"R{k}" for k in range(X.shape[1])])
    ad.raw = SimpleNamespace(X=X, var_names=raw_genes)
    tg.rank_genes_groups(ad, "ct", groups=["a"])                  # use_raw=None with a raw: raw.X
    assert ad.uns["rank_genes_groups"]["params"]["use_raw"] is True
    check_group(ad.uns["rank_genes_groups"], X, lab, raw_genes, "a")
    ad2 = adata_of(np.zeros_like(X), lab)
    ad2.layers = {"counts": sp.csc_matrix(X)}
    tg.rank_genes_groups(ad2, "ct", groups=["d"], layer="counts")
    assert ad2.uns["rank_genes_groups"]["params"]["layer"] == "counts"
    check_group(ad2.uns["rank_genes_groups"], X, lab, ad2.var_names, "d")


def test_refusals():
    X, lab = expression(seed=8)
    lab = lab.astype(object)
    lab[:2] = "solo"
    lab[2] = "one"
    ad = adata_of(X, lab)
    with pytest.raises(ValueError, match="groupby='nope'"):
        tg.rank_genes_groups(ad, "nope")
    with pytest.raises(ValueError, match=r"\['zz'\] are not groups"):
        tg.rank_genes_groups(ad, "ct", groups=["a", "zz"])
    with pytest.raises(ValueError, match="reference='zz'"):
        tg.rank_genes_groups(ad, "ct", groups=["a"], reference="zz")
    with pytest.raises(ValueError, match=r"\['one'\].*fewer than 2 cells"):
        tg.rank_genes_groups(ad, "ct")
    with pytest.raises(ValueError, match=r"\['one'\].*fewer than 2 cells"):
        tg.rank_genes_groups(ad, "ct", groups=["a"], reference="one")
    tg.rank_genes_groups(ad, "ct", groups=["a", "solo"])           # 2 cells are enough; "one" is not selected
    with pytest.raises(ValueError, match="names a group twice"):
        tg.rank_genes_groups(ad, "ct", groups=["a", "a"])
    with pytest.raises(ValueError, match="no raw"):
        tg.rank_genes_groups(ad, "ct", use_raw=True)
    with pytest.raises(ValueError, match="layer"):
        tg.rank_genes_groups(ad, "ct", layer="counts", use_raw=True)
    with pytest.raises(ValueError, match="not in adata.layers"):
        tg.rank_genes_groups(ad, "ct", layer="counts")
    for m in ("wilcoxon", "logreg"):
        with pytest.raises(NotImplementedError, match=m):
            tg.rank_genes_groups(ad, "ct", method=m)
    with pytest.raises(ValueError, match="method='t-test_foo'"):
        tg.rank_genes_groups(ad, "ct", method="t-test_foo")
    with pytest.raises(ValueError, match="corr_method='holm'"):
        tg.rank_genes_groups(ad, "ct", corr_method="holm")
    assert set(ad.uns) == {"rank_genes_groups"} and list(ad.uns["rank_genes_groups"]["names"].dtype.names) == ["a", "solo"]


def test_ctg_is_the_unique_top_names():
    X, lab = expression(N=400, G=260, seed=9)
    ad = adata_of(sp.csr_matrix(X), lab, categorical=True)
    got = tg.ctg(ad, "ct")
    tops = set()
    for g in "abcd":
        sc = restate(X, lab, g)[0]
        tops |= set(np.asarray(ad.var_names)[np.argsort(-sc, kind="stable")[:150]])
    assert got == sorted(tops) and len(got) > 150
    assert ad.uns["rank_genes_groups"]["params"]["use_raw"] is False
    assert tg.ctg(ad, "ct", n_top=3) == sorted({n for g in "abcd" for n in ad.uns["rank_genes_groups"]["names"][g][:3]})


def test_tutorial_flow_into_pp_adatas():
    """rank_genes_groups -> the top 100 markers of each group -> pp_adatas(genes=markers), as in the tutorials."""
    X, lab = expression(N=300, G=160, seed=10)
    ad_sc = adata_of(sp.csr_matrix(X), lab, categorical=True)
    ad_sc.var.index = [f"Gene{k}" for k in range(X.shape[1])]
    rng = np.random.default_rng(11)
    sp_genes = [f"Gene{k}" for k in range(0, 160, 2)] + ["Other"]
    ad_sp = MiniAnnData(X=rng.random((20, len(sp_genes))).astype(np.float32), var=pd.DataFrame(index=sp_genes))
    tg.rank_genes_groups(ad_sc, groupby="ct", use_raw=False)
    markers = list(np.unique(pd.DataFrame(ad_sc.uns["rank_genes_groups"]["names"]).iloc[0:100, :].melt().value.values))
    tg.pp_adatas(ad_sc, ad_sp, genes=markers)
    expect = {m.lower() for m in markers} & {g.lower() for g in sp_genes}
    assert sorted(ad_sc.uns["training_genes"]) == sorted(expect) and len(expect) > 0


def test_group_stats_refusals_without_patch(monkeypatch):
    monkeypatch.undo()
    gs = gene_selection.group_stats
    assert gs is not group_stats_f64
    with pytest.raises(ValueError, match="shape"):
        gs(np.ones((3, 2), np.float32), [0, 0], 1)
    with pytest.raises(ValueError, match=r"labels must lie in \[-1, 2\)"):
        gs(np.ones((3, 2), np.float32), [0, 2, 1], 2)
    with pytest.raises(ValueError, match="n_labels=0"):
        gs(np.ones((3, 2), np.float32), [0, 0, 0], 0)
    with pytest.raises(ValueError, match="malformed CSR|column index"):
        bad = sp.csr_matrix((np.ones(2, np.float32), np.array([0, 5]), np.array([0, 1, 2, 2])), shape=(3, 2))
        gs(bad, [0, 0, 0], 1)
    if not _has_gpu():
        with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
            gs(np.ones((3, 2), np.float32), [0, 0, -1], 1)


def test_entry_point_checks_arguments():
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    lab = np.array([0, 1, -1, 2], dtype=np.int32)
    s, q, n = np.empty((3, 4)), np.empty((3, 4)), np.empty((3, 4), np.int64)
    out = (_lib.ptr(s), _lib.ptr(q), _lib.ptr(n))

    def call(X=fake, x_ld=4, indptr=None, rows=4, n_genes=4, labels=lab, T=3, outs=out, block=0):
        return lib.tgb200_group_stats(X, x_ld, indptr, None, None, 0, rows, n_genes, _lib.ptr(labels), T, *outs, block,
                                      0, None)
    assert call(X=None) == -1 and b"exactly one of X" in lib.tgb200_last_error()
    assert call(indptr=fake) == -1 and b"exactly one of X" in lib.tgb200_last_error()
    assert call(x_ld=3) == -1 and b"bad shape" in lib.tgb200_last_error()
    assert call(rows=0) == -1 and b"bad shape" in lib.tgb200_last_error()
    assert call(outs=(None, _lib.ptr(q), None)) == -1 and b"null argument" in lib.tgb200_last_error()
    assert call(T=0) == -1 and b"n_labels=0" in lib.tgb200_last_error()
    assert call(block=1024) == -1 and b"block_rows=1024 is not a multiple of 2048" in lib.tgb200_last_error()
    assert call(T=2) == -1 and b"label 2 of row 3 is outside [-1, 2)" in lib.tgb200_last_error()
    assert call(labels=np.array([0, -2, 0, 0], np.int32)) == -1 and b"label -2 of row 1" in lib.tgb200_last_error()
    if not _has_gpu():
        assert call() == -5 and b"no CPU fallback" in lib.tgb200_last_error()
