"""tgb200_group_stats and rank_genes_groups on the H100.

* the per-label sums and sums of squares within 1e-12 of float64 numpy, the nonzero counts exact: rows not a multiple of
  2048, genes not a multiple of 4 or 1024, a row stride beyond the genes, empty rows, explicit zeros, unsorted and
  duplicate CSR (canonicalised on a copy), a label in one range only, labels without rows, every row unlabelled, a single
  label, NaN, and a strided CUDA tensor;
* identical bits for dense and CSR, host and device data, block_rows 2048, 6144 and the default, and a re-run;
* every invalid input returns its status, and the library stays usable;
* rank_genes_groups on the device equals the float64 host stand-in run on dense, CSR and CUDA-tensor X, and one run at
  50k cells x 2k genes x 40 labels equals the scipy restatement.
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
from tests.test_rank_genes import group_stats_f64, restate  # noqa: E402

DEV = torch.cuda.current_device()


def f64_stats(X, labels, T):
    """Per-label float64 sums, sums of squares and nonzero counts through a one-hot product (labels -1 left out)."""
    X = sp.csr_matrix(X, dtype=np.float64) if sp.issparse(X) else sp.csr_matrix(np.asarray(X, dtype=np.float64))
    lab = np.asarray(labels)
    keep = lab >= 0
    H = sp.csr_matrix((np.ones(keep.sum()), (lab[keep], np.nonzero(keep)[0])), shape=(T, X.shape[0]))
    nz = X.copy()
    nz.data = (nz.data != 0).astype(np.float64)
    sq = X.multiply(X).tocsr()
    return (np.asarray((H @ X).todense()), np.asarray((H @ sq).todense()),
            np.rint(np.asarray((H @ nz).todense())).astype(np.int64))


def check(got, want):
    s, q, n = got
    ws, wq, wn = want
    for a, b in ((s, ws), (q, wq)):
        scale = np.abs(b).max() if b.size else 1.0
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12 * max(scale, 1.0))
    np.testing.assert_array_equal(n, wn)


def bits(got):
    return tuple(np.ascontiguousarray(a).view(np.uint8).tobytes() for a in got)


def raw_call(labels, T, *, X=None, x_ld=0, csr=None, rows=None, n_genes=None, block=0, out=None):
    """tgb200_group_stats on numpy arrays or torch tensors (host or device) -> (status, (sum, sumsq, nnz))."""
    lab = np.ascontiguousarray(labels, dtype=np.int32)
    rows = len(lab) if rows is None else rows
    G = n_genes
    s, q, n = out if out is not None else (np.zeros((T, G)), np.zeros((T, G)), np.zeros((T, G), np.int64))
    if csr is not None:
        ip, ix, dv = csr
        x = (None, 0, _lib.ptr(ip), _lib.ptr(ix), _lib.ptr(dv), int(ix.shape[0]))
    else:
        x = (_lib.ptr(X), x_ld, None, None, None, 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)
    st = _lib.load().tgb200_group_stats(*x, rows, G, _lib.ptr(lab), T, _lib.ptr(s), _lib.ptr(q), _lib.ptr(n), block, DEV,
                                        stream)
    if out is not None:
        torch.cuda.synchronize()
        s, q, n = (a.cpu().numpy() for a in out)
    return st, (s, q, n)


def sample(N, G, T, seed, density=0.3, unlabelled=0.1):
    rng = np.random.default_rng(seed)
    X = (rng.gamma(1.2, 1.5, (N, G)) * (rng.random((N, G)) < density)).astype(np.float32)
    lab = rng.integers(0, T, N).astype(np.int32)
    lab[rng.random(N) < unlabelled] = -1
    return X, lab


def test_against_float64_awkward_shapes():
    X, lab = sample(5000, 1030, 7, seed=1)
    X[17] = 0.0                                              # an empty row
    lab[lab == 5] = 2                                        # label 5 without rows
    lab[2048:4096][lab[2048:4096] == 1] = 6                  # label 6 in ...
    lab[:2048][lab[:2048] == 6] = 0                          # ... the second range only
    lab[4096:][lab[4096:] == 6] = 0
    want = f64_stats(X, lab, 7)
    check(gene_selection.group_stats(X, lab, 7), want)
    check(gene_selection.group_stats(sp.csr_matrix(X), lab, 7), want)
    Xw = np.zeros((5000, 1035), np.float32)                  # host rows with a stride beyond the genes
    Xw[:, :1030] = X
    st, got = raw_call(lab, 7, X=Xw, x_ld=1035, n_genes=1030)
    assert st == 0
    check(got, want)
    assert np.all(got[0][5] == 0) and np.all(got[2][5] == 0)


def test_explicit_zeros_unsorted_and_duplicate_csr():
    rng = np.random.default_rng(2)
    N, G = 3000, 70
    rows = rng.integers(0, N, 20000)
    cols = rng.integers(0, G, 20000)
    vals = rng.standard_normal(20000).astype(np.float32)
    vals[::9] = 0.0                                           # explicit zeros
    indptr = np.r_[0, np.cumsum(np.bincount(rows, minlength=N))]
    order = np.argsort(rows, kind="stable")
    csr = sp.csr_matrix((vals[order], cols[order], indptr), shape=(N, G))          # unsorted, with repeats
    before = (csr.indptr.copy(), csr.indices.copy(), csr.data.copy())
    lab = rng.integers(-1, 4, N).astype(np.int32)
    got = gene_selection.group_stats(csr, lab, 4)
    for a, b in zip(before, (csr.indptr, csr.indices, csr.data)):
        np.testing.assert_array_equal(a, b)                  # the input is canonicalised on a copy
    dense = csr.toarray()
    check(got, f64_stats(dense, lab, 4))
    assert bits(got) == bits(gene_selection.group_stats(dense, lab, 4))


def test_degenerate_labels_and_nan():
    X, _ = sample(2500, 40, 1, seed=3)
    none = np.full(2500, -1, np.int32)
    s, q, n = gene_selection.group_stats(X, none, 3)
    assert not s.any() and not q.any() and not n.any()
    one = np.zeros(2500, np.int32)
    check(gene_selection.group_stats(sp.csr_matrix(X), one, 1), f64_stats(X, one, 1))
    X[100, 3] = np.nan
    lab = (np.arange(2500) % 2).astype(np.int32)
    s, q, n = gene_selection.group_stats(X, lab, 2)
    assert np.isnan(s[0, 3]) and np.isnan(q[0, 3]) and not np.isnan(s[1]).any()
    assert n[0, 3] == (X[lab == 0, 3] != 0).sum()            # NaN counts as nonzero
    ok = np.ones(40, bool)
    ok[3] = False
    check(tuple(a[:, ok] for a in (s, q, n)), tuple(a[:, ok] for a in f64_stats(X, lab, 2)))


def test_strided_cuda_tensor():
    X, lab = sample(4100, 300, 5, seed=4)
    big = torch.zeros((4100, 333), dtype=torch.float32, device=DEV)
    big[:, 10:310] = torch.from_numpy(X).to(DEV)
    view = big[:, 10:310]                                     # row stride 333, not 16-byte aligned
    got = gene_selection.group_stats(view, lab, 5)
    check(got, f64_stats(X, lab, 5))
    assert bits(got) == bits(gene_selection.group_stats(X, lab, 5))


def test_bits_identical_however_staged():
    X, lab = sample(9000, 1100, 9, seed=5, density=0.2)
    csr = sp.csr_matrix(X)
    ip, ix, dv = csr.indptr.astype(np.int64), csr.indices.astype(np.int32), csr.data.astype(np.float32)
    dip, dix, ddv = (torch.from_numpy(a).to(DEV) for a in (ip, ix, dv))
    dX = torch.from_numpy(X).to(DEV)
    ref = None
    for block in (2048, 6144, 0):
        runs = [raw_call(lab, 9, X=X, x_ld=1100, n_genes=1100, block=block),
                raw_call(lab, 9, X=dX, x_ld=1100, n_genes=1100, block=block),
                raw_call(lab, 9, csr=(ip, ix, dv), n_genes=1100, block=block),
                raw_call(lab, 9, csr=(dip, dix, ddv), n_genes=1100, block=block)]
        dev_out = tuple(torch.empty((9, 1100), dtype=d, device=DEV) for d in (torch.float64, torch.float64, torch.int64))
        runs.append(raw_call(lab, 9, csr=(ip, ix, dv), n_genes=1100, block=block, out=dev_out))
        for st, got in runs:
            assert st == 0, _lib.load().tgb200_last_error()
            ref = ref or bits(got)
            assert bits(got) == ref
    check(raw_call(lab, 9, X=X, x_ld=1100, n_genes=1100)[1], f64_stats(X, lab, 9))


def test_invalid_input_keeps_library_usable():
    lib = _lib.load()
    X, lab = sample(3000, 20, 3, seed=6)
    csr = sp.csr_matrix(X)
    ip, ix, dv = csr.indptr.astype(np.int64), csr.indices.astype(np.int32), csr.data.copy()

    def bad(expect, **kw):
        st, _ = raw_call(kw.pop("labels", lab), 3, n_genes=20, **kw)
        assert st == -1, st
        assert expect in lib.tgb200_last_error()
    bad(b"indptr runs from", csr=(ip + 1, ix, dv))
    ip2 = ip.copy()
    ip2[5] = ip2[7]
    bad(b"indptr decreases", csr=(ip2, ix, dv))
    ix2 = ix.copy()
    ix2[3] = 20
    bad(b"outside [0, 20)", csr=(ip, ix2, dv))
    r = int(np.nonzero(np.diff(ip) >= 2)[0][0])
    ix3 = ix.copy()
    ix3[ip[r]], ix3[ip[r] + 1] = ix3[ip[r] + 1], ix3[ip[r]]
    bad(b"not strictly increasing", csr=(torch.from_numpy(ip).to(DEV), torch.from_numpy(ix3).to(DEV),
                                         torch.from_numpy(dv).to(DEV)))
    lab2 = lab.copy()
    lab2[2999] = 3
    bad(b"label 3 of row 2999", X=X, x_ld=20, labels=lab2)
    bad(b"not a multiple of 2048", X=X, x_ld=20, block=3000)
    st, _ = raw_call(lab, 3, X=X, x_ld=19, n_genes=20)
    assert st == -1 and b"bad shape" in lib.tgb200_last_error()
    # 2^20 labels x 2^20 genes of output cannot fit: refused before anything is read or written
    st = lib.tgb200_group_stats(_lib.ptr(X), 1 << 20, None, None, None, 0, 3000, 1 << 20,
                                _lib.ptr(np.zeros(3000, np.int32)), 1 << 20, ctypes.c_void_p(8), ctypes.c_void_p(8),
                                None, 0, DEV, None)
    assert st == -1 and b"GiB are free" in lib.tgb200_last_error()
    st, got = raw_call(lab, 3, csr=(ip, ix, dv), n_genes=20)
    assert st == 0
    check(got, f64_stats(X, lab, 3))


def separated(N, G, seed):
    """Groups with their own marker genes, so scores are well apart (names compare exactly)."""
    rng = np.random.default_rng(seed)
    lab = np.array(list("pqrst"))[rng.integers(0, 5, N)]
    X = rng.gamma(1.0, 1.0, (N, G)) * (rng.random((N, G)) < 0.4) + np.linspace(0, 0.5, G)
    for k, g in enumerate("pqrst"):
        X[lab == g, 4 * k:4 * k + 4] += 1.0 + 0.7 * k + np.arange(4) * 0.31
    return np.log1p(X).astype(np.float32), lab


@pytest.mark.parametrize("kind", ["dense", "csr", "cuda"])
def test_rank_genes_groups_matches_host_stand_in(kind, monkeypatch):
    X, lab = separated(6000, 90, seed=7)
    Xin = {"dense": X, "csr": sp.csr_matrix(X), "cuda": torch.from_numpy(X).to(DEV)}[kind]
    obs = pd.DataFrame({"ct": pd.Categorical(lab)}, index=[f"c{i}" for i in range(len(lab))])
    var = pd.DataFrame(index=[f"G{k}" for k in range(X.shape[1])])
    ad = MiniAnnData(X=Xin, obs=obs, var=var)
    tg.rank_genes_groups(ad, "ct", pts=True)
    with monkeypatch.context() as m:
        m.setattr(gene_selection, "group_stats", group_stats_f64)
        ad_h = MiniAnnData(X=X, obs=obs, var=var)
        tg.rank_genes_groups(ad_h, "ct", pts=True)
    g, h = ad.uns["rank_genes_groups"], ad_h.uns["rank_genes_groups"]
    for grp in "pqrst":
        assert list(g["names"][grp]) == list(h["names"][grp])
        np.testing.assert_allclose(g["scores"][grp], h["scores"][grp], rtol=1e-6)       # float32 outputs
        np.testing.assert_allclose(g["pvals"][grp], h["pvals"][grp], rtol=1e-8, atol=1e-300)
    pd.testing.assert_frame_equal(g["pts"], h["pts"])
    # the statistics the float64 scores are computed from
    codes = pd.Categorical(lab).codes
    check(gene_selection.group_stats(Xin, codes, 5), group_stats_f64(X, codes, 5))


def test_larger_sample_against_restatement():
    rng = np.random.default_rng(8)
    N, G, T = 50000, 2000, 40
    X = sp.random(N, G, density=0.08, format="csr", dtype=np.float32, random_state=rng, data_rvs=lambda k:
                  np.log1p(rng.gamma(1.5, 2.0, k)).astype(np.float32))
    lab = rng.integers(0, T, N)
    for t in range(T):                                        # a marker block per label
        rows = np.nonzero(lab == t)[0]
        X = X + sp.csr_matrix((np.full(len(rows), 1.0 + 0.05 * t, np.float32), (rows, np.full(len(rows), 7 * t))),
                              shape=(N, G))
    X = X.tocsr().astype(np.float32)
    check(gene_selection.group_stats(X, lab, T), f64_stats(X, lab, T))
    names = [f"t{t:02d}" for t in range(T)]
    obs = pd.DataFrame({"ct": pd.Categorical(np.array(names)[lab], categories=names)},
                       index=[f"c{i}" for i in range(N)])
    ad = MiniAnnData(X=X, obs=obs, var=pd.DataFrame(index=[f"G{k}" for k in range(G)]))
    tg.rank_genes_groups(ad, "ct", n_genes=50)
    uns = ad.uns["rank_genes_groups"]
    dense = X.toarray()
    labels = np.array(names, dtype=object)[lab]
    for t in (0, 17, 39):
        sc, p, adj, lfc = restate(dense, labels, names[t])
        top = np.argsort(-sc, kind="stable")[:50]
        np.testing.assert_allclose(uns["scores"][names[t]], sc[top].astype(np.float32), rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(uns["pvals_adj"][names[t]], adj[top], rtol=1e-6, atol=1e-300)
        assert uns["names"][names[t]][0] == f"G{7 * t}"
