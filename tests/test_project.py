"""`project` without a GPU: malformed input is refused on the host before any device call, sparse inputs of every
layout are canonicalised to what toarray() holds without touching the caller's matrix, the C entry point checks its
arguments, and without a GPU `project` refuses while project_genes keeps its host GEMM."""
import ctypes

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp


def _has_gpu():
    import torch
    return torch.cuda.is_available()


@pytest.fixture
def no_device_calls(monkeypatch):
    """Any attempt to pick a device or load the library fails the test."""
    from tangram_b200 import _lib, utils

    def boom(*a, **k):
        raise AssertionError("device call before the arguments were checked")
    monkeypatch.setattr(utils, "_require_device", boom)
    monkeypatch.setattr(_lib, "load", boom)


def test_public_name():
    import tangram_b200 as tg
    from tangram_b200 import utils
    assert tg.project is utils.project


def _csr(seed=0, shape=(6, 5)):
    rng = np.random.default_rng(seed)
    A = rng.random(shape) * (rng.random(shape) < 0.5)
    return sp.csr_matrix(A.astype(np.float32))


@pytest.mark.parametrize("case", ["dense_rows", "sparse_rows", "indptr_decreasing", "indptr_end", "indptr_start",
                                  "indptr_length", "index_high", "index_negative", "mapping_1d"])
def test_malformed_input_is_refused_on_the_host(case, no_device_calls):
    from tangram_b200 import utils
    M = np.full((6, 3), 1 / 3, dtype=np.float32)
    X = _csr()
    if case == "dense_rows":
        X = np.ones((5, 4), np.float32)
    elif case == "sparse_rows":
        X = _csr(shape=(7, 5))
    elif case == "indptr_decreasing":
        X.indptr[2], X.indptr[3] = X.indptr[3] + 1, X.indptr[2]
    elif case == "indptr_end":
        X.indptr[-1] -= 1
    elif case == "indptr_start":
        X.indptr[0] = 1
    elif case == "indptr_length":
        X.indptr = X.indptr[:-1]
    elif case == "index_high":
        X.indices[-1] = 5
    elif case == "index_negative":
        X.indices[0] = -1
    elif case == "mapping_1d":
        M = M[:, 0]
    with pytest.raises(ValueError):
        utils.project(M, X)


def _messy(kind):
    """-> (a sparse matrix in layout `kind`, the dense float32 matrix toarray() gives for it)."""
    rng = np.random.default_rng(3)
    if kind == "csc":
        m = sp.csc_matrix(rng.random((7, 9)) * (rng.random((7, 9)) < 0.4))
    elif kind == "coo":                                                     # duplicates summed by tocsr
        m = sp.coo_matrix((np.array([1.0, 2.0, 0.5, 4.0]), (np.array([0, 0, 3, 6]), np.array([2, 2, 8, 0]))), shape=(7, 9))
    elif kind == "unsorted":
        m = sp.csr_matrix((np.array([3.0, 1.0, 2.0, 5.0], np.float32), np.array([4, 1, 2, 0]), np.array([0, 3, 3, 4, 4, 4, 4, 4])),
                          shape=(7, 9))
    elif kind == "duplicates":                                              # summed in float64, as toarray() sums
        m = sp.csr_matrix((np.array([0.1, 0.2, 0.7, 1e-9, 1.0]), np.array([3, 3, 5, 5, 8]), np.array([0, 2, 4, 4, 4, 4, 5, 5])),
                          shape=(7, 9))
    elif kind == "explicit_zeros":
        m = sp.csr_matrix((np.array([0.0, 1.5, 0.0], np.float32), np.array([0, 4, 8]), np.array([0, 1, 3, 3, 3, 3, 3, 3])),
                          shape=(7, 9))
    elif kind == "int_data":
        m = sp.csr_matrix(rng.integers(0, 3, (7, 9)))
    return m, m.toarray().astype(np.float32)


@pytest.mark.parametrize("kind", ["csc", "coo", "unsorted", "duplicates", "explicit_zeros", "int_data"])
def test_canonical_csr_equals_toarray_and_leaves_the_input(kind):
    from tangram_b200 import utils
    m, want = _messy(kind)
    ref = m.copy()
    indptr, indices, data, n_genes = utils._canonical_csr(m, 7)
    assert indptr.dtype == np.int64 and indices.dtype == np.int32 and data.dtype == np.float32 and n_genes == 9
    assert indptr[0] == 0 and indptr[-1] == len(indices) == len(data)
    for r in range(7):
        cols = indices[indptr[r]:indptr[r + 1]]
        assert (np.diff(cols) > 0).all()                                    # strictly increasing: sorted, no repeats
    got = sp.csr_matrix((data, indices, indptr), shape=(7, 9)).toarray()
    assert np.array_equal(got, want)
    for a in ("data", "indices", "indptr", "row", "col"):                  # the caller's matrix stays as it was
        if hasattr(ref, a):
            assert np.array_equal(getattr(m, a), getattr(ref, a)), a


def test_canonical_csr_passes_canonical_input_through():
    from tangram_b200 import utils
    X = _csr(5, shape=(50, 40))
    indptr, indices, data, _ = utils._canonical_csr(X, 50)
    assert np.array_equal(indptr, X.indptr) and np.array_equal(indices, X.indices) and np.array_equal(data, X.data)
    assert np.shares_memory(data, X.data) and np.shares_memory(indices, X.indices)     # no copy of the entries


def test_entry_point_checks_arguments():
    from tangram_b200 import _lib
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    ip = np.array([0, 1, 2], dtype=np.int64)
    out = np.empty((3, 4), np.float32)

    def call(map_=fake, rows=2, cols=3, ld=3, X=fake, x_ld=4, indptr=None, nnz=0, n_genes=4, block=0):
        return lib.tgb200_project_map(map_, rows, cols, ld, X, x_ld, indptr, fake if indptr else None,
                                      fake if indptr else None, nnz, n_genes, _lib.ptr(out), block, 0, None)
    assert call(map_=None) == -1
    assert call(ld=2) == -1 and b"bad shape" in lib.tgb200_last_error()
    assert call(x_ld=3) == -1 and b"bad shape" in lib.tgb200_last_error()
    assert call(n_genes=0) == -1
    assert call(indptr=_lib.ptr(ip), nnz=2) == -1 and b"exactly one" in lib.tgb200_last_error()
    assert call(X=None) == -1 and b"exactly one" in lib.tgb200_last_error()
    assert call(X=None, indptr=_lib.ptr(ip), nnz=-1) == -1
    assert call(block=1000) == -1 and b"multiple of 2048" in lib.tgb200_last_error()
    if not _has_gpu():
        assert call() == -5 and b"no CPU fallback" in lib.tgb200_last_error()


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_without_gpu_project_refuses_and_project_genes_stays_on_the_host():
    from tangram_b200 import MiniAnnData, _lib, utils
    rng = np.random.default_rng(1)
    N, V, K = 40, 6, 9
    M = rng.random((N, V)).astype(np.float32)
    M /= M.sum(axis=1, keepdims=True)
    X = sp.csr_matrix((rng.random((N, K)) * (rng.random((N, K)) < 0.3) + np.eye(N, K)).astype(np.float32))
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        utils.project(M, X)
    cells, spots, genes = [f"c{i}" for i in range(N)], [f"s{j}" for j in range(V)], [f"G{k}" for k in range(K)]
    ad_map = MiniAnnData(X=M, obs=pd.DataFrame(index=cells), var=pd.DataFrame(index=spots),
                         uns={"train_genes_df": pd.DataFrame(index=["g1", "g4"])})
    ad_sc = MiniAnnData(X=X, obs=pd.DataFrame(index=cells), var=pd.DataFrame(index=genes), uns={"overlap_genes": ["g1"]})
    ge = utils.project_genes(ad_map, ad_sc)
    assert np.array_equal(ge.X, M.T @ X.toarray())
    assert list(ge.obs.index) == spots and list(ge.var.index) == [g.lower() for g in genes]
    assert list(ge.var["is_training"]) == [k in (1, 4) for k in range(K)]
    assert ge.uns is ad_sc.uns and sp.issparse(ad_sc.X)
