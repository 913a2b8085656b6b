"""`project` / tgb200_project_map on the H100: mapping^T X against float64, bit-identical however the data is staged, and
project_genes on a released mapper with a CSR that must not be densified.

Error bound (u = 2^-24, the fp32 unit roundoff), for mapping entries >= 0 and scale = mapping^T |X|:
  * both operands are split into three bf16 planes that reconstruct them to 2^-26 relative, and the three dropped
    partial products (m,l) (l,m) (l,l) are below 2^-26 |a||b|: 4 u;
  * one chain of c <= 512 cells runs its six partial products into one truncating fp32 accumulator, one wgmma add of up
    to one ulp (2 u) per 16 cells and product: 2 (6 ceil(c / 16) + 16) u;
  * the ceil(N / 512) chains are added in fp32, round-to-nearest: one u each.
  |err| <= (4 + 2 (6 ceil(c / 16) + 16) + chains) u scale elementwise, as tests/test_stages_gpu.py derives it for the
  forward contraction; rel-Frobenius <= 3e-6, the bound tgb200_project is held to."""
import ctypes
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

from tests.helpers import GOLDEN_DIR, rel_fro

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _mapping(N, V, seed):
    rng = np.random.default_rng(seed)
    M = rng.standard_normal((N, V)).astype(np.float32)
    M = np.exp(M - M.max(axis=1, keepdims=True))
    return (M / M.sum(axis=1, keepdims=True)).astype(np.float32)


def _csr(N, K, density, seed):
    rng = np.random.default_rng(seed)
    X = sp.random(N, K, density=density, format="csr", dtype=np.float32, random_state=rng)
    X.data *= 10.0
    return X


def _check(got, M, X):
    M64 = M.astype(np.float64)
    Xd = X.toarray() if sp.issparse(X) else np.asarray(X)
    ref = M64.T @ Xd.astype(np.float64)
    scale = M64.T @ np.abs(Xd).astype(np.float64)
    N = M.shape[0]
    c = min(N, 512)
    bound = (4 + 2 * (6 * -(-c // 16) + 16) + -(-N // 512)) * U * scale
    err = np.abs(got.astype(np.float64) - ref)
    assert (err <= bound).all(), f"max err / bound {float((err / np.where(bound > 0, bound, 1)).max()):.3g}"
    if np.linalg.norm(ref) > 0:
        assert rel_fro(got, ref) <= 3e-6


SHAPES = [
    (1, 5, 7),               # one cell
    (1000, 333, 63),         # two chains, the second one ragged
    (2048, 333, 2048 + 77),  # exactly one block; gene columns past one 2048-wide tile
    (5000, 5, 2048 + 77),    # three blocks, ten chains, the last one ragged
    (5000, 333, 63),
    (600, 65600, 7),         # more than 65535 spots
]


@pytest.mark.parametrize("N,V,K", SHAPES)
def test_project_matches_float64(N, V, K):
    from tangram_b200 import utils
    M = _mapping(N, V, seed=N + V)
    X = _csr(N, K, 0.1, seed=K)
    got = utils.project(M, X)
    assert got.shape == (V, K) and got.dtype == np.float32
    _check(got, M, X)
    Xd = np.random.default_rng(1).random((N, K)).astype(np.float32)      # dense, every entry nonzero
    _check(utils.project(M, Xd), M, Xd)


def _raw(M, X_csr, out, block=0, dense=None):
    """tgb200_project_map on torch tensors (host or device) -> status."""
    import torch
    from tangram_b200 import _lib
    lib = _lib.load()
    p = lambda t: None if t is None else _lib._P(t.data_ptr())   # noqa: E731
    dev = torch.cuda.current_device()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    N, V = M.shape
    if dense is not None:
        x = (p(dense), dense.stride(0), None, None, None, 0, dense.shape[1])
    else:
        indptr, indices, data, K = X_csr
        x = (None, 0, p(indptr), p(indices), p(data), indices.shape[0], K)
    return lib.tgb200_project_map(p(M), N, V, M.stride(0), *x, p(out), block, dev, stream)


def test_staging_does_not_change_a_bit():
    import torch
    from tangram_b200 import utils
    N, V, K = 5000, 333, 2048 + 77
    M = _mapping(N, V, seed=3)
    X = _csr(N, K, 0.07, seed=4)
    ref = utils.project(M, X)
    _check(ref, M, X)
    Xd = X.toarray()
    assert np.array_equal(utils.project(M, Xd), ref), "dense X"
    pad = torch.zeros((N, V + 13), dtype=torch.float32, device="cuda")
    pad[:, :V] = torch.from_numpy(M)
    Mv = pad[:, :V]
    assert Mv.stride(0) == V + 13
    assert np.array_equal(utils.project(Mv, X), ref), "device mapping with a padded row stride"
    assert np.array_equal(utils.project(M, torch.from_numpy(Xd).cuda()), ref), "dense X on the device"
    for block in (4096, 6144):                      # the default at 5000 cells is one block of 2048
        assert np.array_equal(utils.project(M, X, _block_rows=block), ref), f"CSR in blocks of {block} cells"
    assert np.array_equal(utils.project(M, Xd, _block_rows=4096), ref), "dense X in blocks of 4096 cells"
    assert np.array_equal(utils.project(M, X), ref), "a second call"
    # device CSR, device out; host CSR, host out, through the C entry point
    indptr, indices, data, _ = utils._canonical_csr(X, N)
    host = [torch.from_numpy(a) for a in (indptr, indices, data)]
    dev = [t.cuda() for t in host]
    out_d = torch.empty((V, K), dtype=torch.float32, device="cuda")
    assert _raw(Mv, (*dev, K), out_d, block=2048) == 0
    assert np.array_equal(out_d.cpu().numpy(), ref), "device CSR, device out"
    out_h = torch.empty((V, K), dtype=torch.float32)
    assert _raw(torch.from_numpy(M), (*host, K), out_h) == 0
    assert np.array_equal(out_h.numpy(), ref), "host CSR, host out"


@pytest.mark.parametrize("precision,chunks", [("fp32", None), ("bf16x3", None), ("bf16", None), ("bf16", "2")])
def test_mapper_project_equals_project_of_its_mapping(precision, chunks, monkeypatch):
    """Mapper.project (tgb200_project: the row pass writes each block's planes from M) is `project` of the mapping
    get_mapping returns, bit for bit, after training steps: three 2048-cell blocks, the last one ragged, V ragged, more
    than 2048 genes, into host and device out.  bf16 with two cell chunks projects while P holds the update's state."""
    import torch
    from oracle.tangram_oracle import synthetic_inputs
    from tangram_b200 import Mapper, utils
    if chunks:
        monkeypatch.setenv("TGB200_CHUNKS", chunks)
    N, V, K = 6000, 333, 40
    inp = synthetic_inputs(N, V, K, seed=21)
    M0 = np.random.default_rng(22).standard_normal((N, V)).astype(np.float32)
    m = Mapper(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, M0=M0, precision=precision, device="cuda:0")
    if chunks:
        assert int(m._engine.debug("shape")[4]) == int(chunks)
    m.train(3, print_each=None)
    P = m._engine.get_mapping(np.empty((N, V), dtype=np.float32))
    X = np.random.default_rng(23).random((N, 2048 + 77)).astype(np.float32)
    ref = utils.project(P, X)
    _check(ref, P, X)
    assert np.array_equal(m.project(X), ref), "host out"
    out = torch.empty((V, X.shape[1]), dtype=torch.float32, device="cuda:0")
    m.project(X, out=out)
    assert np.array_equal(out.cpu().numpy(), ref), "device out"


def test_default_blocks_larger_than_2048_equal_forced_2048():
    """20000 cells: the default block is 4096 cells (five blocks); forced 2048-cell blocks (ten) give the same bits."""
    from tangram_b200 import utils
    N, V, K = 20000, 64, 100
    M = _mapping(N, V, 11)
    X = _csr(N, K, 0.1, seed=12)
    ref = utils.project(M, X)
    _check(ref, M, X)
    assert np.array_equal(utils.project(M, X, _block_rows=2048), ref)


def test_all_rows_empty_gives_zeros():
    from tangram_b200 import utils
    N, V, K = 3000, 70, 90
    got = utils.project(_mapping(N, V, 1), sp.csr_matrix((N, K), dtype=np.float32))
    assert got.shape == (V, K) and not got.any()


def test_malformed_device_csr_is_refused_and_the_device_stays_usable():
    """Column indices past n_genes, negative or repeated within a row reach the kernel (device pointers, so nothing checks
    them on the host): the call returns TGB200_ERR_INVALID, writes nothing out of bounds, and the next call succeeds."""
    import torch
    from tangram_b200 import _lib, utils
    N, V, K = 2100, 40, 30
    M = _mapping(N, V, 7)
    X = _csr(N, K, 0.2, seed=8)
    indptr, indices, data, _ = utils._canonical_csr(X, N)
    lib = _lib.load()
    Md = torch.from_numpy(M).cuda()
    out = torch.empty((V, K), dtype=torch.float32, device="cuda")
    row = int(np.argmax(np.diff(indptr) >= 2))
    for what, bad in (("past n_genes", lambda i: i.__setitem__(indptr[row + 1] - 1, K + 1000)),
                      ("negative", lambda i: i.__setitem__(indptr[row], -5)),
                      ("repeated", lambda i: i.__setitem__(indptr[row] + 1, i[indptr[row]]))):
        idx = indices.copy()
        bad(idx)
        dev = [torch.from_numpy(a).cuda() for a in (indptr, idx, data)]
        assert _raw(Md, (*dev, K), out) == -1, what
        assert b"column index" in lib.tgb200_last_error()
    dev = [torch.from_numpy(a).cuda() for a in (indptr, indices, data)]
    assert _raw(Md, (*dev, K), out) == 0
    assert np.array_equal(out.cpu().numpy(), utils.project(M, X))
    bad_ptr = indptr.copy()
    bad_ptr[5] = bad_ptr[6] + 1
    dev = [torch.from_numpy(a).cuda() for a in (bad_ptr, indices, data)]
    assert _raw(Md, (*dev, K), out) == -1 and b"indptr" in lib.tgb200_last_error()


class _NoDense(sp.csr_matrix):
    def toarray(self, *a, **k):
        raise AssertionError("adata_sc.X was densified")

    def todense(self, *a, **k):
        raise AssertionError("adata_sc.X was densified")


def test_project_genes_streams_the_reference_csr(monkeypatch):
    """The reference's 5000-cell CSR (17 % dense) onto 9852 spots through a released mapper: the device path equals
    float64 within the bound, never densifies adata_sc.X, and returns the host path's AnnData."""
    import tangram_b200 as tg
    from tangram_b200 import utils
    z = np.load(os.path.join(GOLDEN_DIR, "c1_reference.npz"))
    S0 = sp.csr_matrix((z["S_data"], z["S_indices"], z["S_indptr"]), shape=tuple(z["S_shape"]))
    G = z["G"]
    N, K = S0.shape
    genes = [f"Gene{k}" for k in range(K)]
    ad_sc = tg.MiniAnnData(X=S0.copy(), obs=pd.DataFrame(index=[f"c{i}" for i in range(N)]), var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=G.copy(), obs=pd.DataFrame(index=[f"s{j}" for j in range(G.shape[0])]),
                           var=pd.DataFrame(index=list(genes)))
    tg.pp_adatas(ad_sc, ad_sp)
    ad_map = tg.map_cells_to_space(ad_sc, ad_sp, device="cuda:0", num_epochs=5, random_state=1, verbose=False)
    assert not hasattr(ad_map, "_tgb200_mapper")
    S = sp.csr_matrix(ad_sc.X)                       # the genes pp_adatas kept
    X = _NoDense(S)
    ad_sc.X = X
    ge = tg.project_genes(ad_map, ad_sc)
    assert ad_sc.X is X and sp.issparse(ad_sc.X)
    keep = np.asarray((S != 0).sum(axis=0)).reshape(-1) >= 1
    _check(ge.X, ad_map.X, S[:, keep])
    monkeypatch.setattr(utils, "_sm90_device", lambda mapping: None)
    ad_sc.X = S.copy()
    host = tg.project_genes(ad_map, ad_sc)
    assert rel_fro(ge.X, host.X) < 3e-6
    pd.testing.assert_frame_equal(ge.obs, host.obs)
    pd.testing.assert_frame_equal(ge.var, host.var)
    assert ge.uns is host.uns


def test_fullsize_host_inputs_multi_block():
    """100k x 10k mapping and a 100k x 20k CSR at 7 % on the host: seven cell blocks; float64 on a voxel sample."""
    import torch
    from tangram_b200 import utils
    N, V, K = 100_000, 10_000, 20_000
    g = torch.Generator(device="cuda").manual_seed(0)
    M = torch.rand((N, V), generator=g, device="cuda")
    M /= M.sum(dim=1, keepdim=True)
    Mh = M.cpu().numpy()
    del M
    parts_i, parts_v, counts = [], [], []
    for r0 in range(0, N, 10_000):
        mask = torch.rand((10_000, K), generator=g, device="cuda") < 0.07
        rc = mask.nonzero()
        counts.append(torch.bincount(rc[:, 0], minlength=10_000).cpu())
        parts_i.append(rc[:, 1].int().cpu())
        parts_v.append(torch.rand(rc.shape[0], generator=g, device="cuda").cpu())
        del mask, rc
    torch.cuda.empty_cache()
    indptr = np.concatenate([[0], np.cumsum(torch.cat(counts).numpy())]).astype(np.int64)
    X = sp.csr_matrix((torch.cat(parts_v).numpy(), torch.cat(parts_i).numpy(), indptr), shape=(N, K))
    assert 0.065 < X.nnz / (N * K) < 0.075
    got = utils.project(Mh, X)
    rng = np.random.default_rng(0)
    js, ks = np.sort(rng.choice(V, 48, replace=False)), np.sort(rng.choice(K, 48, replace=False))
    Ms = Mh[:, js].astype(np.float64)
    Xs = X[:, ks].toarray().astype(np.float64)
    ref = Ms.T @ Xs
    err = rel_fro(got[np.ix_(js, ks)], ref)
    print(f"project {N}x{V} onto {K} genes (CSR, {X.nnz / (N * K):.3f} dense): rel err vs float64 {err:.2e}")
    assert err <= 1e-5
    bound = (4 + 2 * (6 * 32 + 16) + -(-N // 512)) * U * ref        # X >= 0: scale = ref
    assert (np.abs(got[np.ix_(js, ks)] - ref) <= bound).all()
