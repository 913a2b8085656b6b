"""spatial_neighbors without a GPU: the Python layer runs with float64 numpy brute-force stand-ins for the device pass
(`_knn`, tgb200_spatial_knn, and `_radius`, tgb200_spatial_radius) and is compared with independent restatements of
squidpy's gr.spatial_neighbors.

* every refusal (ValueError, KeyError / TypeError for library_key, NotImplementedError) and the coord_type choice;
* the grid cut on a jittered hexagonal lattice with holes (boundary spots keep fewer than 6 neighbours), and rings 1-3
  against a breadth-first search over the cut graph;
* set_diag, scalar and interval radius, coincident points (connected, no distance entry);
* three libraries in shuffled obs order, the obsp / uns keys, key_added and copy=True;
* spatial_weights on the result for the three (standardized, self_inclusion) pairs the Mapper's terms use;
* the stand-ins' distance against numpy's np.sqrt(((C[j] - C[i]) ** 2).sum()), bit for bit.
"""
import sys

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp

import tangram_b200 as tg
from tangram_b200 import MiniAnnData
from tangram_b200.spatial_weights import spatial_weights

snb = sys.modules["tangram_b200.spatial_neighbors"]     # the module; tg.spatial_neighbors is the function

CALLS = []


def pair_dist(C, rows):
    """(len(rows), n) distances d(i, j) = sqrt((dx*dx + dy*dy) + dz*dz), dx = C[j] - C[i], each operation rounded."""
    D = C[None, :, :] - C[rows][:, None, :]
    s = D[..., 0] * D[..., 0]
    for a in range(1, C.shape[1]):
        s = s + D[..., a] * D[..., a]
    return np.sqrt(s)


def _blocks(n, size=512):
    for r0 in range(0, n, size):
        yield np.arange(r0, min(n, r0 + size))


def knn_f64(C, k, device=None):
    """The device k-nearest query in float64 numpy: the k nearest j != i ranked by np.lexsort((j, d)), listed by j."""
    CALLS.append(("knn", k))
    C = np.asarray(C, dtype=np.float64)
    n = C.shape[0]
    idx = np.empty((n, k), dtype=np.int32)
    dst = np.empty((n, k))
    for rows in _blocks(n):
        d = pair_dist(C, rows)
        for t, i in enumerate(rows):
            order = np.lexsort((np.arange(n), d[t]))
            order = order[order != i][:k]
            order.sort()
            idx[i], dst[i] = order, d[t, order]
    return idx, dst


def radius_f64(C, r, device=None):
    """The device radius query in float64 numpy: every j != i with d <= r, each row in decreasing j (any search order)."""
    CALLS.append(("radius", r))
    C = np.asarray(C, dtype=np.float64)
    n = C.shape[0]
    indptr, idx, dst = [0], [], []
    for rows in _blocks(n):
        d = pair_dist(C, rows)
        for t, i in enumerate(rows):
            j = np.nonzero(d[t] <= r)[0]
            j = j[j != i][::-1]
            idx.append(j)
            dst.append(d[t, j])
            indptr.append(indptr[-1] + len(j))
    return (np.asarray(indptr, dtype=np.int64), np.concatenate(idx).astype(np.int32), np.concatenate(dst))


@pytest.fixture(autouse=True)
def host_search(monkeypatch):
    monkeypatch.setattr(snb, "_knn", knn_f64)
    monkeypatch.setattr(snb, "_radius", radius_f64)
    CALLS.clear()


def adata_of(C, uns=None, obs=None):
    n = C.shape[0]
    obs = obs if obs is not None else pd.DataFrame(index=[f"s{i}" for i in range(n)])
    return MiniAnnData(X=np.zeros((n, 1), np.float32), obs=obs, uns=uns or {}, obsm={"spatial": C})


def hex_lattice(rows=12, cols=12, jitter=0.02, holes=(), seed=0):
    """Visium-like spots at unit spacing with a little jitter, minus the (row, col) holes -> (coords, lattice index)."""
    rng = np.random.default_rng(seed)
    pts, rc = [], []
    for r in range(rows):
        for c in range(cols):
            if (r, c) in holes:
                continue
            pts.append((c + 0.5 * (r % 2), r * np.sqrt(3) / 2))
            rc.append((r, c))
    C = np.asarray(pts) + rng.uniform(-jitter, jitter, (len(pts), 2))
    return C, rc


def lattice_neighbours(rc):
    """The hexagonal lattice's own adjacency (offset rows) among the present spots, as a set of (i, j)."""
    at = {p: i for i, p in enumerate(rc)}
    out = set()
    for i, (r, c) in enumerate(rc):
        odd = r % 2
        for dr, dc in ((0, -1), (0, 1), (-1, odd - 1), (-1, odd), (1, odd - 1), (1, odd)):
            j = at.get((r + dr, c + dc))
            if j is not None:
                out.add((i, j))
    return out


def entries(m):
    m = m.tocoo()
    return {(int(i), int(j)): float(v) for i, j, v in zip(m.row, m.col, m.data)}


def canonical(m):
    assert sp.isspmatrix_csr(m) and m.dtype == np.float64
    assert m.has_canonical_format
    return True


# ---- refusals and the mode choice ---------------------------------------------------------------------------------------

def test_refusals():
    C = np.random.default_rng(0).random((20, 2))
    ad = adata_of(C)
    for kw, exc, msg in (
            (dict(delaunay=True), NotImplementedError, "delaunay"),
            (dict(percentile=99.0), NotImplementedError, "percentile"),
            (dict(transform="cosine"), NotImplementedError, "transform"),
            (dict(spatial_key="nope"), ValueError, "spatial_key"),
            (dict(n_neighs=0), ValueError, "n_neighs"),
            (dict(n_rings=0), ValueError, "n_rings"),
            (dict(n_neighs=20), ValueError, "n_neighs"),
            (dict(n_neighs=65), ValueError, "n_neighs"),
            (dict(radius=-1.0), ValueError, "radius"),
            (dict(radius=np.inf), ValueError, "radius"),
            (dict(radius=(1.0, 2.0, 3.0)), ValueError, "radius"),
            (dict(coord_type="hex"), ValueError, "coord_type")):
        with pytest.raises(exc, match=msg):
            tg.spatial_neighbors(ad, **kw)
    for bad in (C[:, :1], np.c_[C, C], np.r_[C[:19], [[np.nan, 0.0]]], np.r_[C[:19], [[0.0, np.inf]]]):
        with pytest.raises(ValueError, match="spatial"):
            tg.spatial_neighbors(adata_of(bad))
    obs = pd.DataFrame({"lib": pd.Categorical(["a"] * 14 + ["b"] * 6)}, index=ad.obs.index)
    with pytest.raises(ValueError, match="n_neighs"):             # counted per library: b has 6 points
        tg.spatial_neighbors(adata_of(C, obs=obs), library_key="lib")
    tg.spatial_neighbors(adata_of(C, obs=obs), library_key="lib", n_neighs=5)
    with pytest.raises(KeyError, match="library_key"):
        tg.spatial_neighbors(ad, library_key="lib")
    obs["lib"] = obs["lib"].astype(str)
    with pytest.raises(TypeError, match="categorical"):
        tg.spatial_neighbors(adata_of(C, obs=obs), library_key="lib")
    obs["lib"] = pd.Categorical([None] + ["a"] * 19)
    with pytest.raises(ValueError, match="missing"):
        tg.spatial_neighbors(adata_of(C, obs=obs), library_key="lib")
    assert CALLS[-1] == ("knn", 5) and len(CALLS) == 2             # only the one good call reached the search


def test_coord_type_follows_uns():
    C, _ = hex_lattice(6, 6)
    ad = adata_of(C)
    tg.spatial_neighbors(ad)
    assert ad.uns["spatial_neighbors"]["params"]["coord_type"] == "generic"
    assert sorted(set(ad.obsp["spatial_distances"].data)) != [1.0]
    ad = adata_of(C, uns={"spatial": {}})
    tg.spatial_neighbors(ad)
    assert ad.uns["spatial_neighbors"]["params"]["coord_type"] == "grid"
    assert set(ad.obsp["spatial_distances"].data) == {1.0}
    with pytest.warns(UserWarning, match="radius"):
        tg.spatial_neighbors(ad, radius=5.0, key_added="g")
    assert entries(ad.obsp["g_connectivities"]) == entries(ad.obsp["spatial_connectivities"])


# ---- grid mode --------------------------------------------------------------------------------------------------------

HOLES = ((3, 3), (3, 4), (7, 8), (8, 2))


def test_grid_cut_on_a_hexagonal_lattice_with_holes():
    C, rc = hex_lattice(12, 12, holes=HOLES)
    ad = adata_of(C)
    tg.spatial_neighbors(ad, coord_type="grid")
    A, D = ad.obsp["spatial_connectivities"], ad.obsp["spatial_distances"]
    assert canonical(A) and canonical(D)
    want = lattice_neighbours(rc)
    assert set(entries(A)) == want
    assert set(entries(D)) == want and set(D.data) == {1.0} and set(A.data) == {1.0}
    deg = np.diff(A.indptr)
    assert deg.max() == 6 and (deg < 6).sum() > 40                   # the edges and the spots around the holes
    assert all(deg[rc.index((r, c))] < 6 for r, c in ((3, 2), (2, 3), (4, 4), (8, 1)))


def bfs_rings(A, n_rings):
    """{(i, j): ring} for j != i reachable from i in at most n_rings steps along A's rows."""
    nbrs = [A.indices[A.indptr[i]:A.indptr[i + 1]] for i in range(A.shape[0])]
    out = {}
    for i in range(A.shape[0]):
        seen, front = {i}, [i]
        for ring in range(1, n_rings + 1):
            nxt = []
            for u in front:
                for v in nbrs[u]:
                    if v not in seen:
                        seen.add(v)
                        nxt.append(v)
                        out[(i, int(v))] = float(ring)
            front = nxt
    return out


@pytest.mark.parametrize("n_rings", [1, 2, 3])
@pytest.mark.parametrize("set_diag", [False, True])
def test_grid_rings_against_breadth_first_search(n_rings, set_diag):
    C, rc = hex_lattice(10, 11, holes=HOLES[:2], seed=n_rings)
    base = sp.csr_matrix((np.ones(len(lattice_neighbours(rc))),
                          tuple(np.array(sorted(lattice_neighbours(rc))).T)), shape=(len(rc),) * 2)
    want = bfs_rings(base, n_rings)
    A, D = tg.spatial_neighbors(adata_of(C, uns={"spatial": {}}), n_rings=n_rings, set_diag=set_diag, copy=True)
    assert canonical(A) and canonical(D)
    assert entries(D) == want
    diag = {(i, i): 1.0 for i in range(len(rc))} if set_diag else {}
    assert entries(A) == {**{p: 1.0 for p in want}, **diag}


def test_grid_cut_median_is_per_library():
    C1, _ = hex_lattice(8, 8, seed=1)
    C2, _ = hex_lattice(8, 8, seed=2)
    C = np.r_[C1, 3.0 * C2 + 100.0]                    # the second library at 3x the spacing
    obs = pd.DataFrame({"lib": pd.Categorical(["a"] * 64 + ["b"] * 64)}, index=[f"s{i}" for i in range(128)])
    A, D = tg.spatial_neighbors(adata_of(C, uns={"spatial": {}}, obs=obs), library_key="lib", copy=True)
    A1, _ = tg.spatial_neighbors(adata_of(C1, uns={"spatial": {}}), copy=True)
    assert entries(A[:64, :64]) == entries(A1) and entries(A[64:, 64:]) == entries(A1)
    assert A[:64, 64:].nnz == 0 and A[64:, :64].nnz == 0


# ---- generic mode -----------------------------------------------------------------------------------------------------

def brute(C, lo, hi):
    d = pair_dist(C, np.arange(C.shape[0]))
    np.fill_diagonal(d, np.inf)
    return {(int(i), int(j)): float(d[i, j]) for i, j in zip(*np.nonzero((d >= lo) & (d <= hi)))}


def test_generic_knn_with_and_without_diagonal():
    rng = np.random.default_rng(3)
    C = rng.random((300, 3)) * [5, 5, 1]
    d = pair_dist(C, np.arange(300))
    for set_diag in (False, True):
        ad = adata_of(C)
        tg.spatial_neighbors(ad, n_neighs=7, set_diag=set_diag)
        A, D = ad.obsp["spatial_connectivities"], ad.obsp["spatial_distances"]
        assert canonical(A) and canonical(D)
        want = {}
        for i in range(300):
            order = [j for j in np.lexsort((np.arange(300), d[i])) if j != i][:7]
            want.update({(i, int(j)): float(d[i, j]) for j in order})
        assert entries(D) == want
        assert entries(A) == {**{p: 1.0 for p in want}, **({(i, i): 1.0 for i in range(300)} if set_diag else {})}


@pytest.mark.parametrize("radius", [0.1, (0.05, 0.12), (0.12, 0.05), 10.0])
def test_generic_radius_scalar_and_interval(radius):
    C = np.random.default_rng(4).random((400, 2))
    A, D = tg.spatial_neighbors(adata_of(C), radius=radius, copy=True)
    lo, hi = (0.0, radius) if np.isscalar(radius) else (min(radius), max(radius))
    want = brute(C, lo, hi)
    assert canonical(A) and canonical(D)
    assert entries(D) == want and entries(A) == {p: 1.0 for p in want}
    assert CALLS == [("radius", hi)]


def test_coincident_points_stay_connected_without_a_distance():
    rng = np.random.default_rng(5)
    C = rng.random((50, 2))
    C[10] = C[20] = C[30] = C[3]                         # four coincident spots
    for kw in (dict(n_neighs=4), dict(radius=0.2), dict(radius=0.0)):
        A, D = tg.spatial_neighbors(adata_of(C), copy=True, **kw)
        group = (3, 10, 20, 30)
        for i in group:
            for j in group:
                if i != j:
                    assert A[i, j] == 1.0 and (i, j) not in entries(D), (kw, i, j)
        assert (D.data > 0).all() and np.diff(D.indptr).sum() == D.nnz
    A, D = tg.spatial_neighbors(adata_of(C), n_neighs=2, copy=True)  # more than n_neighs + 1 coincide: smallest indices
    assert list(A[3].indices) == [10, 20] and list(A[30].indices) == [3, 10]


def test_libraries_in_shuffled_obs_order_keys_and_copy():
    rng = np.random.default_rng(6)
    n = 240
    lib = rng.permutation(np.repeat(["x", "y", "z"], [100, 80, 60]))
    C = rng.random((n, 2)) * 10                                       # overlapping extents: only the library separates
    obs = pd.DataFrame({"lib": pd.Categorical(lib, categories=["z", "x", "y"])}, index=[f"s{i}" for i in range(n)])
    ad = adata_of(C, obs=obs)
    out = tg.spatial_neighbors(ad, library_key="lib", n_neighs=5, key_added="nb")
    assert out is None
    assert set(ad.obsp) == {"nb_connectivities", "nb_distances"}
    assert ad.uns["nb_neighbors"] == {"connectivities_key": "nb_connectivities", "distances_key": "nb_distances",
                                      "params": {"n_neighbors": 5, "coord_type": "generic", "radius": None,
                                                 "transform": None}}
    A, D = ad.obsp["nb_connectivities"], ad.obsp["nb_distances"]
    assert canonical(A) and canonical(D)
    want = {}
    for name in ("x", "y", "z"):
        g = np.nonzero(lib == name)[0]
        _, Dg = tg.spatial_neighbors(adata_of(C[g]), n_neighs=5, copy=True)
        want.update({(int(g[i]), int(g[j])): v for (i, j), v in entries(Dg).items()})
    assert entries(D) == want and entries(A) == {p: 1.0 for p in want}
    ad2 = adata_of(C, obs=obs)
    A2, D2 = tg.spatial_neighbors(ad2, library_key="lib", n_neighs=5, copy=True)
    assert ad2.obsp == {} and "spatial_neighbors" not in ad2.uns
    assert entries(A2) == entries(A) and entries(D2) == entries(D)


@pytest.mark.parametrize("standardized,self_inclusion", [(True, True), (False, False), (False, True)])
def test_spatial_weights_accept_the_graph(standardized, self_inclusion):
    C = np.random.default_rng(7).random((120, 2))
    C[5] = C[6]                                                       # a connection without a distance entry
    ad = adata_of(C)
    tg.spatial_neighbors(ad, n_neighs=6)
    w = spatial_weights(ad, standardized=standardized, self_inclusion=self_inclusion)
    conn = ad.obsp["spatial_connectivities"].toarray()
    dist = ad.obsp["spatial_distances"].toarray()
    if standardized:
        rs = np.abs(dist).sum(axis=1, keepdims=True)
        rs[rs == 0] = 1.0
        want = (dist / rs) * (conn != 0)
    else:
        want = conn.copy()
    if self_inclusion:
        want = want + np.eye(120)
    assert w.shape == (120, 120) and w.dtype == np.float32
    np.testing.assert_allclose(w.toarray(), want.astype(np.float32), rtol=1e-6, atol=0)


def test_stand_in_distance_is_numpys():
    rng = np.random.default_rng(8)
    for dim in (2, 3):
        C = rng.standard_normal((40, dim)) * 1e3 + 1e6
        d = pair_dist(C, np.arange(40))
        for i, j in rng.integers(0, 40, (200, 2)):
            assert d[i, j] == np.sqrt(((C[j] - C[i]) ** 2).sum())


def test_entry_points_check_arguments():
    import torch
    from tangram_b200 import _lib
    lib = _lib.load()
    C = np.random.default_rng(9).random((10, 2))
    idx, dst, ip = np.empty((10, 64), np.int32), np.empty((10, 64)), np.empty(11, np.int64)

    def knn(coords=C, n=10, dim=2, k=3, outs=True):
        o = (_lib.ptr(idx), _lib.ptr(dst)) if outs else (None, None)
        return lib.tgb200_spatial_knn(_lib.ptr(coords), n, dim, k, *o, 0, None)

    def radius(r=0.5, cap=0, outs=False, dim=2, n=10):
        o = (_lib.ptr(idx), _lib.ptr(dst)) if outs else (None, None)
        return lib.tgb200_spatial_radius(_lib.ptr(C), n, dim, r, _lib.ptr(ip), *o, cap, 0, None)

    def err():
        return lib.tgb200_last_error()
    assert knn(dim=4) == -1 and b"dim=4" in err()
    assert knn(n=1) == -1 and b"n=1" in err()
    assert knn(n=2 ** 31) == -1 and b"n=2147483648" in err()
    assert knn(k=65) == -1 and b"[1, 64]" in err()
    assert knn(k=0) == -1 and b"k=0" in err()
    assert knn(k=10) == -1 and b"more than k points" in err()
    assert knn(outs=False) == -1 and b"null output" in err()
    assert knn(coords=None) == -1 and b"null coordinates" in err()
    assert radius(r=-1.0) == -1 and b"radius" in err()
    assert radius(r=float("nan")) == -1 and b"radius" in err()
    assert radius(cap=5) == -1 and b"capacity=5" in err()
    assert radius(n=0) == -1 and b"n=0" in err()
    if not torch.cuda.is_available():
        assert knn() == -5 and b"no CPU fallback" in err()
        assert radius() == -5 and b"no CPU fallback" in err()


def test_device_pass_refuses_without_gpu(monkeypatch):
    import torch
    from tangram_b200 import _lib
    monkeypatch.undo()
    if torch.cuda.is_available():
        pytest.skip("a CUDA device is visible")
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        tg.spatial_neighbors(adata_of(np.random.default_rng(0).random((10, 2))))
