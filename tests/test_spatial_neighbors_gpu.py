"""tgb200_spatial_knn, tgb200_spatial_radius and spatial_neighbors on the H100.

* the k-nearest query equals a float64 numpy brute force ranked by np.lexsort((j, d)) -- indices exactly, distances bit
  for bit -- on uniform points, an exact square lattice (ties at the k-th place, points on cell edges), a hexagonal
  lattice, duplicates, all-identical points, collinear points (on an axis and on a diagonal), 3-D points, coordinates
  offset by 1e6, n = k + 1, and a skewed set with half the points in a 1e-6 box, for k = 1, 6 and 64;
* the radius query equals the brute force on the same inputs for a scalar radius, an interval and a radius covering
  every pair; two runs of either query give identical bits;
* at 1M uniform 2-D points, k = 6 equals scipy's cKDTree.query(k=7) without the point itself;
* spatial_neighbors on a MiniAnnData equals the float64 stand-in's result exactly in generic, radius, grid (1 and 2
  rings) and library modes, and map_cells_to_space with the three spatial terms gives the same history and mapping
  bits with the device graph as with the stand-in's.
"""
import sys

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

import tangram_b200 as tg  # noqa: E402
from tests.test_spatial_neighbors import adata_of, entries, hex_lattice, knn_f64, radius_f64  # noqa: E402

snb = sys.modules["tangram_b200.spatial_neighbors"]


def inputs():
    rng = np.random.default_rng(0)
    sq = np.stack(np.meshgrid(np.arange(30.0), np.arange(30.0)), -1).reshape(-1, 2)
    base = rng.random((400, 2))
    skew = np.r_[rng.random((500, 2)), 0.5 + 1e-6 * rng.random((500, 2))]
    t = rng.random(300)
    return {
        "uniform": rng.random((2000, 2)) * 50,
        "square_lattice": sq,
        "hex_lattice": hex_lattice(25, 25, jitter=0.0)[0],
        "duplicates": np.repeat(base, 3, axis=0)[rng.permutation(1200)],
        "identical": np.full((100, 2), 3.25),
        "collinear_axis": np.c_[rng.random(300) * 10, np.full(300, -7.0)],
        "collinear_diagonal": np.c_[t, 2 * t + 1],
        "uniform_3d": rng.random((1500, 3)) * [10, 10, 2],
        "offset_1e6": rng.random((1000, 2)) + 1e6,
        "skewed": skew,
    }


INPUTS = inputs()


def knn_pairs():
    for name, C in INPUTS.items():
        for k in (1, 6, 64):
            if k < C.shape[0]:
                yield name, k
    yield "n_eq_k_plus_1", 1
    yield "n_eq_k_plus_1", 6
    yield "n_eq_k_plus_1", 64


def coords(name, k=None):
    if name == "n_eq_k_plus_1":
        return np.random.default_rng(k).random((k + 1, 2))
    return INPUTS[name]


@pytest.mark.parametrize("name,k", list(knn_pairs()))
def test_knn_equals_brute_force(name, k):
    C = coords(name, k)
    idx, dst = snb._knn(C, k)
    widx, wdst = knn_f64(C, k)
    assert np.array_equal(idx, widx)
    assert np.array_equal(dst.view(np.uint64), wdst.view(np.uint64))
    idx2, dst2 = snb._knn(C, k)
    assert np.array_equal(idx2, idx) and np.array_equal(dst2.view(np.uint64), dst.view(np.uint64))


def rows_of(indptr, idx, dst):
    """Each row's (column, distance bits) pairs, sorted by column."""
    out = []
    for i in range(len(indptr) - 1):
        j, d = idx[indptr[i]:indptr[i + 1]], dst[indptr[i]:indptr[i + 1]]
        o = np.argsort(j, kind="stable")
        out.append((j[o].tolist(), d[o].view(np.uint64).tolist()))
    return out


@pytest.mark.parametrize("name", list(INPUTS))
def test_radius_equals_brute_force(name):
    C = INPUTS[name]
    _, d6 = knn_f64(C, min(6, C.shape[0] - 1))
    r = float(np.median(d6[:, -1]))
    span = float(np.sqrt(((C.max(0) - C.min(0)) ** 2).sum()))
    for radius in (r, 2 * span + 1.0):
        got = snb._radius(C, radius)
        want = radius_f64(C, radius)
        assert np.array_equal(got[0], want[0]), (name, radius)
        assert rows_of(*got) == rows_of(*want), (name, radius)
        again = snb._radius(C, radius)
        assert np.array_equal(again[0], got[0]) and rows_of(*again) == rows_of(*got)   # rows come in search order
    # the interval through the public layer, against the stand-in run of the same layer
    A, D = tg.spatial_neighbors(adata_of(C), radius=(0.5 * r, r), copy=True)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(snb, "_radius", radius_f64)
        A0, D0 = tg.spatial_neighbors(adata_of(C), radius=(0.5 * r, r), copy=True)
    assert entries(A) == entries(A0) and entries(D) == entries(D0)


def test_radius_zero_finds_coincident_points():
    C = INPUTS["duplicates"]
    got = snb._radius(C, 0.0)
    assert np.array_equal(np.diff(got[0]), np.full(1200, 2))
    assert rows_of(*got) == rows_of(*radius_f64(C, 0.0))


def test_million_uniform_points_against_ckdtree():
    from scipy.spatial import cKDTree
    C = np.random.default_rng(1).random((1_000_000, 2))
    idx, dst = snb._knn(C, 6)
    d7, i7 = cKDTree(C).query(C, k=7, workers=-1)
    self_col = i7 == np.arange(len(C))[:, None]
    assert (self_col.sum(axis=1) == 1).all()
    want_i = i7[~self_col].reshape(-1, 6)
    want_d = d7[~self_col].reshape(-1, 6)
    o = np.argsort(want_i, axis=1)
    assert np.array_equal(idx, np.take_along_axis(want_i, o, axis=1))
    np.testing.assert_allclose(dst, np.take_along_axis(want_d, o, axis=1), rtol=1e-14, atol=0)


CASES = {
    "generic": dict(n_neighs=6),
    "generic_diag": dict(n_neighs=9, set_diag=True),
    "radius": dict(radius=0.04),
    "interval": dict(radius=(0.02, 0.05)),
    "grid": dict(coord_type="grid"),
    "grid_rings2": dict(coord_type="grid", n_rings=2, set_diag=True),
    "library": dict(library_key="lib", n_neighs=5),
    "library_grid": dict(library_key="lib", coord_type="grid", n_rings=2),
}


@pytest.mark.parametrize("case", list(CASES))
def test_public_api_equals_the_stand_in(case):
    rng = np.random.default_rng(2)
    if case.startswith("grid") or case == "library_grid":
        C, _ = hex_lattice(40, 40, holes=((5, 5), (20, 21), (30, 3)))
        C = C / 40.0
    else:
        C = rng.random((3000, 2))
    C[7] = C[8]
    n = C.shape[0]
    obs = pd.DataFrame({"lib": pd.Categorical(rng.choice(["a", "b", "c"], n))}, index=[f"s{i}" for i in range(n)])
    ad = adata_of(C, obs=obs)
    tg.spatial_neighbors(ad, **CASES[case])
    ref = adata_of(C, obs=obs)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(snb, "_knn", knn_f64)
        mp.setattr(snb, "_radius", radius_f64)
        tg.spatial_neighbors(ref, **CASES[case])
    for key in ("spatial_connectivities", "spatial_distances"):
        a, b = ad.obsp[key], ref.obsp[key]
        assert a.has_canonical_format and a.dtype == np.float64
        assert np.array_equal(a.indptr, b.indptr) and np.array_equal(a.indices, b.indices)
        assert np.array_equal(a.data.view(np.uint64), b.data.view(np.uint64))
    assert ad.uns["spatial_neighbors"] == ref.uns["spatial_neighbors"]


def test_map_cells_to_space_with_the_device_graph():
    from oracle.tangram_oracle import synthetic_inputs
    N, K = 300, 50
    C, _ = hex_lattice(10, 12, holes=((4, 4),))
    V = C.shape[0]
    inp = synthetic_inputs(N, V, K, seed=5)
    genes = [f"Gene{i}" for i in range(K)]

    def run(stand_in):
        ad_sc = tg.MiniAnnData(X=inp["S"].copy(), obs=pd.DataFrame({"lab": [f"t{i % 3}" for i in range(N)]},
                               index=[f"c{i}" for i in range(N)]), var=pd.DataFrame(index=genes))
        ad_sp = tg.MiniAnnData(X=inp["G"].copy(), obs=pd.DataFrame(index=[f"v{i}" for i in range(V)]),
                               var=pd.DataFrame(index=genes), obsm={"spatial": C.copy()})
        tg.pp_adatas(ad_sc, ad_sp)
        with pytest.MonkeyPatch.context() as mp:
            if stand_in:
                mp.setattr(snb, "_knn", knn_f64)
            tg.spatial_neighbors(ad_sp)
        ad_map = tg.map_cells_to_space(ad_sc, ad_sp, device="cuda:0", num_epochs=20, random_state=3, verbose=False,
                                       cluster_label="lab", lambda_neighborhood_g1=0.5, lambda_ct_islands=0.5,
                                       lambda_getis_ord=0.5)
        return ad_map, ad_sp

    got, sp_got = run(False)
    want, sp_want = run(True)
    assert entries(sp_got.obsp["spatial_distances"]) == entries(sp_want.obsp["spatial_distances"])
    assert np.array_equal(got.X, want.X)
    hg, hw = got.uns["training_history"], want.uns["training_history"]
    assert set(hg) == set(hw)
    for key in hg:
        a, b = np.asarray(hg[key], dtype=np.float64), np.asarray(hw[key], dtype=np.float64)
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), key
