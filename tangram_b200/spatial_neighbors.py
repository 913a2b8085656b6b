"""The spatial neighbour graph on the GPU, without squidpy: `spatial_neighbors` stands in for squidpy 1.x's
`sq.gr.spatial_neighbors` (what the reference's pp_adatas calls when adata_sp.obsm["spatial"] exists) and writes what it
writes, so the Mapper's spatial terms (lambda_neighborhood_g1, lambda_ct_islands, lambda_getis_ord, through
`spatial_weights`) can read it:

    tg.spatial_neighbors(ad_sp, set_diag=False)        # obsp["spatial_connectivities"], obsp["spatial_distances"]

The search -- exact k nearest or radius neighbours in float64 -- is one device pass per library (tgb200_spatial_knn,
tgb200_spatial_radius); the grid cut, the rings, the diagonal, the interval pruning and the zero elimination are
numpy / scipy on its output.  Departures from squidpy: k-nearest ties are ranked by (distance, index), and a point is
excluded from its own row by index only, so when more than n_neighs + 1 points coincide the row holds the smallest other
indices (sklearn may return any of them, the point itself included); Delaunay graphs, `percentile` and `transform` are
not implemented.  Parity with squidpy itself was not checked: squidpy is not a dependency, and this module restates its
documented behaviour.
"""
import ctypes
import numbers
import warnings

import numpy as np
import pandas as pd

from . import _lib
from .engine import _require_device

MAX_K = 64                              # largest n_neighs of the device k-nearest query
_GRID_CUT = 1.3                         # squidpy's grid mode keeps d < 1.3 * median of the k-nearest distances


def _stream(dev):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _knn(C, k, device=None):
    """tgb200_spatial_knn: -> (indices (n, k) int32, distances (n, k) float64), each row the k nearest j != i ranked by
    (distance, j) and listed in increasing j."""
    dev = _require_device("cuda" if device is None else device)
    C = np.ascontiguousarray(C, dtype=np.float64)
    n, dim = C.shape
    idx = np.empty((n, k), dtype=np.int32)
    dst = np.empty((n, k), dtype=np.float64)
    _lib.check(_lib.load().tgb200_spatial_knn(_lib.ptr(C), n, dim, int(k), _lib.ptr(idx), _lib.ptr(dst), dev,
                                              _stream(dev)))
    return idx, dst


def _radius(C, r, device=None):
    """tgb200_spatial_radius: -> (indptr (n + 1) int64, indices int32, distances float64) of every j != i with
    distance <= r, each row in search order (not sorted)."""
    dev = _require_device("cuda" if device is None else device)
    C = np.ascontiguousarray(C, dtype=np.float64)
    n, dim = C.shape
    lib = _lib.load()
    indptr = np.empty(n + 1, dtype=np.int64)
    _lib.check(lib.tgb200_spatial_radius(_lib.ptr(C), n, dim, float(r), _lib.ptr(indptr), None, None, 0, dev,
                                         _stream(dev)))
    nnz = int(indptr[-1])
    idx = np.empty(nnz, dtype=np.int32)
    dst = np.empty(nnz, dtype=np.float64)
    if nnz:
        _lib.check(lib.tgb200_spatial_radius(_lib.ptr(C), n, dim, float(r), _lib.ptr(indptr), _lib.ptr(idx),
                                             _lib.ptr(dst), nnz, dev, _stream(dev)))
    return indptr, idx, dst


def _csr(n, indptr, indices, data):
    import scipy.sparse as sp
    m = sp.csr_matrix((data, indices, indptr), shape=(n, n))
    m.sort_indices()
    return m


def _keep(indptr, indices, data, keep):
    """The CSR triplet without the entries where `keep` is False."""
    if keep.all():
        return indptr, indices, data
    n = indptr.shape[0] - 1
    rows = np.repeat(np.arange(n), np.diff(indptr))[keep]
    out = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(np.bincount(rows, minlength=n), out=out[1:])
    return out, indices[keep], data[keep]


def _pattern(m):
    """The connectivities of a graph: its pattern with value 1."""
    import scipy.sparse as sp
    return sp.csr_matrix((np.ones_like(m.data), m.indices.copy(), m.indptr.copy()), shape=m.shape)


def _generic(C, n_neighs, radius, device):
    n = C.shape[0]
    if radius is None:
        idx, dst = _knn(C, n_neighs, device)
        D = _csr(n, np.arange(n + 1, dtype=np.int64) * n_neighs, idx.ravel(), dst.ravel())
    else:
        lo, hi = (0.0, float(radius)) if _is_scalar(radius) else (min(radius), max(radius))
        indptr, idx, dst = _radius(C, hi, device)
        D = _csr(n, *_keep(indptr, idx, dst, dst >= lo))
    return _pattern(D), D


def _grid(C, n_neighs, n_rings, device):
    """squidpy's _build_grid: the k-nearest graph cut at 1.3 x its median distance, then rings of walks on it."""
    import scipy.sparse as sp
    n = C.shape[0]
    idx, dst = _knn(C, n_neighs, device)
    cut = _GRID_CUT * np.median(dst)
    indptr, idx, dst = _keep(np.arange(n + 1, dtype=np.int64) * n_neighs, idx.ravel(), dst.ravel(), dst.ravel() < cut)
    A = _csr(n, indptr, idx, np.ones_like(dst))
    if n_rings == 1:
        return A, A.copy()
    A = (A + sp.identity(n, format="csr")).tocsr()
    A.data[:] = 1.0
    res, walk = A.copy(), A
    for r in range(1, n_rings):
        walk = (walk @ A).tocsr()
        walk.data[:] = 1.0
        walk = (walk - walk.multiply(res != 0)).tocsr()     # ring r + 1: reached now, not before
        walk.eliminate_zeros()
        walk.data[:] = r + 1.0
        res = (res + walk).tocsr()
    res.setdiag(0.0)
    res.eliminate_zeros()
    res.sort_indices()
    return _pattern(res), res


def _graph(C, coord_type, n_neighs, radius, n_rings, device):
    if coord_type == "grid":
        return _grid(C, n_neighs, n_rings, device)
    return _generic(C, n_neighs, radius, device)


def _assemble(n, parts):
    """The libraries' graphs [(obs rows, Adj, Dst)] as two (n, n) canonical CSR matrices in obs order."""
    import scipy.sparse as sp
    out = []
    for which in (1, 2):
        rows, cols, vals = [], [], []
        for part in parts:
            g, m = part[0], part[which].tocoo()
            rows.append(g[m.row])
            cols.append(g[m.col])
            vals.append(m.data)
        m = sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n),
                          dtype=np.float64)
        m.sum_duplicates()
        m.sort_indices()
        out.append(m)
    return out


def _is_scalar(radius):
    return isinstance(radius, numbers.Real) or (np.ndim(radius) == 0 and np.isreal(radius))


def _check_radius(radius):
    if radius is None:
        return
    vals = [radius] if _is_scalar(radius) else list(radius)
    if len(vals) not in (1, 2) or not all(isinstance(v, numbers.Real) or np.ndim(v) == 0 for v in vals):
        raise ValueError(f"radius must be a number or a pair of numbers, got {radius!r}")
    if not all(np.isfinite(float(v)) and float(v) >= 0 for v in vals):
        raise ValueError(f"radius must be finite and non-negative, got {radius!r}")


def spatial_neighbors(adata, spatial_key="spatial", library_key=None, coord_type=None, n_neighs=6, radius=None,
                      delaunay=False, n_rings=1, percentile=None, transform=None, set_diag=False, key_added="spatial",
                      copy=False, *, device=None):
    """squidpy's gr.spatial_neighbors on the GPU: the spatial graph of adata.obsm[spatial_key] (2 or 3 finite columns).

    coord_type: "grid" (squidpy's default when spatial_key is in adata.uns) or "generic".
      generic, radius None: the n_neighs nearest j != i, ranked by (distance, j); connectivities 1, distances d.
      generic, radius r: every j != i with d <= r; radius (a, b): min(a, b) <= d <= max(a, b).
      grid: the n_neighs-nearest graph cut at d >= 1.3 * its median distance (per library), connectivities and distances
        1; with n_rings > 1 the rings of walks on it (and the diagonal), distances the ring number.  radius is ignored
        there, with a warning.
    d = sqrt(sum (C[j] - C[i]) ** 2) in float64, as numpy computes it.  set_diag puts 1 on the connectivities' diagonal;
    the distances never keep it, and their entries equal to 0 (coincident points) are dropped, so such points stay
    connected with no distance entry.  library_key: a categorical obs column; one graph per library, assembled in obs
    order.  Writes obsp[key_added + "_connectivities"] and obsp[key_added + "_distances"] (canonical float64 CSR) and
    uns[key_added + "_neighbors"], or with copy=True returns (connectivities, distances) and writes nothing.

    ValueError for a missing or malformed spatial_key, n_neighs < 1, n_rings < 1, a bad radius, and when a library has
    no more than n_neighs points for a k-nearest query (generic without radius, and grid); NotImplementedError for
    delaunay=True, percentile and transform.  The search runs on `device` (default: torch's current CUDA device)."""
    import scipy.sparse as sp
    if delaunay:
        raise NotImplementedError("delaunay=True is not implemented")
    if percentile is not None:
        raise NotImplementedError("percentile is not implemented")
    if transform is not None:
        raise NotImplementedError("transform is not implemented")
    if spatial_key not in adata.obsm:
        raise ValueError(f"spatial_key {spatial_key!r} is not in adata.obsm")
    C = np.asarray(adata.obsm[spatial_key])
    if C.ndim != 2 or C.shape[1] not in (2, 3):
        raise ValueError(f"adata.obsm[{spatial_key!r}] has shape {C.shape}, expected (n_obs, 2) or (n_obs, 3)")
    C = C.astype(np.float64)
    if not np.isfinite(C).all():
        raise ValueError(f"adata.obsm[{spatial_key!r}] holds values that are not finite")
    if n_neighs < 1:
        raise ValueError(f"n_neighs={n_neighs}, must be at least 1")
    if n_rings < 1:
        raise ValueError(f"n_rings={n_rings}, must be at least 1")
    n_neighs, n_rings = int(n_neighs), int(n_rings)
    if coord_type is None:
        coord_type = "grid" if spatial_key in adata.uns else "generic"
    if coord_type not in ("grid", "generic"):
        raise ValueError(f"coord_type={coord_type!r}, must be 'grid', 'generic' or None")
    _check_radius(radius)
    if coord_type == "grid" and radius is not None:
        warnings.warn(f"radius={radius!r} is ignored for coord_type='grid'", stacklevel=2)
    knn = coord_type == "grid" or radius is None
    if knn and n_neighs > MAX_K:
        raise ValueError(f"n_neighs={n_neighs}, the k-nearest query supports at most {MAX_K}")

    n = C.shape[0]
    if library_key is None:
        groups = [np.arange(n)]
    else:
        if library_key not in adata.obs:
            raise KeyError(f"library_key {library_key!r} is not in adata.obs")
        lib = adata.obs[library_key]
        if not isinstance(lib.dtype, pd.CategoricalDtype):
            raise TypeError(f"adata.obs[{library_key!r}] must be categorical, it is {lib.dtype}")
        codes = np.asarray(lib.cat.codes)
        if (codes < 0).any():
            raise ValueError(f"adata.obs[{library_key!r}] has missing values")
        groups = [g for g in (np.nonzero(codes == c)[0] for c in range(len(lib.cat.categories))) if len(g)]
    if knn:
        for g in groups:
            if n_neighs >= len(g):
                raise ValueError(f"n_neighs={n_neighs} needs more than n_neighs points, a library has {len(g)}")

    if library_key is None:
        Adj, Dst = _graph(C, coord_type, n_neighs, radius, n_rings, device)
    else:
        Adj, Dst = _assemble(n, [(g, *_graph(C[g], coord_type, n_neighs, radius, n_rings, device)) for g in groups])
    if set_diag:
        Adj = (Adj + sp.identity(n, format="csr", dtype=np.float64)).tocsr()
        Adj.sort_indices()
    Dst.eliminate_zeros()
    if copy:
        return Adj, Dst
    conns_key, dists_key = f"{key_added}_connectivities", f"{key_added}_distances"
    adata.obsp[conns_key] = Adj
    adata.obsp[dists_key] = Dst
    adata.uns[f"{key_added}_neighbors"] = {
        "connectivities_key": conns_key, "distances_key": dists_key,
        "params": {"n_neighbors": n_neighs, "coord_type": coord_type, "radius": radius, "transform": transform}}
    return None
