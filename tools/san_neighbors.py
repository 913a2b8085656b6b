"""Dev tool: target for `compute-sanitizer --tool memcheck` over tgb200_spatial_knn and tgb200_spatial_radius at small
shapes -- ragged n around the 128-thread blocks and the 2048-value scan tiles (1, 2, 127, 129, 2049 and 5000 points),
2-D and 3-D, a skewed set with half its points in a 1e-6 box, the k-nearest query at k = 1, 6 and 64 and the radius
query's count and fill calls -- each checked against the float64 brute force of tests/test_spatial_neighbors.py, then
refused calls (k above the cap, and a NaN coordinate, which is refused after the device pass that finds it) followed by
a good call.

    compute-sanitizer --tool memcheck python tools/san_neighbors.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tangram_b200 import _lib  # noqa: E402
from tests.test_spatial_neighbors import knn_f64, radius_f64  # noqa: E402

snb = sys.modules["tangram_b200.spatial_neighbors"]
rng = np.random.default_rng(0)


def check_knn(C, k):
    idx, dst = snb._knn(C, k)
    widx, wdst = knn_f64(C, k)
    assert np.array_equal(idx, widx) and np.array_equal(dst, wdst), (C.shape, k)


def check_radius(C, r):
    ip, ix, dv = snb._radius(C, r)
    wip, wix, wdv = radius_f64(C, r)
    assert np.array_equal(ip, wip), (C.shape, r)
    for i in range(C.shape[0]):
        o, w = np.argsort(ix[ip[i]:ip[i + 1]]), np.argsort(wix[wip[i]:wip[i + 1]])
        assert np.array_equal(ix[ip[i]:ip[i + 1]][o], wix[wip[i]:wip[i + 1]][w])
        assert np.array_equal(dv[ip[i]:ip[i + 1]][o], wdv[wip[i]:wip[i + 1]][w])


for n in (1, 2, 127, 129, 2049, 5000):
    for dim in (2, 3):
        C = rng.random((n, dim))
        for k in (1, 6, 64):
            if k < n:
                check_knn(C, k)
        check_radius(C, 0.05 if n > 1000 else 0.3)
    print(n, "ok", flush=True)
S = np.r_[rng.random((1500, 2)), 0.5 + 1e-6 * rng.random((1500, 2))]
check_knn(S, 6)
check_radius(S, 1e-6)
print("skewed ok", flush=True)

lib = _lib.load()
C = rng.random((300, 2))
idx, dst = np.empty((300, 65), np.int32), np.empty((300, 65))
assert lib.tgb200_spatial_knn(_lib.ptr(C), 300, 2, 65, _lib.ptr(idx), _lib.ptr(dst), 0, None) == -1
print("k = 65 refused:", lib.tgb200_last_error().decode(), flush=True)
bad = C.copy()
bad[123, 1] = np.nan
assert lib.tgb200_spatial_knn(_lib.ptr(bad), 300, 2, 6, _lib.ptr(idx), _lib.ptr(dst), 0, None) == -1
print("NaN refused:", lib.tgb200_last_error().decode(), flush=True)
check_knn(C, 6)
print("done")
