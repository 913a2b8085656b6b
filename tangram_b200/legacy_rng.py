"""The reference's initial draw on the device.  Mapper's default M0 is `np.random.normal(0, 1, (N, V))` after
`np.random.seed(random_state)` (mapping_optimizer.py:147-157): numpy's legacy polar method on MT19937.
tgb200_init_mapping_legacy reproduces that stream bit for bit on the GPU and returns the generator state numpy holds
after the host draw, so the global generator ends where it would have.  The device formula equals numpy's arithmetic
as long as numpy's C code rounds x1*x1 and x2*x2 separately; `device_draw_supported` checks that once per process."""
import ctypes
import math
import warnings

import numpy as np

from . import _lib

_PROBE = None


def polar_normals(state, n):
    """The first n values of np.random.normal(0, 1, n) from `state` (an np.random.get_state() tuple), computed the way
    the device does: a cached value first if there is one, then attempts of 4 MT19937 words, d = ((w0 >> 5) * 2^26 +
    (w1 >> 6)) / 2^53, x = 2 d - 1, rejected unless 0 < x1*x1 + x2*x2 < 1, then f*x2 and f*x1 with
    f = sqrt(-2 log(r2) / r2) from libm (math.log, math.sqrt)."""
    _, key, pos, has_gauss, gauss = state
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": np.asarray(key, dtype=np.uint32), "pos": int(pos)}}
    out = [float(gauss)] if has_gauss else []
    while len(out) < n:
        w = [int(x) for x in bg.random_raw(4)]
        x1 = 2.0 * (((w[0] >> 5) * 67108864.0 + (w[1] >> 6)) / 9007199254740992.0) - 1.0
        x2 = 2.0 * (((w[2] >> 5) * 67108864.0 + (w[3] >> 6)) / 9007199254740992.0) - 1.0
        r2 = x1 * x1 + x2 * x2
        if r2 >= 1.0 or r2 == 0.0:
            continue
        f = math.sqrt(-2.0 * math.log(r2) / r2)
        out += [f * x2, f * x1]
    return np.array(out[:n], dtype=np.float64)


def device_draw_supported(n=4000):
    """True if this numpy's np.random.normal equals the device formula on n values of a private RandomState (checked
    once per process).  A numpy built to contract x1*x1 + x2*x2 into an FMA (possible on aarch64) fails it; Mapper
    then keeps the host draw and warns."""
    global _PROBE
    if _PROBE is None:
        rs = np.random.RandomState(20250917)
        want = polar_normals(rs.get_state(), n)
        got = rs.normal(0, 1, n)
        _PROBE = bool(np.array_equal(want.view(np.uint64), got.view(np.uint64)))
        if not _PROBE:
            warnings.warn("numpy's legacy normal generator does not match the device formula on this host: "
                          "the initial mapping is drawn on the host", RuntimeWarning, stacklevel=3)
    return _PROBE


def draw_global(engine, skip, first_row, end_normal):
    """The draw from numpy's global generator into `engine` (Engine.init_mapping_legacy), which leaves the generator
    where the host draw would leave it."""
    end, n_fixed = engine.init_mapping_legacy(np.random.get_state(), skip, first_row, end_normal)
    np.random.set_state(end)
    return n_fixed


def jump(state, n_words):
    """numpy's generator state after n_words more MT19937 words (host only: tgb200_mt19937_jump)."""
    out = _lib.MtState()
    _lib.check(_lib.load().tgb200_mt19937_jump(ctypes.byref(_lib.MtState.from_numpy(state)), int(n_words),
                                               ctypes.byref(out)))
    return out.to_numpy()
