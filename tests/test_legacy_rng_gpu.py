"""The device draw of numpy's legacy normal stream (tgb200_init_mapping_legacy) against np.random.normal: float32 bit
patterns of the mapping and the generator state left behind, for seeded and unseeded starts, odd shapes, more than
65535 voxels, 2e8 values, shard slices and the constrained draw; then Mapper / MapperConstrained end to end."""
import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs
from tangram_b200 import Mapper, MapperConstrained, _lib
from tangram_b200.engine import Engine
from tangram_b200.mapping_optimizer import legacy_normal_rows
from tangram_b200.sharded import shard_rows

pytestmark = pytest.mark.gpu


def _start(name):
    if name == "unseeded":
        rs = np.random.RandomState()
        rs.normal(size=1001)                # leaves a cached normal
        rs.random_sample(77)
        return rs
    return np.random.RandomState({"seed42": 42, "seed7": 7, "seed2^32-1": 2**32 - 1}[name])


def _device_draw(n_rows, V, state, skip=0, first_row=0, end_normal=None):
    e = Engine(n_rows, V, 8, precision="fp32", density_mode=_lib.DENSITY_NONE)
    try:
        end, n_fixed = e.init_mapping_legacy(state, skip, first_row, end_normal)
        M = np.empty((n_rows, V), dtype=np.float32)
        e.get_state(M=M)
        stats = e.debug("legacy_init")
    finally:
        e.close()
    return M, end, n_fixed, stats


def _assert_same_state(a, b):
    assert np.array_equal(np.asarray(a[1], np.uint32), np.asarray(b[1], np.uint32))
    assert a[2] == b[2] and a[3] == b[3]
    assert np.float64(a[4]).view(np.uint64) == np.float64(b[4]).view(np.uint64)


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


@pytest.mark.parametrize("shape", [(3, 1001), (1000, 999), (64, 70001)])
@pytest.mark.parametrize("start", ["seed42", "seed7", "seed2^32-1", "unseeded"])
def test_device_draw_is_bit_equal_to_numpy(start, shape):
    rs = _start(start)
    n, V = shape
    M, end, n_fixed, stats = _device_draw(n, V, rs.get_state())
    want = rs.normal(0, 1, (n, V)).astype(np.float32)
    assert _bits_equal(M, want)
    _assert_same_state(end, rs.get_state())
    print(f"{start} {n}x{V}: {n_fixed} values recomputed on the host, {int(stats[7])} changed by it")


def test_device_draw_of_2e8_values():
    rs = np.random.RandomState(42)
    n, V = 20000, 10000
    M, end, n_fixed, stats = _device_draw(n, V, rs.get_state())
    for r in range(0, n, 2000):                 # the host draw in slices: 1.6 GB of float64 at most
        assert _bits_equal(M[r:r + 2000], rs.normal(0, 1, (2000, V)).astype(np.float32)), r
    _assert_same_state(end, rs.get_state())
    print(f"2e8 values: {n_fixed} recomputed on the host, {int(stats[7])} changed; jump {stats[0]:.2f} ms, "
          f"count+scan {stats[1]:.2f} ms, emit {stats[2]:.2f} ms, fix-up {stats[3]:.2f} ms, {int(stats[5])} draw blocks")


@pytest.mark.parametrize("start", ["seed7", "unseeded"])
def test_shard_slices_match_the_full_draw(start):
    rs = _start(start)
    st = rs.get_state()
    n, V = 1000, 333
    full = rs.normal(0, 1, (n, V)).astype(np.float32)
    for rank in range(3):
        r0, r1 = shard_rows(n, rank, 3)
        M, end, _, _ = _device_draw(r1 - r0, V, st, 0, r0, r1 * V)
        assert _bits_equal(M, full[r0:r1]), rank
        ref = np.random.RandomState()
        ref.set_state(st)
        ref.normal(0, 1, r1 * V)
        _assert_same_state(end, ref.get_state())


def test_constrained_draw_skips_the_first_matrix():
    rs = np.random.RandomState(11)
    st = rs.get_state()
    n, V = 500, 77
    M, end, _, _ = _device_draw(n, V, st, skip=n * V, end_normal=2 * n * V)
    rs.normal(0, 1, (n, V))
    assert _bits_equal(M, rs.normal(0, 1, (n, V)).astype(np.float32))
    _assert_same_state(end, rs.get_state())


def _inputs():
    inp = synthetic_inputs(700, 130, 60, seed=3)
    return dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_mapper_default_draw_equals_an_explicit_host_draw(precision):
    kw = _inputs()
    N, V = kw["S"].shape[0], kw["G"].shape[0]
    a = Mapper(random_state=42, precision=precision, **kw)
    state_a = np.random.get_state()
    M0 = legacy_normal_rows(42, N, V, 0, N)
    _assert_same_state(state_a, np.random.get_state())
    b = Mapper(M0=M0, precision=precision, **kw)
    assert _bits_equal(a.state()[0], M0)
    out_a, hist_a = a.train(10, print_each=None)
    out_b, hist_b = b.train(10, print_each=None)
    assert _bits_equal(out_a, out_b)
    assert np.array_equal(a.history_matrix, b.history_matrix, equal_nan=True)
    for k in hist_a:
        assert np.array_equal(np.array(hist_a[k], np.float64), np.array(hist_b[k], np.float64), equal_nan=True), k


def test_mapper_shard_keeps_its_rows_of_the_full_draw():
    kw = _inputs()
    N, V = kw["S"].shape[0], kw["G"].shape[0]
    r0, r1 = shard_rows(N, 1, 3)
    m = Mapper(random_state=9, shard=(r0, r1), **kw)
    state = np.random.get_state()
    want = legacy_normal_rows(9, N, V, r0, r1)
    _assert_same_state(state, np.random.get_state())
    assert _bits_equal(m.state()[0], want)


def test_mapper_constrained_draws_the_same_M0_and_F0():
    kw = _inputs()
    N, V = kw["S"].shape[0], kw["G"].shape[0]
    m = MapperConstrained(kw["S"], kw["G"], kw["d"], random_state=5)
    state = np.random.get_state()
    np.random.seed(5)
    np.random.normal(0, 1, (N, V))
    M0 = np.random.normal(0, 1, (N, V))
    F0 = np.random.normal(0, 1, N)
    _assert_same_state(state, np.random.get_state())
    M, F, _ = m.state()
    assert _bits_equal(M, M0.astype(np.float32))
    assert _bits_equal(F, F0.astype(np.float32))
