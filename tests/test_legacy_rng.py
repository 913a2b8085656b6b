"""numpy's legacy normal stream without a GPU: the host MT19937 skip-ahead (tgb200_mt19937_jump) against numpy's own
generator, and a numpy model of the device draw's indexing (draw blocks -> accepted counts -> exclusive scan -> emit)
against np.random.normal, so that the indexing is pinned before any kernel runs."""
import math

import numpy as np
import pytest

from tangram_b200 import _lib, legacy_rng


def _rs_state(seed, pre_words=0, pre_normals=0):
    rs = np.random.RandomState(seed)
    if pre_words:
        rs.random_sample(pre_words // 2)          # 2 words per double
    if pre_normals:
        rs.normal(size=pre_normals)
    return rs


def _raw_after(state, n):
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": np.asarray(state[1], np.uint32), "pos": int(state[2])}}
    bg.random_raw(n)
    return bg.state["state"]


@pytest.mark.parametrize("start", ["fresh", "mid_block"])
@pytest.mark.parametrize("n", [0, 1, 3, 623, 624, 625, 10**6 + 3])
def test_jump_equals_random_raw(start, n):
    rs = _rs_state(42) if start == "fresh" else _rs_state(5, pre_words=2 * 117 + 1000)
    st = rs.get_state()
    assert (st[2] == 624) == (start == "fresh")
    got = legacy_rng.jump(st, n)
    want = _raw_after(st, n)
    assert np.array_equal(got[1], want["key"])
    assert got[2] == want["pos"]


def test_jump_by_2_128_agrees_with_numpy_jumped():
    """numpy's MT19937.jumped() applies x^(2^128) mod phi by Horner's rule to the circular buffer read from `pos` (624
    read as 0) and leaves `pos` where its Horner steps end, so its key holds the 624-word window that starts 2^128 words
    after the block's first word, rotated to begin at the new pos.  Read from its oldest word, that window continues as
    the stream 2^128 words after a fresh seed's: (window, pos=624) and our jump of (key, 624) by 2^128 words produce the
    same words.  (From a mid-block pos, numpy's window is not a contiguous piece of the stream, so there is nothing to
    compare.)"""
    bg = np.random.MT19937()
    bg._legacy_seeding(12345)
    st = bg.state["state"]
    assert st["pos"] == 624
    j = bg.jumped(1).state["state"]
    window = np.roll(j["key"], -j["pos"])
    ours = _lib.MtState()
    src = _lib.MtState.from_numpy(("MT19937", st["key"], 624, 0, 0.0))
    _lib.check(_lib.load().tgb200_mt19937_jump_pow2(src, 128, ours))
    a = np.random.MT19937()
    a.state = {"bit_generator": "MT19937", "state": {"key": window, "pos": 624}}
    b = np.random.MT19937()
    b.state = {"bit_generator": "MT19937", "state": {"key": np.ctypeslib.as_array(ours.key).copy(), "pos": ours.pos}}
    assert np.array_equal(a.random_raw(2000), b.random_raw(2000))


def test_jump_pow2_small_equals_jump():
    st = _rs_state(9, pre_words=300).get_state()
    lib = _lib.load()
    for e in (0, 5, 20):
        out = _lib.MtState()
        _lib.check(lib.tgb200_mt19937_jump_pow2(_lib.MtState.from_numpy(st), e, out))
        want = _raw_after(st, 1 << e)
        assert np.array_equal(np.ctypeslib.as_array(out.key), want["key"]) and out.pos == want["pos"]


def test_jump_rejects_a_bad_state():
    lib = _lib.load()
    st = _lib.MtState.from_numpy(np.random.RandomState(1).get_state())
    st.pos = 625
    assert lib.tgb200_mt19937_jump(st, 5, _lib.MtState()) == -1
    assert b"bad generator state" in lib.tgb200_last_error()


def test_probe_and_host_twin_match_numpy():
    assert legacy_rng.device_draw_supported()
    for rs in (_rs_state(42), _rs_state(7, pre_normals=3), _rs_state(3, pre_words=101)):
        st = rs.get_state()
        assert np.array_equal(legacy_rng.polar_normals(st, 5001).view(np.uint64), rs.normal(0, 1, 5001).view(np.uint64))


def _model_draw(state, V, skip, r0, r1, block_words):
    """The device draw in numpy: attempts in draw blocks of block_words words, accepted counts per block, exclusive scan,
    then each accepted attempt a writes normals has_gauss + 2a (f x2) and + 1 (f x1) into rows [r0, r1) of the draw
    that starts `skip` normals in.  Returns (rows, state after normal skip + r1 V)."""
    assert block_words % 4 == 0
    _, key, pos, hg, gauss = state
    t_lo, t_hi = skip + r0 * V, skip + r1 * V
    end = t_hi
    a_end = (end - hg + 1) // 2 - 1
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": np.asarray(key, np.uint32), "pos": int(pos)}}
    blocks, counts = [], []
    while sum(counts) <= a_end:                      # count pass
        w = bg.random_raw(block_words).reshape(-1, 4).astype(np.uint64)
        d1 = ((w[:, 0] >> 5).astype(np.float64) * 67108864.0 + (w[:, 1] >> 6)) / 9007199254740992.0
        d2 = ((w[:, 2] >> 5).astype(np.float64) * 67108864.0 + (w[:, 3] >> 6)) / 9007199254740992.0
        x1, x2 = 2.0 * d1 - 1.0, 2.0 * d2 - 1.0
        r2 = x1 * x1 + x2 * x2
        acc = (r2 < 1.0) & (r2 != 0.0)
        blocks.append((x1, x2, r2, acc))
        counts.append(int(acc.sum()))
    offs = np.concatenate([[0], np.cumsum(counts)])   # exclusive scan
    out = np.zeros((r1 - r0) * V)
    if hg and t_lo == 0:
        out[0] = gauss
    end_attempt, end_val = None, None
    for b, (x1, x2, r2, acc) in enumerate(blocks):    # emit pass
        for rank, i in enumerate(np.nonzero(acc)[0]):
            a = offs[b] + rank
            f = math.sqrt(-2.0 * math.log(r2[i]) / r2[i])
            for comp, x in ((0, x2[i]), (1, x1[i])):
                t = hg + 2 * a + comp
                if t_lo <= t < t_hi:
                    out[t - t_lo] = f * x
            if a == a_end:
                end_attempt, end_val = b * (block_words // 4) + i, f * x1[i]
    key_end = legacy_rng.jump(state, 4 * (end_attempt + 1))
    odd = (end - hg) % 2 == 1
    return out.reshape(r1 - r0, V), ("MT19937", key_end[1], key_end[2], int(odd), end_val if odd else 0.0)


@pytest.mark.parametrize("case", [
    dict(seed=42, V=7, n_rows=40, skip=0, rows=(0, 40), block_words=64),
    dict(seed=7, pre=3, V=11, n_rows=30, skip=0, rows=(0, 30), block_words=48),       # has_gauss = 1
    dict(seed=7, pre=3, V=9, n_rows=25, skip=0, rows=(8, 17), block_words=100),       # has_gauss = 1, a row slice
    dict(seed=2**32 - 1, V=13, n_rows=20, skip=20 * 13, rows=(0, 20), block_words=36),  # the constrained draw
    dict(seed=3, pre=5, V=5, n_rows=50, skip=17, rows=(33, 50), block_words=4),       # odd skip and V, last shard
])
def test_model_of_device_indexing_equals_np_random_normal(case):
    rs = np.random.RandomState(case["seed"])
    if case.get("pre"):
        rs.normal(size=case["pre"])
    st = rs.get_state()
    V, n_rows, skip = case["V"], case["n_rows"], case["skip"]
    r0, r1 = case["rows"]
    rows, end = _model_draw(st, V, skip, r0, r1, case["block_words"])
    rs.normal(0, 1, skip)
    full = rs.normal(0, 1, (n_rows, V))
    assert np.array_equal(rows.view(np.uint64), full[r0:r1].view(np.uint64))
    ref = np.random.RandomState()
    ref.set_state(st)
    ref.normal(0, 1, skip + r1 * V)
    want = ref.get_state()
    assert np.array_equal(end[1], want[1]) and end[2] == want[2] and end[3] == want[3]
    assert np.float64(end[4]).view(np.uint64) == np.float64(want[4]).view(np.uint64)
