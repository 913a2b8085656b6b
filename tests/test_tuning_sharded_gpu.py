"""The row-sharded agreement pass (tgb200_agreement_sample / _partials / _pearson) and the sharded tuner trial
(train_multiple_Mapper(process_group=)) on one GPU.

Row splits.  A cube is cut into blocks of rows, each block is one shard: its sample sums are added in float64 on the host
and divided, its partials are taken about that shared shift and added in float64 on the host, and the Pearson values come
from the sums with the whole cube's element count.  They are checked against np.corrcoef in float64 within
tests/test_agreement_gpu.py's a-priori bound (`_reference`), evaluated with the shared shift and with the longest
addition chain of the split: the deepest block's chain (`_kernel_depth` of its rows) plus one addition per block on the
host.  Covered: every R = 1..8, one-row blocks, blocks that end inside a warp stride (not on a multiple of the 8 rows a
CTA takes at a time), 20011 rows cut into three blocks, common offsets of 1e3 to 1e4 (where the unshifted one-pass sums
through the same entry points miss the bound) and one block whose mean lies far from the others.  Each block's per-row
entropies equal the matching rows of the unsharded tgb200_agreement, bit for bit, and one block holding every row gives
tgb200_agreement's Pearson bits.

Trial.  On a one-rank NCCL group, train_multiple_Mapper(process_group=) on the `default` and `spatial` trial inputs of
tests/golden/tuning.npz returns the unsharded trial's metrics, cubes and validation scores bit for bit, and leaves numpy's
generator where the unsharded trial leaves it.  A gloo group is refused before anything is drawn.  With one rank every
all-reduce is the identity: tests/test_tuning_sharded_multigpu.py, on two GPUs, checks the sums.
"""
import ctypes

import numpy as np
import pytest
import torch

from tangram_b200 import _lib
from tangram_b200 import mapping_parameter_tuning as mpt
from tests import test_agreement_gpu as tag
from tests.test_tuning_gpu import _trial_inputs

pytestmark = pytest.mark.gpu


def _call(fn, *args):
    _lib.check(fn(*args))


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream(0).cuda_stream)


def _ptrs(runs):
    return (_lib._P * len(runs))(*[r.data_ptr() for r in runs])


def _split(cube, cuts):
    """(R, N, V) CUDA cube -> its row blocks [0, c0), [c0, c1), ..., [c_last, N) as lists of R (rows, V) views."""
    edges = [0] + list(cuts) + [cube.shape[1]]
    return [list(cube[:, a:b].unbind(0)) for a, b in zip(edges[:-1], edges[1:])]


def _sharded(blocks, rows=False, shift=None):
    """The three entry points over row blocks, the sums added in float64 on the host in block order.
    -> (pearson, [per block (vote, cons) or None], shared shift, summed sample)."""
    lib = _lib.load()
    R, V = len(blocks[0]), blocks[0][0].shape[1]
    ld = blocks[0][0].stride(0)
    sample = np.zeros(R + 1)
    for b in blocks:
        s = np.empty(R + 1)
        _call(lib.tgb200_agreement_sample, _ptrs(b), R, b[0].shape[0], V, ld, _lib.ptr(s), 0, _stream())
        sample += s
    if shift is None:
        shift = sample[:R] / sample[R]
    shift = np.ascontiguousarray(shift, dtype=np.float64)
    NS = R + R * (R + 1) // 2
    sums, per_block = np.zeros(NS), []
    for b in blocks:
        n = b[0].shape[0]
        part = np.empty(NS)
        v, c = (np.empty(n, np.float32), np.empty(n, np.float32)) if rows else (None, None)
        _call(lib.tgb200_agreement_partials, _ptrs(b), R, n, V, ld, _lib.ptr(shift), _lib.ptr(part), _lib.ptr(v),
              _lib.ptr(c), 0, _stream())
        sums += part
        per_block.append((v, c) if rows else None)
    p = np.empty(R * (R - 1) // 2)
    _call(lib.tgb200_agreement_pearson, _lib.ptr(sums), R, sum(b[0].shape[0] for b in blocks), V, _lib.ptr(p), 0,
          _stream())
    return p, per_block, shift, sample


def _block_sample(runs):
    """float64 sums and size of one block's shift sample, from its definition (tests/test_agreement_gpu._shift)."""
    N, V = runs[0].shape
    total = N * V
    ns = min(total, tag.SAMPLE)
    k = torch.arange(ns, device=runs[0].device, dtype=torch.int64)
    e = total // ns * k + (total % ns) * k // ns
    return torch.stack([r[e // V, e % V] for r in runs]).double().sum(1).cpu().numpy(), ns


def _reference(cube, blocks, shift, monkeypatch):
    """tests/test_agreement_gpu._reference with the split's shared shift and its longest addition chain."""
    N, V = cube.shape[1:]
    depth = max(tag._kernel_depth(b[0].shape[0], V) for b in blocks) + len(blocks)
    c = torch.from_numpy(shift).cuda()
    with monkeypatch.context() as m:
        m.setattr(tag, "_shift", lambda runs: c)
        m.setattr(tag, "_kernel_depth", lambda n, v: depth)
        return tag._reference(list(cube.unbind(0)))


def _check_split(what, cube, cuts, monkeypatch):
    blocks = _split(cube, cuts)
    R = cube.shape[0]
    p, per_block, shift, sample = _sharded(blocks, rows=True)
    # the shared shift: the blocks' samples added, as their definition gives them
    want = [_block_sample(b) for b in blocks]
    assert sample[R] == sum(ns for _, ns in want)
    np.testing.assert_allclose(sample[:R], np.sum([s for s, _ in want], axis=0), rtol=1e-12, atol=1e-300)
    ref = _reference(cube, blocks, shift, monkeypatch)
    r = tag._close(what + " pearson", p, ref["pearson"], ref["pearson_bound"])
    # the per-row entropies: the unsharded call's rows, bit for bit
    _, v, c = mpt.agreement(cube, pearson=False, vote=True, consensus=True)
    edges = [0] + list(cuts) + [cube.shape[1]]
    for (bv, bc), a, b in zip(per_block, edges[:-1], edges[1:]):
        assert np.array_equal(bv.view(np.uint32), v[a:b].view(np.uint32)), f"{what}: vote entropy of rows {a}:{b}"
        assert np.array_equal(bc.view(np.uint32), c[a:b].view(np.uint32)), f"{what}: consensus entropy of rows {a}:{b}"
    print(f"{what}: {len(blocks)} blocks, Pearson max err / bound {r:.3g}")
    return p, ref


# (R, rows, cols, cuts): every R; one-row blocks at the start, in the middle and at the end; cuts off the 8-row stride a
# CTA takes (13, 101, 5003); 20011 rows in three blocks; float4 bodies with a tail (260, 1001) and the scalar path
SPLITS = [
    (1, 7, 5, [3]),
    (2, 20011, 4, [1]),
    (3, 20011, 5, [6700, 13401]),
    (4, 2000, 128, [13, 1999]),
    (5, 777, 129, [100, 101]),
    (6, 8, 127, [4]),
    (7, 9, 1001, [8]),
    (8, 20011, 260, [5003, 12011]),
]


@pytest.mark.parametrize("R,N,V,cuts", SPLITS)
def test_row_splits_against_float64(R, N, V, cuts, monkeypatch):
    cube = tag._softmax_cube(R, N, V, seed=R * 100 + V)
    _check_split(f"R={R} {N}x{V} cut at {cuts}", cube, cuts, monkeypatch)


def test_common_offsets_need_the_shared_shift(monkeypatch):
    """Runs of offset_r + unit noise, offsets 1e3 .. 1e4 (test_agreement_gpu's offsets case), cut into three blocks:
    within the bound about the shared shift; the same blocks summed about a zero shift miss it."""
    rng = np.random.default_rng(11)
    R, N, V = 4, 2000, 1000
    z = rng.standard_normal((N, V))
    off, a, b = [1e3, 2.5e3, 5e3, 1e4], [1.0, 0.8, -0.9, 0.3], [0.5, 1.0, 0.4, 1.0]
    x = np.stack([off[r] + a[r] * z + b[r] * rng.standard_normal((N, V)) for r in range(R)]).astype(np.float32)
    cube = torch.from_numpy(x).cuda()
    cuts = [333, 1501]
    _, ref = _check_split("offsets", cube, cuts, monkeypatch)
    assert np.any(ref["pearson"] < -0.5) and np.any(ref["pearson"] > 0.5)
    p0 = _sharded(_split(cube, cuts), shift=np.zeros(R))[0]
    miss = np.abs(p0 - ref["pearson"]) / ref["pearson_bound"]
    print(f"zero shift: err / bound {miss.min():.3g} .. {miss.max():.3g}")
    assert np.all(miss > 1), miss


def test_one_block_far_from_the_others(monkeypatch):
    """Ten rows of 1000 + noise between blocks of unit noise: the shared shift is pulled away from the global mean by the
    far block's sample, and the bound holds about it."""
    g = torch.Generator(device="cuda").manual_seed(21)
    R, N, V = 3, 3000, 300
    base = torch.randn((N, V), device="cuda", generator=g)
    cube = torch.stack([base + 0.5 * (r + 1) * torch.randn((N, V), device="cuda", generator=g) for r in range(R)])
    cube[:, 1000:1010] += 1000.0
    _check_split("far block", cube, [1000, 1010], monkeypatch)


@pytest.mark.parametrize("R,N,V", [(2, 20011, 4), (3, 4099, 1001), (8, 777, 129)])
def test_one_block_is_the_unsharded_call(R, N, V):
    cube = tag._softmax_cube(R, N, V, seed=7 + R)
    want = mpt.agreement(cube)[0]
    got = _sharded(_split(cube, []))[0]
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (got, want)


@pytest.fixture
def nccl_group(monkeypatch):
    """A one-rank NCCL process group on cuda:0."""
    import torch.distributed as dist
    monkeypatch.setenv("NCCL_SOCKET_IFNAME", "lo")
    torch.cuda.set_device(0)
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


def test_agreement_on_a_one_rank_group(nccl_group):
    cube = tag._softmax_cube(3, 4099, 1001, seed=3)
    want = mpt.agreement(cube, vote=True, consensus=True)
    got = mpt.agreement(cube, vote=True, consensus=True, process_group=nccl_group)
    for w, g in zip(want, got):
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8))


def _rng_state():
    _, key, pos, has_gauss, gauss = np.random.get_state()
    return key.tobytes(), pos, has_gauss, gauss


@pytest.mark.parametrize("name", ["default", "spatial"])
def test_trial_on_a_one_rank_group(name, nccl_group):
    data, config, seed = _trial_inputs(name)
    np.random.seed(seed)
    ref_det = {}
    want = mpt.train_multiple_Mapper(config, data, details=ref_det)
    want_state = _rng_state()
    np.random.seed(seed)
    det = {}
    got = mpt.train_multiple_Mapper(config, data, details=det, process_group=nccl_group)
    assert _rng_state() == want_state
    print(f"{name}: {got}")
    assert got == want
    assert det["shard_rows"] == (0, data[0].shape[0])
    for k in ("cell_cube", "gene_cube"):
        assert torch.equal(det[k].view(torch.int32), ref_det[k].view(torch.int32)), k
    assert det["val_gene_sim"] == ref_det["val_gene_sim"]


def test_gloo_group_is_refused_before_training():
    import torch.distributed as dist
    data, config, seed = _trial_inputs("default")
    np.random.seed(seed)
    state = _rng_state()
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        with pytest.raises(ValueError, match="needs an NCCL process group"):
            mpt.train_multiple_Mapper(config, data, process_group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
    assert _rng_state() == state, "the refused trial drew from numpy's generator"
