"""state_memory="auto" without a GPU: the library's split planner (tgb200_plan_state) against hand-computed splits in
bf16 and bf16x3, the placement's acceptance by the Python layer and the C-ABI, the fp32 refusal, and the messages of the
check that runs before an auto handle is allocated."""
import ctypes

import pytest

from tangram_b200 import _lib
from tangram_b200.engine import Engine, check_auto_state_fits, check_state_memory, plan_state

MiB = 1 << 20
N, V, K = 20000, 2000, 80
LD = 2048                                  # V rounded up to 64 columns


def page(b):
    """What the planner counts for one allocation: whole 2 MiB pages."""
    return 0 if b <= 0 else -(-b // (2 * MiB)) * 2 * MiB


def state_dev(precision, R, rb):
    """Device bytes of rows [0, R) of M, m / mb, v and of a ring of two slots of rb rows."""
    mb = 2 if precision == "bf16" else 4
    return 2 * page(4 * R * LD) + page(mb * R * LD) + 2 * (2 * page(4 * rb * LD) + page(mb * rb * LD))


def row_bytes(precision):
    return LD * (10 if precision == "bf16" else 12)


def cfg(precision, state_memory="auto", **kw):
    c = _lib.Config(struct_size=ctypes.sizeof(_lib.Config), device=0, n_cells=N, n_voxels=V, n_genes=K,
                    precision=_lib.PREC[precision], density_mode=_lib.DENSITY_CELLS, lambda_g1=1.0, lambda_d=1.0,
                    state_memory=_lib.STATE_MEMORY[state_memory])
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@pytest.fixture
def blocks(monkeypatch):
    """Eight rows per ring slot and no forced split, so that every figure below follows from the arithmetic alone."""
    _lib.load(build_if_missing=False)
    monkeypatch.setenv("TGB200_STATE_BLOCK_ROWS", "8")
    monkeypatch.delenv("TGB200_STATE_RESIDENT_ROWS", raising=False)
    return monkeypatch


def operands(precision):
    """The operand bytes the planner counts, from the device plan: everything but the N resident rows."""
    p = plan_state(cfg(precision, "device"), 1 << 40)
    assert (p.resident_rows, p.block_rows, p.host_bytes) == (N, 0, 0)
    ops = p.device_bytes - state_dev(precision, N, 0)
    assert ops > 0 and ops % (2 * MiB) == 0
    return ops, p.reserve_bytes


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_plan_everything_fits(precision, blocks):
    ops, res = operands(precision)
    assert res >= 1 << 30
    for free in (1 << 40, ops + res + state_dev(precision, N, 0)):           # plenty, and exactly enough
        p = plan_state(cfg(precision), free)
        assert (p.resident_rows, p.block_rows, p.host_bytes) == (N, 0, 0)
        assert p.device_bytes == ops + state_dev(precision, N, 0)
    p = plan_state(cfg(precision), ops + res + state_dev(precision, N, 0) - 1)    # one byte short: rows go to the host
    assert p.resident_rows < N and p.host_bytes > 0


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_plan_only_the_operands_fit(precision, blocks):
    ops, res = operands(precision)
    p = plan_state(cfg(precision), ops + res)
    assert (p.resident_rows, p.block_rows) == (0, 1)
    assert p.host_bytes == N * row_bytes(precision)
    assert p.device_bytes == ops + state_dev(precision, 0, 1)


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
@pytest.mark.parametrize("rows", [1000, 10000, 18000])
def test_plan_in_between(precision, rows, blocks):
    """`rows` rows of state fit besides the operands, the reserve and the rounding of nine allocations: two slots of
    eight rows and rows - 16 resident rows."""
    ops, res = operands(precision)
    free = ops + res + 9 * 2 * MiB + rows * row_bytes(precision) + row_bytes(precision) // 2
    p = plan_state(cfg(precision), free)
    R = rows - 16
    assert (p.resident_rows, p.block_rows) == (R, 8)
    assert p.host_bytes == (N - R) * row_bytes(precision)
    assert p.device_bytes == ops + state_dev(precision, R, 8)
    assert p.device_bytes + p.reserve_bytes <= free


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_plan_small_budget_shrinks_the_ring(precision, blocks):
    """Fewer rows fit than two slots of the block rows: the slots shrink to half of what fits."""
    ops, res = operands(precision)
    p = plan_state(cfg(precision), ops + res + 9 * 2 * MiB + 11 * row_bytes(precision))
    assert (p.resident_rows, p.block_rows) == (1, 5)


@pytest.mark.parametrize("precision", ["bf16", "bf16x3"])
def test_plan_ring_larger_than_the_remainder(precision, blocks):
    """A forced split that leaves fewer host rows than a block: the ring holds just those rows."""
    ops, _ = operands(precision)
    blocks.setenv("TGB200_STATE_RESIDENT_ROWS", str(N - 3))
    p = plan_state(cfg(precision), 1 << 40)
    assert (p.resident_rows, p.block_rows) == (N - 3, 3)
    assert p.host_bytes == 3 * row_bytes(precision)
    assert p.device_bytes == ops + state_dev(precision, N - 3, 3)
    blocks.setenv("TGB200_STATE_RESIDENT_ROWS", str(N + 5))             # clamped to N: the device handle
    p = plan_state(cfg(precision), 0)
    assert (p.resident_rows, p.block_rows, p.host_bytes) == (N, 0, 0)
    blocks.setenv("TGB200_STATE_RESIDENT_ROWS", "0")
    p = plan_state(cfg(precision), 1 << 40)
    assert (p.resident_rows, p.block_rows, p.host_bytes) == (0, 8, N * row_bytes(precision))


def test_plan_host_state_keeps_no_rows(blocks):
    p = plan_state(cfg("bf16", "host"), 1 << 40)
    assert (p.resident_rows, p.block_rows, p.host_bytes) == (0, 8, N * row_bytes("bf16"))


def test_auto_is_accepted_and_fp32_is_refused():
    check_state_memory("auto", "bf16")
    check_state_memory("auto", "bf16x3")
    assert _lib.STATE_MEMORY["auto"] == 2
    with pytest.raises(ValueError, match="state_memory='auto' needs precision 'bf16' or 'bf16x3'"):
        Engine(10, 8, 4, precision="fp32", state_memory="auto")
    lib = _lib.load(build_if_missing=False)
    c = cfg("fp32")
    p = _lib.StatePlan()
    assert lib.tgb200_plan_state(ctypes.byref(c), 1 << 40, ctypes.byref(p)) == -4      # TGB200_ERR_UNSUPPORTED
    assert "state_memory = auto" in lib.tgb200_last_error().decode()
    h = ctypes.c_void_p()
    assert lib.tgb200_create(ctypes.byref(c), ctypes.byref(h)) == -4
    assert "state_memory = auto" in lib.tgb200_last_error().decode()


def test_cabi_accepts_auto():
    """The C-ABI takes TGB200_STATE_AUTO: created, or no sm_90 device here -- never an invalid placement."""
    lib = _lib.load(build_if_missing=False)
    c = _lib.Config(struct_size=ctypes.sizeof(_lib.Config), device=0, n_cells=10, n_voxels=8, n_genes=4,
                    precision=_lib.PREC["bf16"], density_mode=_lib.DENSITY_NONE, lambda_g1=1.0,
                    state_memory=_lib.STATE_MEMORY["auto"])
    h = ctypes.c_void_p()
    st = lib.tgb200_create(ctypes.byref(c), ctypes.byref(h))
    if st == 0:
        r = ctypes.c_int32()
        assert lib.tgb200_resident_rows(h, ctypes.byref(r)) == 0 and r.value == 10
        lib.tgb200_destroy(h)
    assert st in (0, -5), lib.tgb200_last_error()
    c.state_memory = 3
    assert lib.tgb200_create(ctypes.byref(c), ctypes.byref(h)) == -1


def test_auto_check_messages(blocks):
    ops, res = operands("bf16x3")
    free = ops + res + 9 * 2 * MiB + 1016 * row_bytes("bf16x3")                  # 1000 rows resident
    with pytest.raises(_lib.TangramB200Error) as e:
        check_auto_state_fits(cfg("bf16x3"), host_available=1 << 20, device_free=free)
    msg = str(e.value)
    assert "keeps 1000 of 20000 rows on cuda:0" in msg and "other 19000 rows" in msg and "MemAvailable is 0.0 GiB" in msg
    with pytest.raises(_lib.TangramB200Error, match=r"state_memory='auto' needs .* GiB on cuda:0 .* with 0 rows resident"):
        check_auto_state_fits(cfg("bf16x3"), host_available=1 << 40, device_free=ops)
    p = check_auto_state_fits(cfg("bf16x3"), host_available=1 << 40, device_free=free)
    assert p.resident_rows == 1000
    p = check_auto_state_fits(cfg("bf16x3"), host_available=0, device_free=1 << 40)   # no host rows: no host check
    assert p.resident_rows == N and p.host_bytes == 0
