"""Argument checks of state_memory= that need no GPU: unknown placements, fp32 with host state, and the host-memory check
that runs before a host-state handle is allocated."""
import ctypes

import numpy as np
import pytest

from tangram_b200 import Mapper, MapperConstrained, _lib
from tangram_b200.engine import Engine, check_host_state_fits, host_memory_available


@pytest.mark.parametrize("bad", ["disk", "HOST", None, 1])
def test_unknown_state_memory_is_refused(bad):
    with pytest.raises(ValueError, match="state_memory must be one of"):
        Engine(10, 8, 4, precision="bf16", state_memory=bad)
    S, G = np.ones((10, 4), np.float32), np.ones((8, 4), np.float32)
    with pytest.raises(ValueError, match="state_memory must be one of"):
        Mapper(S, G, state_memory=bad)
    with pytest.raises(ValueError, match="state_memory must be one of"):
        MapperConstrained(S, G, None, state_memory=bad)


def test_fp32_host_state_is_refused():
    with pytest.raises(ValueError, match="needs precision 'bf16' or 'bf16x3'"):
        Engine(10, 8, 4, precision="fp32", state_memory="host")


def _create(**fields):
    lib = _lib.load(build_if_missing=False)
    cfg = _lib.Config(struct_size=ctypes.sizeof(_lib.Config), device=0, n_cells=10, n_voxels=8, n_genes=4,
                      precision=_lib.PREC["bf16"], density_mode=_lib.DENSITY_NONE, lambda_g1=1.0)
    for k, v in fields.items():
        setattr(cfg, k, v)
    h = ctypes.c_void_p()
    return lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)), lib.tgb200_last_error().decode()


def test_cabi_checks_state_memory_before_the_device():
    """The C-ABI refuses a bad placement before it looks for a device."""
    st, msg = _create(state_memory=7)
    assert st == -1 and "state_memory" in msg                                # TGB200_ERR_INVALID
    st, msg = _create(state_memory=_lib.STATE_MEMORY["host"], precision=_lib.PREC["fp32"])
    assert st == -4 and "fp32" in msg                                        # TGB200_ERR_UNSUPPORTED


def test_host_memory_check_message():
    # 100k x 24k in bf16x3: 12 B per element of M, m and v on the host
    with pytest.raises(_lib.TangramB200Error) as e:
        check_host_state_fits(100_000, 24_000, 500, "bf16x3", 0, host_available=8 << 30, device_free=80 << 30)
    msg = str(e.value)
    assert "pinned host memory" in msg and "26.8 GiB" in msg and "MemAvailable is 8.0 GiB" in msg
    with pytest.raises(_lib.TangramB200Error, match=r"4\.6 GiB on cuda:0 .* 1\.0 GiB are free"):
        check_host_state_fits(100_000, 10_000, 500, "bf16", 0, host_available=64 << 30, device_free=1 << 30)
    check_host_state_fits(100_000, 10_000, 500, "bf16", 0, host_available=64 << 30, device_free=80 << 30)


def test_host_memory_available_reads_meminfo():
    avail = host_memory_available()
    assert avail is None or avail > 0


def test_cabi_accepts_the_config_without_state_memory():
    """A caller whose tgb200_config ends before state_memory passes the size guard (and keeps its state on the device)."""
    lib = _lib.load(build_if_missing=False)
    cfg = _lib.Config(device=0, n_cells=10, n_voxels=8, n_genes=4, precision=_lib.PREC["bf16"],
                      density_mode=_lib.DENSITY_NONE, lambda_g1=1.0)
    cfg.struct_size = _lib.Config.state_memory.offset
    h = ctypes.c_void_p()
    st = lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h))
    if st == 0:
        lib.tgb200_destroy(h)
    assert st in (0, -5), lib.tgb200_last_error()                 # created, or no sm_90 device here
    cfg.struct_size = ctypes.sizeof(_lib.Config) - 16
    assert lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
