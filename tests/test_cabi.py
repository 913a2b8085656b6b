"""The C-ABI boundary: the library loads, exports every symbol include/tangram_b200.h declares,
the ctypes mirror of tgb200_config matches the C layout, and -- without a GPU -- the product
path fails loudly instead of falling back to anything.  No compute calls here."""
import ctypes
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "tangram_b200.h")


def declared_symbols():
    text = open(HEADER).read()
    return sorted(set(re.findall(r"TGB200_API\s+[\w\s\*]+?\b(tgb200_\w+)\s*\(", text)))


def test_header_declares_expected_surface():
    syms = declared_symbols()
    for must in ("tgb200_create", "tgb200_run", "tgb200_step_begin", "tgb200_step_end", "tgb200_get_mapping",
                 "tgb200_get_history", "tgb200_project", "tgb200_last_error", "tgb200_destroy"):
        assert must in syms


def test_library_exports_every_declared_symbol():
    from tangram_b200 import _lib
    lib = _lib.load()
    for name in declared_symbols():
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature"
    assert set(_lib.SIGNATURES) == set(declared_symbols())
    assert b"sm_90a" in lib.tgb200_version()


def test_config_struct_layout_matches_c(tmp_path):
    from tangram_b200 import _lib
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "tangram_b200.h"\n'
                   'int main(){printf("%zu %zu %zu %zu\\n", sizeof(tgb200_config), offsetof(tgb200_config, n_cells_global),'
                   ' offsetof(tgb200_config, lambda_g1), offsetof(tgb200_config, adam_eps));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, o1, o2, o3 = map(int, subprocess.check_output([str(exe)]).split())
    assert size == ctypes.sizeof(_lib.Config)
    assert o1 == _lib.Config.n_cells_global.offset
    assert o2 == _lib.Config.lambda_g1.offset
    assert o3 == _lib.Config.adam_eps.offset


def test_header_is_plain_c():
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-fsyntax-only", "-x", "c", HEADER])


def _has_gpu():
    import torch
    return torch.cuda.is_available()


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_no_gpu_fails_loudly_no_cpu_fallback():
    import numpy as np
    from tangram_b200 import Mapper, _lib
    S = np.ones((4, 3), dtype=np.float32)
    G = np.ones((5, 3), dtype=np.float32)
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback|CUDA"):
        Mapper(S, G, device="cuda:0", random_state=1)
    with pytest.raises(ValueError, match="H100 GPUs only"):
        Mapper(S, G, device="cpu", random_state=1)


def test_bad_config_is_rejected_before_touching_the_device():
    from tangram_b200 import _lib
    lib = _lib.load()
    cfg = _lib.Config()
    cfg.struct_size = 4   # wrong on purpose
    h = ctypes.c_void_p()
    assert lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    assert b"struct_size" in lib.tgb200_last_error()
    cfg.struct_size = ctypes.sizeof(_lib.Config)
    cfg.n_cells, cfg.n_voxels, cfg.n_genes = 4, 4, 4
    cfg.lambda_g1 = 0.0
    assert lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
    assert b"lambda_g1 cannot be 0" in lib.tgb200_last_error()
    # a shard of fewer global cells than its own rows would count itself sharded and divide the density by the wrong N
    cfg.lambda_g1 = 1.0
    for n_global in (1, 3):
        cfg.n_cells_global = n_global
        assert lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)) == -1
        assert f"n_cells_global={n_global} < n_cells=4".encode() in lib.tgb200_last_error()
        assert not h.value
    assert lib.tgb200_destroy(None) == 0


def test_mapper_refuses_fewer_global_cells_than_rows_given():
    """Mapper(n_cells_global=) below the rows of S is refused before any device work (so also without a GPU)."""
    import numpy as np
    from tangram_b200 import Mapper
    S = np.ones((6, 3), dtype=np.float32)
    G = np.ones((5, 3), dtype=np.float32)
    with pytest.raises(ValueError, match="n_cells_global=5 is smaller than the 6 rows"):
        Mapper(S, G, device="cuda:0", M0=np.zeros((6, 5), dtype=np.float32), n_cells_global=5)


@pytest.mark.gpu
def test_integration_stub_runs():
    """The ctypes block of INTEGRATION.md section 3, executed verbatim (only N, V, K, S, G, d, M0 and the library path are
    supplied from here), must run and agree with the oracle."""
    import numpy as np
    from oracle.tangram_oracle import OracleMapper, synthetic_inputs
    from tangram_b200 import _build, _lib
    _lib.load()                                               # builds the library if needed
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    block = re.search(r"## 3\. The ctypes stub.*?```python\n(.*?)```", text, re.S).group(1)
    block = block.replace('ctypes.CDLL("libtangram_b200.so")', f'ctypes.CDLL({_build.LIB!r})')
    N, V, K = 300, 70, 40
    inp = synthetic_inputs(N, V, K, seed=5)
    M0 = np.random.default_rng(1).standard_normal((N, V))
    env = dict(N=N, V=V, K=K, S=inp["S"], G=inp["G"], d=inp["d"], M0=M0)
    block = block.replace("1000", "30")                       # epochs (run / history calls)
    exec(compile(block, "INTEGRATION.md", "exec"), env)
    o = OracleMapper(S=inp["S"], G=inp["G"], d=inp["d"], lambda_g1=1.0, lambda_d=1.0, M0=M0.astype(np.float32))
    ref_out, ref_hist = o.train(30, learning_rate=0.1, print_each=None)
    assert np.allclose(env["hist"][:, 0], np.array([float(x) for x in ref_hist["total_loss"]]), rtol=1e-4, atol=1e-6)
    assert np.linalg.norm(env["out"] - ref_out) / np.linalg.norm(ref_out) < 1e-4


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU behaviour")
def test_host_pin_without_gpu_reports_an_error_and_leaves_the_buffer_usable():
    """The result-buffer helper is optional plumbing: with no device it must return an error code (never crash), and
    Mapper.train's _ResultBuffer then simply keeps the pageable array."""
    import numpy as np
    from tangram_b200 import _lib
    from tangram_b200.mapping_optimizer import _ResultBuffer
    lib = _lib.load()
    buf = np.empty(1 << 20, dtype=np.float32)
    assert lib.tgb200_host_pin(_lib.ptr(buf), buf.nbytes, 4, 0) != 0
    assert lib.tgb200_last_error()
    buf[:] = 1.0
    old = _ResultBuffer.MIN_BYTES
    _ResultBuffer.MIN_BYTES = 1 << 10
    try:
        r = _ResultBuffer(lib, (64, 64), 0)
        arr = r.ready()
        assert arr.shape == (64, 64) and not r._pinned
        r.release()
    finally:
        _ResultBuffer.MIN_BYTES = old
