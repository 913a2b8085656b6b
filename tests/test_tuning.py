"""The tuner's trial without a GPU: the module imports, every call refuses loudly instead of computing on the host, the
C entry point validates its arguments, and the golden file is self-consistent (its stored reference outputs follow from
its stored cubes by the reference's formulas)."""
import ctypes
import os

import numpy as np
import pytest
import scipy.stats

from tests.helpers import GOLDEN_DIR

GOLDEN = os.path.join(GOLDEN_DIR, "tuning.npz")
METRIC_CASES = ["r2_37x129", "r3_37x129", "r3_64x200", "r5_29x131"]


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def test_import_without_gpu():
    import tangram_b200 as tg
    from tangram_b200 import mapping_parameter_tuning as mpt
    assert tg.train_multiple_Mapper is mpt.train_multiple_Mapper
    for name in ("pearson_corr", "vote_entropy", "consensus_entropy", "train_multiple_Mapper"):
        assert callable(getattr(mpt, name))


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_metrics_and_trial_refuse_without_gpu():
    from tangram_b200 import _lib
    from tangram_b200 import mapping_parameter_tuning as mpt
    cube = np.full((3, 4, 5), 0.2, dtype=np.float32)
    for fn in (mpt.pearson_corr, mpt.vote_entropy, mpt.consensus_entropy):
        with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
            fn(cube)
    S = np.ones((4, 3), dtype=np.float32)
    G = np.ones((5, 3), dtype=np.float32)
    data = [S, G, None, None, "cuda:0", None, None, None, None, None, [0, 1, 2], [0, 1]]
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        mpt.train_multiple_Mapper({"num_epochs": 2}, data)
    data[4] = "cpu"
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        mpt.train_multiple_Mapper({"num_epochs": 2}, data)


def test_agreement_entry_point_checks_arguments():
    from tangram_b200 import _lib
    lib = _lib.load()
    fake = (_lib._P * 9)(*([16] * 9))
    assert lib.tgb200_agreement(None, 3, 4, 4, 4, None, None, None, 0, None) == -1
    assert lib.tgb200_agreement(fake, 0, 4, 4, 4, None, None, None, 0, None) == -1
    assert lib.tgb200_agreement(fake, 9, 4, 4, 4, None, None, None, 0, None) == -1
    assert lib.tgb200_agreement(fake, 3, 4, 5, 4, None, None, None, 0, None) == -1       # ld < cols
    assert b"bad shape" in lib.tgb200_last_error()
    if not _has_gpu():
        out = np.empty(3)
        assert lib.tgb200_agreement(fake, 3, 4, 4, 4, out.ctypes.data_as(ctypes.c_void_p), None, None, 0, None) == -5
        assert b"no CPU fallback" in lib.tgb200_last_error()


def test_golden_file_is_consistent():
    assert os.path.getsize(GOLDEN) < 1 << 20
    z = np.load(GOLDEN)
    for name in METRIC_CASES:
        cube = z[f"m_{name}_cube"]
        R, N, V = cube.shape
        assert cube.dtype == np.float32
        p = np.corrcoef(cube.reshape(R, -1))[np.tril_indices(R, -1)]
        assert np.allclose(z[f"m_{name}_pearson"], p, rtol=0, atol=1e-12)
        votes = cube.argmax(axis=2)
        counts = np.stack([(votes == votes[r]).sum(axis=0) for r in range(R)])        # votes for each run's choice
        h = np.zeros(N)
        for i in range(N):
            _, c = np.unique(votes[:, i], return_counts=True)
            h[i] = scipy.stats.entropy(c / R) / np.log(V)
        assert np.allclose(z[f"m_{name}_vote"], h, rtol=0, atol=1e-12)
        assert (counts < R).any() and (counts == R).any()                             # agreeing and split votes
        mean = cube.astype(np.float64).mean(axis=0)
        assert np.allclose(z[f"m_{name}_consensus"], scipy.stats.entropy(mean, axis=1) / np.log(V), rtol=0, atol=1e-6)
        # the awkward cases are present: exact argmax ties and exact zeros
        top = cube.max(axis=2, keepdims=True)
        assert ((cube == top).sum(axis=2) > 1).any()
        assert (cube == 0).any() and (cube.sum(axis=0) == 0).any()
    for name in ("default", "spatial"):
        p = f"t_{name}_"
        S, G = z[p + "in_S"], z[p + "in_G"]
        m = z[p + "metrics"]
        assert m.shape == (5,) and np.all(np.isfinite(m)) and np.all((m > 0) & (m <= 1))
        assert z[p + "argmax"].shape == (3, S.shape[0]) and z[p + "argmax"].max() < G.shape[0]
        assert z[p + "gap"].shape == (3, S.shape[0]) and (z[p + "gap"] >= 0).all()
        assert int(z[p + "cfg_num_epochs"]) in range(50, 101)
