"""The sharded tuner trial without a GPU: the three entry points of the row-sharded agreement pass check their arguments
and refuse loudly without a device, and train_multiple_Mapper(process_group=) refuses a non-NCCL group and more than 8
runs before it touches a device."""
import ctypes

import numpy as np
import pytest


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def test_sharded_agreement_entry_points_check_arguments():
    from tangram_b200 import _lib
    lib = _lib.load()
    fake = (_lib._P * 9)(*([16] * 9))
    buf = np.zeros(64)
    out = buf.ctypes.data_as(ctypes.c_void_p)
    # sample: null arrays or output, R outside 1..8, bad shapes
    assert lib.tgb200_agreement_sample(None, 3, 4, 4, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_sample(fake, 3, 4, 4, 4, None, 0, None) == -1
    assert lib.tgb200_agreement_sample(fake, 0, 4, 4, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_sample(fake, 9, 4, 4, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_sample(fake, 3, 4, 5, 4, out, 0, None) == -1            # ld < cols
    assert b"bad shape" in lib.tgb200_last_error()
    assert lib.tgb200_agreement_sample(fake, 3, 0, 4, 4, out, 0, None) == -1
    # partials: null shift or sums, R, shapes
    assert lib.tgb200_agreement_partials(fake, 3, 4, 4, 4, None, out, None, None, 0, None) == -1
    assert lib.tgb200_agreement_partials(fake, 3, 4, 4, 4, out, None, None, None, 0, None) == -1
    assert lib.tgb200_agreement_partials(None, 3, 4, 4, 4, out, out, None, None, 0, None) == -1
    assert lib.tgb200_agreement_partials(fake, 9, 4, 4, 4, out, out, None, None, 0, None) == -1
    assert lib.tgb200_agreement_partials(fake, 3, 4, 0, 4, out, out, None, None, 0, None) == -1
    assert b"bad shape" in lib.tgb200_last_error()
    # pearson: null sums or output, R, element count
    assert lib.tgb200_agreement_pearson(None, 3, 4, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_pearson(out, 3, 4, 4, None, 0, None) == -1
    assert lib.tgb200_agreement_pearson(out, 0, 4, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_pearson(out, 9, 4, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_pearson(out, 3, 0, 4, out, 0, None) == -1
    assert lib.tgb200_agreement_pearson(out, 3, 4, -1, out, 0, None) == -1
    assert b"bad shape" in lib.tgb200_last_error()
    if not _has_gpu():
        for rc in (lib.tgb200_agreement_sample(fake, 3, 4, 4, 4, out, 0, None),
                   lib.tgb200_agreement_partials(fake, 3, 4, 4, 4, out, out, out, out, 0, None),
                   lib.tgb200_agreement_pearson(out, 3, 4, 4, out, 0, None)):
            assert rc == -5
            assert b"no CPU fallback" in lib.tgb200_last_error()


def _trial_data():
    S = np.ones((6, 3), dtype=np.float32)
    G = np.ones((5, 3), dtype=np.float32)
    return [S, G, None, None, "cuda:0", None, None, None, None, None, [0, 1, 2], [0, 1]]


def test_sharded_trial_refusals():
    """A gloo group cannot run the sharded validation; more than 8 runs cannot be scored.  Both are refused before the
    device is touched."""
    import torch.distributed as dist

    from tangram_b200 import mapping_parameter_tuning as mpt
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        with pytest.raises(ValueError, match="needs an NCCL process group"):
            mpt.train_multiple_Mapper({"num_epochs": 2}, _trial_data(), process_group=dist.group.WORLD)
        with pytest.raises(ValueError, match="at most 8 runs"):
            mpt.train_multiple_Mapper({"num_epochs": 2}, _trial_data(), n_runs=9, process_group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_sharded_agreement_refuses_without_gpu():
    import torch.distributed as dist

    from tangram_b200 import _lib
    from tangram_b200 import mapping_parameter_tuning as mpt
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
            mpt.agreement(np.full((3, 4, 5), 0.2, dtype=np.float32), process_group=dist.group.WORLD)
    finally:
        dist.destroy_process_group()
