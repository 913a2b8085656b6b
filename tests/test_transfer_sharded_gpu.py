"""Gene projection and annotation transfer from a cell-sharded mapping on one H100, with the real kernels
(tgb200_annotate, tgb200_project_map) on each rank's rows:

* on a one-rank NCCL group, each of project_genes, project_cell_annotations, cell_type_mapping and
  count_cell_annotations is bit-identical to its call without a group;
* two- and three-process gloo groups on cuda:0 hold uneven blocks of the golden mappings (tests/golden/annotations.npz):
  every rank gets the same results, equal to the reference's golden outputs within the bounds of
  tests/test_annotations_gpu.py (the counts and deconvolved cells exactly), and a CSR adata_sc.X gives the same
  project_genes result as a dense one, bit for bit.
"""
import numpy as np
import pandas as pd
import pytest
import torch

from tests.test_transfer_sharded_gloo import (CASES, Z, _calls_worker, check_against_golden, check_genes,
                                              check_ranks_agree, rel_fro, spawn, transfer)

pytestmark = pytest.mark.gpu


def n_cells(case):
    return Z[f"{case.split('_')[0]}_X"].shape[0]


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


@pytest.mark.parametrize("case", CASES)
def test_one_rank_nccl_group_is_bit_identical(case, nccl_group):
    N = n_cells(case)
    got = transfer(case, 0, N, nccl_group)
    want = transfer(case, 0, N, None)
    assert sorted(got) == sorted(want)
    for key, w in want.items():
        if key == "ge":
            g = got["ge"]
            assert g["X"].dtype == w["X"].dtype == np.float32
            assert np.array_equal(g["X"].view(np.uint32), w["X"].view(np.uint32))
            pd.testing.assert_frame_equal(g["var"], w["var"])
            pd.testing.assert_frame_equal(g["obs"], w["obs"])
        else:
            pd.testing.assert_frame_equal(got[key], w, check_exact=True, obj=f"{case} {key}")
            if key in ("pred", "ct_map"):
                a, b = got[key].to_numpy(), w.to_numpy()
                assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), key


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ranks_on_one_gpu_equal_the_golden_outputs(world):
    want = {case: transfer(case, 0, n_cells(case), None) for case in CASES}
    ranks = spawn(_calls_worker, world, False)
    check_ranks_agree(ranks)
    for r, got in enumerate(ranks):
        for case in CASES:
            check_against_golden(case, got[case], 1e-10, 1e-10)
            check_genes(got[case]["ge"], want[case]["ge"], 1e-6)
            base = case.split("_")[0]
            S = want[case]["ge"]["S"].toarray().astype(np.float64)[:, [k for k in range(24) if k != 5]]
            assert rel_fro(got[case]["ge"]["X"], Z[f"{base}_X"].astype(np.float64).T @ S) <= 1e-5
        # the device projection gives the same bits from a CSR and a dense adata_sc.X
        assert np.array_equal(got["dense_sc"].view(np.uint32), got["mixed"]["ge"]["X"].view(np.uint32)), r
