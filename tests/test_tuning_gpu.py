"""The tuner's trial on the GPU (tangram_b200.mapping_parameter_tuning) against the unmodified reference's outputs stored
in tests/golden/tuning.npz: the three metric functions on awkward cubes, bit-reproducibility, the whole trial in every
precision, Mapper.train(out=...), and a 100k x 10k x 3 agreement pass that must fit beside almost no free memory."""
import os

import numpy as np
import pytest
import torch

from oracle.tangram_oracle import synthetic_inputs
from tangram_b200 import Mapper
from tangram_b200 import mapping_parameter_tuning as mpt
from tests.helpers import GOLDEN_DIR

pytestmark = pytest.mark.gpu

Z = np.load(os.path.join(GOLDEN_DIR, "tuning.npz"))
METRIC_CASES = ["r2_37x129", "r3_37x129", "r3_64x200", "r5_29x131"]
METRICS = ["cell_map_consistency", "cell_map_agreement", "cell_map_certainty", "gene_expr_consistency",
           "gene_expr_correctness"]
DATA_KEYS = ["S", "G", "d_source", "d", "device", "print_each", "voxel_weights", "ct_encode", "neighborhood_filter",
             "spatial_weights", "train_genes_idx", "val_genes_idx"]


def _check_metrics(name, pearson, vote, cons):
    assert pearson.shape == Z[f"m_{name}_pearson"].shape
    assert np.max(np.abs(pearson - Z[f"m_{name}_pearson"])) < 1e-9
    assert np.array_equal(vote, Z[f"m_{name}_vote"].astype(np.float32))          # discrete: exact
    assert np.max(np.abs(cons - Z[f"m_{name}_consensus"])) < 1e-6


@pytest.mark.parametrize("name", METRIC_CASES)
def test_metric_functions_match_the_reference(name):
    cube = Z[f"m_{name}_cube"]
    _check_metrics(name, mpt.pearson_corr(cube), mpt.vote_entropy(cube), mpt.consensus_entropy(cube))


@pytest.mark.parametrize("name", METRIC_CASES)
def test_metric_functions_on_device_layouts(name):
    """A padded device view (leading dimension a multiple of 4: float4 loads plus a ragged tail) and a list of tensors."""
    cube = Z[f"m_{name}_cube"]
    R, N, V = cube.shape
    pad = torch.full((R, N, V + 7 - (V + 7) % 4 + 4), float("nan"), device="cuda")
    pad[:, :, :V] = torch.from_numpy(cube)
    view = pad[:, :, :V]
    assert view.stride(1) % 4 == 0
    _check_metrics(name, *mpt.agreement(view, vote=True, consensus=True))
    runs = [torch.from_numpy(cube[r]).cuda() for r in range(R)]
    _check_metrics(name, *mpt.agreement(runs, vote=True, consensus=True))


def test_agreement_is_bit_reproducible():
    g = torch.Generator(device="cuda").manual_seed(3)
    cube = torch.softmax(torch.randn((3, 4099, 1001), device="cuda", generator=g) * 3, dim=2)
    a = mpt.agreement(cube, vote=True, consensus=True)
    b = mpt.agreement(cube, vote=True, consensus=True)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def _trial_inputs(name):
    p = f"t_{name}_"
    data = [Z[p + "in_" + k] if p + "in_" + k in Z.files else None for k in DATA_KEYS]
    data[DATA_KEYS.index("device")] = "cuda:0"
    config = {k[len(p + "cfg_"):]: Z[k].item() for k in Z.files if k.startswith(p + "cfg_")}
    return data, config, int(Z[p + "seed"])


def _host_entropies(cube):
    """float64 host evaluation of vote_entropy / consensus_entropy (the reference's formulas)."""
    cube = np.asarray(cube)
    R, N, V = cube.shape
    votes = cube.argmax(axis=2)
    vote = np.empty(N)
    for i in range(N):
        _, c = np.unique(votes[:, i], return_counts=True)
        p = c / R
        vote[i] = -(p * np.log(p)).sum() / np.log(V)
    mean = cube.astype(np.float64).mean(axis=0)
    mean /= mean.sum(axis=1, keepdims=True)
    with np.errstate(divide="ignore", invalid="ignore"):
        plogp = np.where(mean > 0, mean * np.log(mean), 0.0)
    return vote, -plogp.sum(axis=1) / np.log(V)


@pytest.mark.parametrize("precision,tol", [("bf16x3", 1e-4), ("fp32", 1e-4), ("bf16", 1e-2)])
@pytest.mark.parametrize("name", ["default", "spatial"])
def test_trial_matches_the_reference_trial(name, precision, tol):
    data, config, seed = _trial_inputs(name)
    np.random.seed(seed)
    det = {}
    got = mpt.train_multiple_Mapper(config, data, precision=precision, details=det)
    cube = det["cell_cube"].cpu().numpy()
    ref = dict(zip(METRICS, Z[f"t_{name}_metrics"]))
    # argmax flips against the reference may only happen at near-ties of the reference mapping; each flipped row moves
    # the mean vote entropy by at most 1/N
    votes, ref_votes, gap = cube.argmax(axis=2), Z[f"t_{name}_argmax"], Z[f"t_{name}_gap"]
    flipped = votes != ref_votes
    n_rows_flipped = int(flipped.any(axis=0).sum())
    if precision != "bf16":
        assert np.all(gap[flipped] < 1e-4), gap[flipped]
    N = cube.shape[1]
    print(f"{name}/{precision}: " + ", ".join(f"{k} {got[k]:.6f} (ref {ref[k]:.6f})" for k in METRICS)
          + f"; {n_rows_flipped} rows with a flipped vote")
    for k in METRICS:
        allow = tol + (n_rows_flipped / N if k == "cell_map_agreement" else 0.0)
        assert abs(got[k] - ref[k]) < allow, (k, got[k], ref[k])
    # on the trial's own mappings the device entropies equal a float64 host evaluation
    vote, cons = mpt.agreement(det["cell_cube"], pearson=False, vote=True, consensus=True)[1:]
    hv, hc = _host_entropies(cube)
    assert np.max(np.abs(vote - hv)) < 1e-7
    assert np.max(np.abs(cons - hc)) < 1e-6
    assert abs(got["cell_map_agreement"] - (1 - hv.mean())) < 1e-6
    assert abs(got["cell_map_certainty"] - (1 - hc.mean())) < 1e-6


def test_train_out_writes_the_same_mapping_to_the_device():
    inp = synthetic_inputs(500, 130, 60, seed=9)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0)
    M0 = np.random.default_rng(2).standard_normal((500, 130)).astype(np.float32)
    a = Mapper(M0=M0, **kw)
    out_a, hist_a = a.train(25, print_each=None, val_each=5)
    b = Mapper(M0=M0, **kw)
    dst = torch.full((500, 130), float("nan"), device="cuda")
    out_b, hist_b = b.train(25, print_each=None, val_each=5, out=dst)
    assert out_b is dst
    assert np.array_equal(out_a.view(np.uint32), dst.cpu().numpy().view(np.uint32))
    assert np.array_equal(a.history_matrix, b.history_matrix, equal_nan=True)
    assert hist_a.keys() == hist_b.keys()
    for k in hist_a:
        assert np.array_equal(np.array(hist_a[k], np.float64), np.array(hist_b[k], np.float64), equal_nan=True), k
    with pytest.raises(ValueError):
        b.train(1, print_each=None, out=torch.empty((130, 500), device="cuda"))
    with pytest.raises(TypeError):
        b.train(1, print_each=None, out=np.empty((500, 130), np.float32))


def test_c3_agreement_needs_no_mapping_sized_scratch():
    """100k x 10k, R = 3, from mappings drawn on the device: the call must succeed with less free device memory than one
    mapping (4 GB) and leave the free memory as it found it."""
    N, V, R = 100_000, 10_000, 3
    g = torch.Generator(device="cuda").manual_seed(7)
    cube = torch.empty((R, N, V), device="cuda")
    for r in range(R):
        cube[r] = torch.softmax(torch.randn((N, V), device="cuda", generator=g) * 4, dim=1)
    mpt.agreement(cube[:, :64], vote=True, consensus=True)         # kernels loaded before the memory is taken
    mpt.agreement(cube[:, :64])
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    filler = torch.empty(free - (1 << 30), dtype=torch.uint8, device="cuda")   # leave 1 GiB: a quarter of one mapping
    try:
        free0, _ = torch.cuda.mem_get_info()
        assert free0 < N * V * 4
        p, v, c = mpt.agreement(cube, vote=True, consensus=True)
        free1, _ = torch.cuda.mem_get_info()
    finally:
        del filler
    assert abs(free1 - free0) <= 32 << 20          # everything the call allocated (O(rows)) was given back
    assert p.shape == (3,) and np.all(np.abs(p) <= 1) and np.all(np.isfinite(p))
    assert v.shape == (N,) and c.shape == (N,) and np.all(np.isfinite(v)) and np.all(np.isfinite(c))
    assert np.all((v >= 0) & (v <= np.log(R) / np.log(V) + 1e-6)) and np.all((c > 0) & (c < 1))
    # spot-check rows against the host evaluation
    rows = np.arange(0, N, 9973)
    hv, hc = _host_entropies(cube[:, rows].cpu().numpy())
    assert np.max(np.abs(v[rows] - hv)) < 1e-7 and np.max(np.abs(c[rows] - hc)) < 1e-6
