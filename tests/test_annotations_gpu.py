"""Annotation transfer on the GPU (tgb200_annotate behind tangram_b200.utils) against the unmodified reference's outputs
in tests/golden/annotations.npz and annotations_frames.pkl.gz: tangram_ct_pred, ct_map, tangram_ct_count, the argmax with
its ties, the deconvolved cells; then bit-reproducibility, padded device layouts, NaN in the argmax, the F_out rule of
cell_type_mapping, and a 100k x 10k, T = 32 call against torch float64 on the same GPU."""
import gzip
import os
import pickle

import numpy as np
import pandas as pd
import pytest
import torch

from tangram_b200 import MiniAnnData, utils
from tests.helpers import GOLDEN_DIR

pytestmark = pytest.mark.gpu

Z = np.load(os.path.join(GOLDEN_DIR, "annotations.npz"))
with open(os.path.join(GOLDEN_DIR, "annotations_frames.pkl.gz"), "rb") as _f:
    FRAMES = pickle.loads(gzip.decompress(_f.read()))
CASES = ["mixed", "wide", "single", "fout", "huge"]
SEGMENTED = ["mixed", "wide", "fout"]


def _adatas(case):
    d, X = FRAMES[case], Z[f"{case}_X"]
    var = d["var"] if "var" in d else pd.DataFrame(index=[f"spot{j}" for j in range(X.shape[1])])
    ad_map = MiniAnnData(X=X, obs=d["obs"].copy(), var=var.copy())
    ad_sp = MiniAnnData(X=np.zeros((X.shape[1], 1), np.float32), obs=var.copy())
    return ad_map, ad_sp


def _close(got, ref, rtol):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.all(np.abs(got[ok] - ref[ok]) <= rtol * np.abs(ref[ok])), np.max(np.abs(got[ok] - ref[ok]))


@pytest.mark.parametrize("case", CASES)
def test_project_cell_annotations_matches_the_reference(case):
    ad_map, ad_sp = _adatas(case)
    utils.project_cell_annotations(ad_map, ad_sp, annotation="cell_type")
    got = ad_sp.obsm["tangram_ct_pred"]
    assert all(got.dtypes == np.float64)
    _close(got.to_numpy(), Z[f"{case}_pred"], 1e-10)
    if "pred" in FRAMES[case]:
        pd.testing.assert_frame_equal(got, FRAMES[case]["pred"], rtol=1e-10)
    else:
        assert got.index.equals(ad_map.var.index) and len(got.columns) == Z[f"{case}_pred"].shape[1]


@pytest.mark.parametrize("case", [c for c in CASES if "ct_map" in FRAMES[c]])
def test_cell_type_mapping_matches_the_reference(case):
    ad_map, _ = _adatas(case)
    utils.cell_type_mapping(ad_map, cell_types_key="cell_type")
    got, ref = ad_map.varm["ct_map"], FRAMES[case]["ct_map"]
    assert got.index.equals(ref.index) and got.columns.equals(ref.columns) and all(got.dtypes == np.float64)
    g, r = got.to_numpy(), ref.to_numpy()
    assert np.array_equal(np.isnan(g), np.isnan(r))
    assert np.nanmax(np.abs(g - r)) <= 1e-10


@pytest.mark.parametrize("case", CASES)
def test_argmax_matches_numpy_ties_included(case):
    X, codes = Z[f"{case}_X"], Z[f"{case}_codes"]
    _, a = utils.annotate(X, np.zeros(len(X), np.int32), 1, sums=False, argmax=True)
    assert np.array_equal(a, Z[f"{case}_argmax"])
    s, a = utils.annotate(X, codes, Z[f"{case}_pred"].shape[1], argmax=True)       # both outputs from one pass
    assert np.array_equal(a, np.where(codes >= 0, Z[f"{case}_argmax"], -1))
    _close(s.T, Z[f"{case}_pred"], 1e-10)


@pytest.mark.parametrize("case", SEGMENTED)
def test_count_and_deconvolve_match_the_reference(case):
    d = FRAMES[case]
    ad_map, ad_sp = _adatas(case)
    ad_sp.obsm.update(image_features=d["image_features"], spatial=d["spatial"])
    utils.project_cell_annotations(ad_map, ad_sp, annotation="cell_type")
    utils.create_segment_cell_df(ad_sp)
    ad_sc = MiniAnnData(X=np.zeros((len(d["obs"]), 1), np.float32), obs=d["obs"][["cell_type"]].copy())
    for key in [k for k in d if k.startswith("count_")]:
        utils.count_cell_annotations(ad_map, ad_sc, ad_sp, annotation="cell_type", threshold=float(key[len("count_"):]))
        pd.testing.assert_frame_equal(ad_sp.obsm["tangram_ct_count"], d[key])
    got = utils.deconvolve_cell_annotations(ad_sp, filter_cell_annotation=d["deconv_filter"])
    pd.testing.assert_frame_equal(got.obs, d["deconv_obs"])


def test_two_calls_are_bit_identical():
    g = torch.Generator(device="cuda").manual_seed(5)
    P = torch.softmax(torch.randn((20_011, 3_001), device="cuda", generator=g) * 3, dim=1)
    lab = np.random.default_rng(0).integers(-1, 40, P.shape[0]).astype(np.int32)
    a = utils.annotate(P, lab, 40, argmax=True)
    b = utils.annotate(P, lab, 40, argmax=True)
    assert np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64)) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("V", [1030, 1031])
def test_padded_device_tensor_equals_the_host_array(V):
    """A CUDA view with a leading dimension larger than V: a multiple of 4 (float4 loads, ragged tail) or not (scalar)."""
    rng = np.random.default_rng(V)
    X = (rng.integers(0, 64, (333, V)) / 64).astype(np.float32)
    lab = rng.integers(-1, 5, 333).astype(np.int32)
    host = utils.annotate(X, lab, 5, argmax=True)
    pad = torch.full((333, V + 9), float("nan"), device="cuda")
    pad[:, :V] = torch.from_numpy(X)
    view = pad[:, :V]
    assert view.stride(0) == V + 9
    dev = utils.annotate(view, lab, 5, argmax=True)
    assert np.array_equal(host[0], dev[0]) and np.array_equal(host[1], dev[1])
    assert np.array_equal(host[1], np.where(lab >= 0, X.argmax(axis=1), -1))
    _close(host[0], np.stack([X[lab == t].astype(np.float64).sum(0) for t in range(5)]), 1e-12)


def test_nan_counts_as_the_maximum():
    X = np.random.default_rng(1).random((6, 2100)).astype(np.float32)
    X[0, 1500] = np.nan
    X[1, [7, 1100]] = np.nan                          # first NaN wins
    X[2, 2099] = np.nan
    X[3] = -np.inf                                    # all equal: column 0
    _, a = utils.annotate(X, np.zeros(6, np.int32), 1, sums=False, argmax=True)
    assert np.array_equal(a, np.argmax(X, axis=1))


def test_cell_type_mapping_keeps_the_cells_that_pass_f_out():
    """Where F_out filters cells out the reference raises; here the kept cells count with their own labels."""
    ad_map, _ = _adatas("fout")
    X, f = Z["fout_X"], ad_map.obs["F_out"].to_numpy()
    labels = ad_map.obs["cell_type"].to_numpy()
    assert (f < 0.5).any() and (f == 0.5).any()
    utils.cell_type_mapping(ad_map, cell_types_key="cell_type")
    columns = list(pd.unique(labels))
    keep = f >= 0.5
    raw = np.stack([X[keep & (labels == c)].astype(np.float64).sum(0) for c in columns], axis=1)
    model = (raw - raw.min(0)) / (raw.max(0) - raw.min(0))
    got = ad_map.varm["ct_map"]
    assert list(got.columns) == columns and got.index.equals(ad_map.var.index)
    assert np.max(np.abs(got.to_numpy() - model)) <= 1e-10
    # without F_out the same call equals project_cell_annotations, normalised
    del ad_map.obs["F_out"]
    utils.cell_type_mapping(ad_map, cell_types_key="cell_type")
    pred = FRAMES["fout"]["pred"]
    assert np.max(np.abs(ad_map.varm["ct_map"].to_numpy() - ((pred - pred.min()) / (pred.max() - pred.min())).to_numpy())) \
        <= 1e-10


def test_c3_sized_call_matches_torch_float64():
    N, V, T = 100_000, 10_000, 32
    g = torch.Generator(device="cuda").manual_seed(11)
    P = torch.softmax(torch.randn((N, V), device="cuda", generator=g) * 4, dim=1)
    lab = torch.randint(0, T, (N,), device="cuda", generator=g)
    sums, amax = utils.annotate(P, lab.cpu().numpy(), T, argmax=True)
    E = torch.nn.functional.one_hot(lab, T).double()
    ref = (P.double().T @ E).T.cpu().numpy()
    assert np.max(np.abs(sums - ref) / np.abs(ref)) < 1e-10
    assert np.array_equal(amax, P.argmax(dim=1).int().cpu().numpy())
