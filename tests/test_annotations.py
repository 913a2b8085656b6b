"""Annotation transfer without a GPU: every device call refuses loudly, the C entry point validates its arguments, the golden
file is self-consistent (its stored reference outputs follow from its stored mappings in numpy float64), the host-only
segmentation ports equal the reference's outputs, the validation messages are the reference's, and MiniAnnData.varm
follows subsetting and copies."""
import ctypes
import gzip
import os
import pickle

import numpy as np
import pandas as pd
import pytest

from tests.helpers import GOLDEN_DIR

Z = np.load(os.path.join(GOLDEN_DIR, "annotations.npz"))
with open(os.path.join(GOLDEN_DIR, "annotations_frames.pkl.gz"), "rb") as _f:
    FRAMES = pickle.loads(gzip.decompress(_f.read()))
CASES = ["mixed", "wide", "single", "fout", "huge"]
SEGMENTED = ["mixed", "wide", "fout"]


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def test_public_names():
    import tangram_b200 as tg
    from tangram_b200 import utils
    for name in ("project_cell_annotations", "cell_type_mapping", "count_cell_annotations", "create_segment_cell_df",
                 "deconvolve_cell_annotations", "df_to_cell_types", "annotate"):
        assert getattr(tg, name) is getattr(utils, name)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure mode")
def test_device_calls_refuse_without_gpu():
    from tangram_b200 import MiniAnnData, _lib
    from tangram_b200 import utils
    X = np.full((4, 3), 0.25, dtype=np.float32)
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        utils.annotate(X, [0, 1, 0, -1], 2)
    obs = pd.DataFrame({"cell_type": list("abab")}, index=list("wxyz"))
    ad_map = MiniAnnData(X=X, obs=obs)
    ad_sp = MiniAnnData(X=np.zeros((3, 1), np.float32), obs=ad_map.var.copy())
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        utils.project_cell_annotations(ad_map, ad_sp)
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        utils.cell_type_mapping(ad_map, cell_types_key="cell_type")
    d = FRAMES["fout"]
    ad_sp.obsm.update(spatial=np.zeros((3, 2)), image_features=d["image_features"].iloc[:3])
    utils.create_segment_cell_df(ad_sp)
    with pytest.raises(_lib.TangramB200Error, match="no CPU fallback"):
        utils.count_cell_annotations(ad_map, ad_map, ad_sp)
    assert "tangram_ct_pred" not in ad_sp.obsm and "ct_map" not in ad_map.varm and "tangram_ct_count" not in ad_sp.obsm


def test_annotate_entry_point_checks_arguments():
    from tangram_b200 import _lib
    lib = _lib.load()
    fake = ctypes.c_void_p(256)
    lab = np.array([0, 1, -1, 2], dtype=np.int32)
    sums = np.empty((3, 4))
    args = (_lib.ptr(lab), 3, _lib.ptr(sums), None, 0, None)
    assert lib.tgb200_annotate(None, 4, 4, 4, *args) == -1
    assert lib.tgb200_annotate(fake, 4, 5, 4, *args) == -1                  # ld < cols
    assert b"bad shape" in lib.tgb200_last_error()
    assert lib.tgb200_annotate(fake, 4, 4, 4, _lib.ptr(lab), 2, _lib.ptr(sums), None, 0, None) == -1
    assert b"label 2 of row 3 is outside [-1, 2)" in lib.tgb200_last_error()
    bad = np.array([0, -2, 0, 0], dtype=np.int32)
    assert lib.tgb200_annotate(fake, 4, 4, 4, _lib.ptr(bad), 3, _lib.ptr(sums), None, 0, None) == -1
    assert b"label -2 of row 1" in lib.tgb200_last_error()
    if not _has_gpu():
        assert lib.tgb200_annotate(fake, 4, 4, 4, *args) == -5
        assert b"no CPU fallback" in lib.tgb200_last_error()


@pytest.mark.parametrize("case", CASES)
def test_golden_file_is_consistent(case):
    """The stored reference sums and argmax follow from the stored mapping and labels, and the awkward cases are there."""
    X, codes, pred, amax = Z[f"{case}_X"], Z[f"{case}_codes"], Z[f"{case}_pred"], Z[f"{case}_argmax"]
    N, V = X.shape
    assert X.dtype == np.float32 and codes.shape == (N,) and pred.shape[0] == V
    T = pred.shape[1]
    expect = np.stack([X[codes == t].astype(np.float64).sum(axis=0) for t in range(T)], axis=1)
    assert np.allclose(pred, expect, rtol=1e-12, atol=0)
    assert np.array_equal(amax, X.argmax(axis=1))
    top = X.max(axis=1, keepdims=True)
    assert ((X == top).sum(axis=1) > 1).mean() > 0.8                                # most rows have a tied maximum
    if V > 1024:                                                                    # ties across 1024-column slabs
        first, last = X.argmax(axis=1), V - 1 - X[:, ::-1].argmax(axis=1)
        assert ((first < 1024) & (last >= 1024)).any()
    names = list(FRAMES[case]["obs"]["cell_type"])
    assert [pd.isna(n) for n in names] == list(codes < 0)
    if case == "mixed":
        assert (codes == codes[17]).sum() == 1 and (codes < 0).sum() == 3
        b = list(FRAMES[case]["pred"].columns).index("B")
        assert (pred[:200, b] == 0).all() and (pred[200:, b] > 0).any()         # a label absent from a column range
    assert {"mixed": 7, "wide": 70, "single": 1, "fout": 4, "huge": 2}[case] == T
    assert (case != "huge") or V > 65535


@pytest.mark.parametrize("case", SEGMENTED)
def test_segmentation_ports_equal_the_reference(case):
    from tangram_b200 import MiniAnnData, utils
    d = FRAMES[case]
    V = len(d["var"])
    ad_sp = MiniAnnData(X=np.zeros((V, 1), np.float32), obs=d["var"].copy(),
                        obsm={"image_features": d["image_features"], "spatial": d["spatial"]})
    utils.create_segment_cell_df(ad_sp)
    pd.testing.assert_frame_equal(ad_sp.uns["tangram_cell_segmentation"], d["segmentation"])
    pd.testing.assert_series_equal(ad_sp.obsm["tangram_spot_centroids"], d["spot_centroids"])
    counts = [k for k in d if k.startswith("count_")]
    ad_sp.obsm["tangram_ct_count"] = d[counts[-1]]                 # the reference's last count, which it deconvolved
    ad_sp.obsm["tangram_ct_pred"] = d["pred"]
    got = utils.deconvolve_cell_annotations(ad_sp, filter_cell_annotation=d["deconv_filter"])
    pd.testing.assert_frame_equal(got.obs, d["deconv_obs"])
    assert np.array_equal(got.obsm["spatial"], d["deconv_obs"][["y", "x"]].to_numpy())
    assert got.uns is ad_sp.uns
    # the default filter (every tangram_ct_pred column) works and takes the types in column order
    default = utils.deconvolve_cell_annotations(ad_sp).obs
    assert set(default["centroids"]) == set(got.obs["centroids"])
    assigned = utils.df_to_cell_types(d[counts[-1]], list(d["deconv_filter"]))
    assert sorted(assigned) == sorted(d["deconv_filter"])
    assert sum(len(v) for v in assigned.values()) >= len(got.obs)


def test_validation_messages_are_the_references():
    from tangram_b200 import MiniAnnData, utils
    ad = MiniAnnData(X=np.zeros((2, 2), np.float32))
    with pytest.raises(ValueError, match=r"^Missing parameter for tangram deconvolution\. Run `sqidpy\.im\.calculate_image_"):
        utils.create_segment_cell_df(ad)
    with pytest.raises(ValueError, match=r"^Missing spatial information in AnnDatas\. Please make sure coordinates are "
                                         r"saved with AnnData\.obsm\['spatial'\]$"):
        utils.count_cell_annotations(ad, ad, ad)
    ad.obsm["spatial"] = np.zeros((2, 2))
    with pytest.raises(ValueError, match=r"^Missing parameter for tangram deconvolution\. Run `sqidpy\.im\.calculate"):
        utils.count_cell_annotations(ad, ad, ad)
    ad.obsm["image_features"] = FRAMES["fout"]["image_features"].iloc[:2]
    with pytest.raises(ValueError, match=r"^Missing parameter for tangram deconvolution\. Run `create_segment_cell_df`\.$"):
        utils.count_cell_annotations(ad, ad, ad)
    with pytest.raises(ValueError, match=r"^Missing tangram parameters\. Run `count_cell_annotations`\.$"):
        utils.deconvolve_cell_annotations(ad)


def test_miniadata_varm_follows_subsets_and_copies():
    from tangram_b200 import MiniAnnData
    var = pd.DataFrame(index=[f"g{i}" for i in range(5)])
    ct = pd.DataFrame({"a": np.arange(5.0), "b": np.arange(5.0) * 2}, index=var.index)
    ad = MiniAnnData(X=np.ones((3, 5), np.float32), var=var, varm={"ct_map": ct, "arr": np.arange(10).reshape(5, 2)})
    sub = ad[:, ["g3", "g1"]]
    pd.testing.assert_frame_equal(sub.varm["ct_map"], ct.iloc[[3, 1]])
    assert np.array_equal(sub.varm["arr"], [[6, 7], [2, 3]])
    assert ad[[0, 2]].varm["ct_map"].shape == (5, 2)                 # a row subset keeps every gene
    cp = ad.copy()
    pd.testing.assert_frame_equal(cp.varm["ct_map"], ct)
    cp.varm["ct_map"].iloc[0, 0] = -1.0
    assert ad.varm["ct_map"].iloc[0, 0] == 0.0                       # the copy does not share the frame
    ad._inplace_subset_var(np.array([True, False, True, False, False]))
    pd.testing.assert_frame_equal(ad.varm["ct_map"], ct.iloc[[0, 2]])
    assert MiniAnnData(X=np.ones((1, 1))).varm == {}
