"""
Golden outputs of the annotation transfer (tangram/utils.py: project_cell_annotations, cell_type_mapping,
create_segment_cell_df, count_cell_annotations, deconvolve_cell_annotations) from the REAL reference.

Needs a Tangram checkout: the one next to this repository, or the one TANGRAM_REFERENCE names (as oracle/build_ref.py):
    python tests/golden/make_annotations_golden.py

The unmodified reference utils.py is loaded by path as `tangram.utils`; `tangram.mapping_utils` is an empty stub module
(these functions do not use it) and `scanpy` a stub whose AnnData is this repository's MiniAnnData.  Writes
  tests/golden/annotations.npz          per case <c>_X (the N x V float32 mapping), <c>_codes (each cell's one-hot
                                        column, -1 for a NaN label), <c>_pred (tangram_ct_pred), <c>_argmax (np.argmax)
  tests/golden/annotations_frames.pkl.gz  per case the AnnData inputs (obs, var, spatial features) and the reference's
                                        output frames, as plain pandas objects (the 66001-column case keeps only obs:
                                        its spots are spot0, spot1, ... and its output is <c>_pred)
Cases: exact argmax ties inside a float4, across warps and across 1024-column slabs; a label with one cell, a NaN label, a
label whose cells are zero over a column range; T = 1 and T = 70; V = 517, 1030 (ragged, over one slab) and 66001 (more
than 65535 columns, five rows); F_out with values below, at and above the thresholds 0.3 and 0.5.
"""
import gzip
import importlib.util
import os
import pickle
import sys
import types

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tangram_b200.adata import MiniAnnData  # noqa: E402

REF = os.environ.get("TANGRAM_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")


class _SizedAnnData(MiniAnnData):
    """count_cell_annotations' F_out branch takes len(adata_sc), as of a real AnnData."""

    def __len__(self):
        return self.n_obs


def load_reference():
    pkg = types.ModuleType("tangram")
    pkg.__path__ = []
    sys.modules["tangram"] = pkg
    sys.modules["tangram.mapping_utils"] = types.ModuleType("tangram.mapping_utils")
    sc = types.ModuleType("scanpy")
    sc.AnnData = lambda X=None, obs=None, **kw: MiniAnnData(X=X, obs=obs, **kw)
    sys.modules["scanpy"] = sc
    spec = importlib.util.spec_from_file_location("tangram.utils", os.path.join(REF, "tangram", "utils.py"))
    ut = importlib.util.module_from_spec(spec)
    sys.modules["tangram.utils"] = ut
    spec.loader.exec_module(ut)
    return ut


def mapping(rng, N, V, density=0.4):
    """Quantised non-negative values (k / 1024, most of them zero): exact ties come naturally and the file compresses."""
    X = rng.integers(1, 1024, (N, V)).astype(np.float32) / 1024
    X[rng.random((N, V)) > density] = 0.0
    return X


def set_ties(X, pairs):
    """Row i gets its maximum at both columns of pairs[i % len(pairs)] (and nowhere else)."""
    for i in range(X.shape[0]):
        a, b = pairs[i % len(pairs)]
        top = X[i].max() + 0.5
        X[i, a] = X[i, b] = top


def segmentation(rng, V, spot_names):
    n = rng.integers(0, 4, V)
    n[0] = 2                  # the reference builds its frame from a list of (y, x) pairs: it must not start with a NaN
    features = pd.DataFrame({"segmentation_label": n,
                             "segmentation_centroid": [[(float(rng.random()), float(rng.random())) for _ in range(k)]
                                                       for k in n]}, index=spot_names)
    return features, rng.random((V, 2))


CASES = {
    # name: N, V, labels, seed, ties, extras
    "mixed": dict(N=301, V=517, seed=1, ties=[(4, 5), (6, 100), (127, 128), (0, 516), (511, 515)]),
    "wide": dict(N=120, V=1030, seed=2, ties=[(1023, 1024), (100, 1028), (127, 128), (0, 1029), (1024, 1029)]),
    "single": dict(N=40, V=33, seed=3, ties=[(1, 2), (0, 32)]),
    "fout": dict(N=200, V=130, seed=4, ties=[(3, 64), (31, 32)]),
    "huge": dict(N=5, V=66001, seed=5, ties=[(65535, 65536), (1023, 66000), (7, 40000)]),
}


def labels_for(name, rng, N):
    if name == "mixed":
        lab = rng.choice(["B", "T", "NK", "Mono", "DC"], N).astype(object)
        lab[17] = "solo"                                  # a label with one cell
        lab[[5, 50, 200]] = np.nan                        # a NaN label: a column, but no cell contributes to it
        return lab
    if name == "wide":
        return np.array([f"L{i % 70:02d}" for i in rng.permutation(N)], dtype=object)   # T = 70
    if name == "single":
        return np.array(["only"] * N, dtype=object)
    if name == "fout":
        return rng.choice(["a", "b", "c", "d"], N).astype(object)
    return np.array(["p", "q", "p", "q", "p"], dtype=object)


def main():
    ut = load_reference()
    arrays, frames = {}, {}
    for name, c in CASES.items():
        rng = np.random.default_rng(c["seed"])
        N, V = c["N"], c["V"]
        X = mapping(rng, N, V, density=0.4 if V < 60000 else 0.002)
        set_ties(X, c["ties"])
        lab = labels_for(name, rng, N)
        if name == "mixed":
            X[lab == "B", :200] = 0.0                     # a label absent from a whole column range
        cells = [f"cell{i}" for i in range(N)]
        spots = [f"spot{j}" for j in range(V)]
        obs = pd.DataFrame({"cell_type": lab}, index=cells)
        var = pd.DataFrame(index=spots)
        if name == "fout":
            f = rng.random(N)
            f[::7] = 0.5                                  # exactly at the 0.5 threshold (>= keeps, > drops)
            f[1::9] = 0.3
            obs["F_out"] = f
        ad_map = MiniAnnData(X=X, obs=obs.copy(), var=var.copy())
        ad_sp = MiniAnnData(X=np.zeros((V, 2), np.float32), obs=var.copy())
        ut.project_cell_annotations(ad_map, ad_sp, annotation="cell_type")
        out = {"obs": obs, "var": var, "pred": ad_sp.obsm["tangram_ct_pred"]}
        if "F_out" not in obs:                            # the reference fails there whenever a cell is filtered out
            ad_ct = MiniAnnData(X=X, obs=obs.copy(), var=var.copy())
            ut.cell_type_mapping(ad_ct, cell_types_key="cell_type")
            out["ct_map"] = ad_ct.varm["ct_map"]
        if name in ("mixed", "wide", "fout"):
            features, spatial = segmentation(rng, V, spots)
            ad_sp.obsm["image_features"] = features
            ad_sp.obsm["spatial"] = spatial
            ut.create_segment_cell_df(ad_sp)
            out.update(image_features=features, spatial=spatial,
                       segmentation=ad_sp.uns["tangram_cell_segmentation"],
                       spot_centroids=ad_sp.obsm["tangram_spot_centroids"])
            # label-based obs[annotation][k] in the F_out branch: a RangeIndex makes it positional
            ad_sc = _SizedAnnData(X=np.zeros((N, 1), np.float32), obs=obs[["cell_type"]].reset_index(drop=True))
            for thr in ((0.5, 0.3) if name == "fout" else (0.5,)):
                ut.count_cell_annotations(ad_map, ad_sc, ad_sp, annotation="cell_type", threshold=thr)
                out[f"count_{thr}"] = ad_sp.obsm["tangram_ct_count"]
            filt = np.array(list(ad_sp.obsm["tangram_ct_pred"].columns), dtype=object)
            filt = filt[pd.notna(filt)][::-1]             # explicit, in another order than the columns
            out["deconv_filter"] = filt
            out["deconv_obs"] = ut.deconvolve_cell_annotations(ad_sp, filter_cell_annotation=filt).obs
        columns = list(out["pred"].columns)
        pos = pd.Index(columns).get_indexer(pd.Series(lab))
        arrays[f"{name}_X"] = X
        arrays[f"{name}_codes"] = np.where(pd.isna(lab), -1, pos).astype(np.int32)
        arrays[f"{name}_pred"] = out["pred"].to_numpy()
        arrays[f"{name}_argmax"] = np.argmax(X, axis=1).astype(np.int32)
        if name == "huge":
            out = {"obs": obs}
        frames[name] = out
        print(name, X.shape, "labels", len(columns), "outputs", sorted(out))
    np.savez_compressed(os.path.join(HERE, "annotations.npz"), **arrays)
    with open(os.path.join(HERE, "annotations_frames.pkl.gz"), "wb") as f:
        f.write(gzip.compress(pickle.dumps(frames, protocol=4), mtime=0))
    for fn in ("annotations.npz", "annotations_frames.pkl.gz"):
        print("->", fn, os.path.getsize(os.path.join(HERE, fn)) // 1024, "KiB")


if __name__ == "__main__":
    main()
