"""Tangram's post-mapping utilities (tangram/utils.py) on the sm_90a (H100) library:

    project_genes(adata_map, adata_sc)                         :338-374  gene expression onto space
    project_cell_annotations(adata_map, adata_sp, annotation)  :126-153  annotation probabilities per spot
    cell_type_mapping(adata_map, cell_types_key)               :820-842  the same, min-max normalised per annotation
    count_cell_annotations(adata_map, adata_sc, adata_sp)      :205-285  cells per spot and annotation
    create_segment_cell_df(adata_sp), deconvolve_cell_annotations(adata_sp), df_to_cell_types(df, cell_types)
                                                               :156-202, 288-335, 790-818  host-side segmentation frames

The annotation calls read the mapping once on the device (`annotate`, tgb200_annotate): per-label fp64 column sums
instead of the reference's float64 upcast GEMM, and the row argmax instead of np.argmax over the host array.  There is
no CPU path.
"""
import ctypes

import numpy as np
import pandas as pd

from . import _lib
from . import mapping_utils as mu
from .adata import make_adata
from .engine import _require_device

_ANN_CHUNK, _ANN_SLAB = 128, 1024       # rows per work item and columns per slab of tgb200_annotate


def project_genes(adata_map, adata_sc, cluster_label=None, scale=True):
    adata_sc.var.index = [g.lower() for g in adata_sc.var.index]                 # :353
    adata_sc.var_names_make_unique()                                              # :356
    keep = np.asarray((adata_sc.X != 0).sum(axis=0)).reshape(-1) >= 1             # :359
    if not keep.all():
        adata_sc = adata_sc[:, keep]
    if cluster_label:
        adata_sc = mu.adata_to_cluster_expression(adata_sc, cluster_label, scale=scale)
    if not adata_map.obs.index.equals(adata_sc.obs.index):
        raise ValueError("The two AnnDatas need to have same `obs` index.")
    X = adata_sc.X.toarray() if hasattr(adata_sc.X, "toarray") else np.asarray(adata_sc.X)
    mapper = getattr(adata_map, "_tgb200_mapper", None)
    if mapper is not None and mapper.n_cells == X.shape[0]:
        X_space = mapper.project(X)               # softmax(M)^T X on the device (:368 is a host GEMM)
    else:
        X_space = np.asarray(adata_map.X).T @ X
    adata_ge = make_adata(X=X_space, obs=adata_map.var, var=adata_sc.var, uns=adata_sc.uns)
    training_genes = adata_map.uns["train_genes_df"].index.values
    adata_ge.var["is_training"] = adata_ge.var.index.isin(training_genes)
    return adata_ge


def _annotate_device_bytes(rows, cols, n_labels, sums, argmax):
    """Device scratch tgb200_annotate allocates for these sizes (at most)."""
    b = 8 * rows
    if sums:
        b += 8 * cols * (rows // _ANN_CHUNK + 2 * n_labels + 1)
    if argmax:
        b += 8 * rows * -(-cols // _ANN_SLAB) + 4 * rows
    return b


def annotate(mapping, labels, n_labels, *, sums=True, argmax=False, device=None):
    """One pass of tgb200_annotate over the (N, V) `mapping` (numpy array or CUDA tensor; read as float32).

    `labels`: N integers in [-1, n_labels); rows labelled -1 are left out.  Returns (sums, argmax):
      sums    (n_labels, V) float64, sums[t] = the sum of the rows labelled t, or None
      argmax  (N,) int32, the first column holding each labelled row's maximum (np.argmax, NaN counting as the maximum),
              -1 for unlabelled rows, or None
    Host data is copied to the device once (`device`, default the current CUDA device); device data is read where it
    lives, with its row stride.  Free device memory is checked first."""
    import torch
    n_labels = int(n_labels)
    if isinstance(mapping, torch.Tensor) and mapping.is_cuda:
        dev = mapping.device.index
        X = mapping
    else:
        dev = _require_device("cuda" if device is None else device)
        X = np.asarray(mapping)
    if X.ndim != 2:
        raise ValueError(f"expected an (N, V) mapping, got shape {tuple(X.shape)}")
    N, V = (int(n) for n in X.shape)
    lab = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
    if lab.shape[0] != N:
        raise ValueError(f"{lab.shape[0]} labels for a mapping of {N} rows")
    if N == 0:
        return (np.zeros((n_labels, V)) if sums else None), (np.empty(0, np.int32) if argmax else None)
    upload = not isinstance(X, torch.Tensor) or X.dtype != torch.float32 or X.stride(1) != 1 or X.stride(0) < V
    need = _annotate_device_bytes(N, V, n_labels, sums, argmax) + (4 * N * V if upload else 0)
    free, _ = torch.cuda.mem_get_info(dev)
    if need > free:
        raise _lib.TangramB200Error(
            f"annotate needs about {need / 2**30:.2f} GiB on cuda:{dev} for a {N} x {V} mapping and {n_labels} labels "
            f"({4 * N * V / 2**30 if upload else 0:.2f} GiB of it to hold the mapping); {free / 2**30:.2f} GiB are free")
    if isinstance(X, torch.Tensor):
        if upload:
            X = X.float().contiguous()
    else:
        X = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(f"cuda:{dev}")
    out_s = np.empty((n_labels, V), dtype=np.float64) if sums else None
    out_a = np.empty(N, dtype=np.int32) if argmax else None
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    lib = _lib.load()
    _lib.check(lib.tgb200_annotate(_lib._P(X.data_ptr()), N, V, X.stride(0), _lib.ptr(lab), n_labels, _lib.ptr(out_s),
                                   _lib.ptr(out_a), dev, stream))
    return out_s, out_a


def _label_columns(series):
    """-> (the one-hot columns of tangram/utils.py:105-123 for `series`: its unique values in order of first appearance, a
    NaN included, each row's position among them).  The positions are taken by position, whatever the index."""
    values = pd.Series(series).reset_index(drop=True)
    columns = pd.unique(values)
    codes = pd.Index(columns).get_indexer(values)
    return columns, values, codes


def _one_hot_codes(series):
    """-> (one-hot columns, per-row column for the one-hot product): a NaN label has a column but matches no row there
    (NaN == NaN is false in one_hot_encoding), so its rows add nothing."""
    columns, values, codes = _label_columns(series)
    return columns, np.where(values.isna().to_numpy(), -1, codes)


def _mapping_of(adata_map):
    X = adata_map.X
    return X.toarray() if hasattr(X, "toarray") else X


def project_cell_annotations(adata_map, adata_sp, annotation="cell_type", threshold=0.5):
    """:126-153 -- transfer `annotation` from the cells onto space: adata_sp.obsm["tangram_ct_pred"] becomes a float64
    (spots x annotations) DataFrame indexed by adata_map.var.index, its columns the annotations in order of first
    appearance, entry [j, t] the mapping probability of spot j summed over the cells annotated t.

    `threshold` has no effect, as in the reference: it filters the cells by adata_map.obs["F_out"] > threshold into a
    variable that is overwritten before use (:144-147), so every cell counts.  The sums are taken on the device in fp64."""
    columns, codes = _one_hot_codes(adata_map.obs[annotation])
    sums, _ = annotate(_mapping_of(adata_map), codes, len(columns))
    adata_sp.obsm["tangram_ct_pred"] = pd.DataFrame(sums.T, index=adata_map.var.index, columns=pd.Index(list(columns)))


def cell_type_mapping(adata_map, cell_types_key="cell_types"):
    """:820-842 -- adata_map.varm["ct_map"]: the (spots x cell types) sums of project_cell_annotations, min-max
    normalised per cell type (a constant column gives NaN, as in the reference).

    Where adata_map.obs has "F_out" (constrained mode), only the cells with F_out >= 0.5 count, each with its own label.
    The reference raises a shape error there whenever a cell is filtered out (:835 multiplies the filtered mapping by the
    unfiltered one-hot frame); where no cell is filtered out the result is the reference's.  The columns are the labels of
    all cells, so a type whose cells are all filtered out has a zero, and so NaN, column."""
    columns, codes = _one_hot_codes(adata_map.obs[cell_types_key])
    if "F_out" in adata_map.obs.keys():
        codes = np.where(np.asarray(adata_map.obs["F_out"]) >= 0.5, codes, -1)
    sums, _ = annotate(_mapping_of(adata_map), codes, len(columns))
    df = pd.DataFrame(sums.T, index=adata_map.var.index, columns=pd.Index(list(columns)))
    vmin, vmax = df.min(), df.max()
    adata_map.varm["ct_map"] = (df - vmin) / (vmax - vmin)


def create_segment_cell_df(adata_sp):
    """:156-202 -- one row per segmented cell: adata_sp.uns["tangram_cell_segmentation"] gets the columns 'spot_idx'
    (the spot's obs name), 'y', 'x' and 'centroids' (the cell's id "<spot>_<k>"; a spot without cells keeps one row of
    NaN), and adata_sp.obsm["tangram_spot_centroids"] the per-spot arrays of cell ids.  Needs
    adata_sp.obsm["image_features"] (squidpy's segmentation features)."""
    if "image_features" not in adata_sp.obsm.keys():
        raise ValueError("Missing parameter for tangram deconvolution. Run `sqidpy.im.calculate_image_features`.")
    features = adata_sp.obsm["image_features"]
    per_spot = features[["segmentation_centroid"]].copy()
    per_spot["centroids_idx"] = [np.array([f"{spot}_{k}" for k in range(n)], dtype="object")
                                 for spot, n in zip(adata_sp.obs.index.values, features["segmentation_label"])]
    coords = per_spot["segmentation_centroid"].explode()
    seg = pd.DataFrame(coords.to_list(), columns=["y", "x"], index=coords.index)
    seg["centroids"] = per_spot["centroids_idx"].explode().values
    seg.index.set_names("spot_idx", inplace=True)
    seg.reset_index(drop=False, inplace=True)
    adata_sp.uns["tangram_cell_segmentation"] = seg
    adata_sp.obsm["tangram_spot_centroids"] = per_spot["centroids_idx"]


def count_cell_annotations(adata_map, adata_sc, adata_sp, annotation="cell_type", threshold=0.5):
    """:205-285 -- adata_sp.obsm["tangram_ct_count"]: per spot its coordinates 'x', 'y', its segmented cell count
    'cell_n', its cell ids 'centroids', and per annotation (adata_sc.obs[annotation], in order of first appearance) the
    number of cells whose most probable spot it is.  Where adata_map.obs has "F_out", only the cells with
    F_out > threshold are counted.

    The most probable spot of each counted cell is the device row argmax of the mapping (first spot on ties, as
    np.argmax); the counts are one np.bincount.  Annotations are read by position in adata_sc.obs."""
    if "spatial" not in adata_sp.obsm.keys():
        raise ValueError(
            "Missing spatial information in AnnDatas. Please make sure coordinates are saved with AnnData.obsm['spatial']")
    if "image_features" not in adata_sp.obsm.keys():
        raise ValueError("Missing parameter for tangram deconvolution. Run `sqidpy.im.calculate_image_features`.")
    if "tangram_cell_segmentation" not in adata_sp.uns.keys() or "tangram_spot_centroids" not in adata_sp.obsm.keys():
        raise ValueError("Missing parameter for tangram deconvolution. Run `create_segment_cell_df`.")
    spatial = np.asarray(adata_sp.obsm["spatial"])
    df = pd.DataFrame(data={"x": spatial[:, 1], "y": spatial[:, 0],
                            "cell_n": adata_sp.obsm["image_features"]["segmentation_label"],
                            "centroids": adata_sp.obsm["tangram_spot_centroids"]},
                      index=list(adata_sp.obs.index))
    columns, _, codes = _label_columns(adata_sc.obs[annotation])
    X = _mapping_of(adata_map)
    N, n = X.shape[0], min(X.shape[0], len(codes))     # cells beyond adata_sc's are not counted (the reference zips)
    labels = np.full(N, -1, dtype=np.int64)
    labels[:n] = codes[:n]
    if "F_out" in adata_map.obs.keys():
        labels[~(np.asarray(adata_map.obs["F_out"]) > threshold)] = -1
    keep = labels >= 0
    _, spot = annotate(X, np.minimum(labels, 0), 1, sums=False, argmax=True)
    counts = np.bincount(spot[keep].astype(np.int64) * len(columns) + labels[keep],
                         minlength=len(df) * len(columns)).reshape(len(df), len(columns))
    for t, c in enumerate(columns):
        df[c] = counts[:, t].astype(np.int64)
    adata_sp.obsm["tangram_ct_count"] = df


def df_to_cell_types(df, cell_types):
    """:790-818 -- {cell type: cell ids} from per-spot counts: in each spot (row of `df`), the ids in df["centroids"] are
    handed out in order, the first count of them to the first type of `cell_types`, the next to the second, and so on.
    Columns not in `cell_types` are ignored."""
    cum = df[cell_types].cumsum(axis=1).to_numpy()
    centroids = df["centroids"].to_numpy()
    mapped = {}
    for t, name in enumerate(cell_types):
        ids = mapped.setdefault(name, [])
        for r in range(len(df)):
            start = cum[r, t - 1] if t > 0 else 0
            ids.extend(np.asarray(centroids[r])[start:cum[r, t]].tolist())
    return mapped


def deconvolve_cell_annotations(adata_sp, filter_cell_annotation=None):
    """:288-335 -- one AnnData row per segmented cell with an assigned annotation: obs has 'y', 'x', 'centroids' and
    'cluster' (the annotation), obsm["spatial"] the (y, x) coordinates, uns is adata_sp.uns.  The cells of each spot are
    assigned from adata_sp.obsm["tangram_ct_count"] by df_to_cell_types; `filter_cell_annotation` (default: every column
    of adata_sp.obsm["tangram_ct_pred"]) names the annotations taken, in order."""
    if "tangram_ct_count" not in adata_sp.obsm.keys() or "tangram_cell_segmentation" not in adata_sp.uns.keys():
        raise ValueError("Missing tangram parameters. Run `count_cell_annotations`.")
    if filter_cell_annotation is None:
        filter_cell_annotation = adata_sp.obsm["tangram_ct_pred"].columns
    cell_types = pd.unique(np.asarray(list(filter_cell_annotation), dtype=object))
    assigned = df_to_cell_types(adata_sp.obsm["tangram_ct_count"], cell_types)
    clusters = pd.concat([pd.DataFrame({"centroids": np.array(ids, dtype="object"), "cluster": name})
                          for name, ids in assigned.items()], axis=0).reset_index(drop=True)
    cells = adata_sp.uns["tangram_cell_segmentation"].merge(clusters, on="centroids", how="inner")
    cells = cells.drop(columns="spot_idx").drop_duplicates().dropna().reset_index(drop=True)
    adata_segment = make_adata(X=np.zeros(cells.shape), obs=cells)
    adata_segment.obsm["spatial"] = cells[["y", "x"]].to_numpy()
    adata_segment.uns = adata_sp.uns
    return adata_segment
