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

project_genes and the three annotation calls take process_group=: `adata_map` is then the rank's block of a cell-sharded
mapping (map_cells_to_space(process_group=)), each rank computes its partial sums from its own rows with the same
kernels, the partials are added over the group, and every rank gets the result of the whole mapping, with no gather.
They run (and an NCCL group sums) on torch's current CUDA device: each rank calls torch.cuda.set_device(rank) first.
"""
import ctypes
import logging

import numpy as np
import pandas as pd

from . import _lib
from . import mapping_utils as mu
from .adata import make_adata
from .engine import _device_index, _require_device

_ANN_CHUNK, _ANN_SLAB = 128, 1024       # rows per work item and columns per slab of tgb200_annotate


def _dense(X):
    return X.toarray() if hasattr(X, "toarray") else np.asarray(X)


def _sm90_device(mapping):
    """The device project_genes contracts on: the CUDA device of a tensor `mapping`, else torch's current one, when it is
    an sm_90 device; None otherwise (then the host GEMM is the only path)."""
    import torch
    if not torch.cuda.is_available():
        return None
    dev = mapping.device.index if isinstance(mapping, torch.Tensor) and mapping.is_cuda else torch.cuda.current_device()
    return dev if torch.cuda.get_device_capability(dev) == (9, 0) else None


def _agree_on_shards(adata_map, process_group, n_cells=None, refusal=None, labels=None):
    """The first collective of a transfer call on a cell-sharded mapping (`adata_map`: the AnnData that
    map_cells_to_space(process_group=) returned on this rank): one all_gather_object of every rank's uns["shard_rows"],
    of what `refusal(r0, r1)` finds wrong on this rank (a message or None) and of `labels`.  Every rank then checks the
    same facts -- every rank has its rows, each mapping holds as many rows as its block, the blocks tile [0, n_cells)
    (default: up to the last block's end) in rank order, no rank refused -- and raises the same ValueError, so no rank is
    left waiting in a reduction the others never enter.  -> (r0, r1, every rank's `labels` in rank order)."""
    import torch.distributed as dist
    rows, refused = adata_map.uns.get("shard_rows"), None
    if rows is not None:
        try:
            r0, r1 = (int(r) for r in rows)
        except (TypeError, ValueError):
            r0 = r1 = None
        if r0 is None:
            rows, refused = None, f"uns['shard_rows'] = {rows!r} is not a pair of rows"
        else:
            rows = (r0, r1)
            if adata_map.X.shape[0] != r1 - r0:
                refused = f"its mapping has {adata_map.X.shape[0]} rows for uns['shard_rows'] = {rows}"
            elif refusal is not None:
                refused = refusal(r0, r1)
    box = [None] * dist.get_world_size(process_group)
    dist.all_gather_object(box, (rows, refused, labels), group=process_group)
    missing = [k for k, (r, _, _) in enumerate(box) if r is None]
    if missing:
        raise ValueError(f"rank(s) {missing} passed a mapping without uns['shard_rows']: every rank must pass the AnnData "
                         "that map_cells_to_space(process_group=) returned on it"
                         + "".join(f"; rank {k}: {box[k][1]}" for k in missing if box[k][1]))
    blocks = [r for r, _, _ in box]
    end = 0
    for r0, r1 in blocks:
        if r0 != end or r1 < r0:
            raise ValueError(f"the ranks' mapping rows {blocks} do not tile the cells in rank order")
        end = r1
    if n_cells is not None and end != n_cells:
        raise ValueError(f"the ranks' mapping rows {blocks} cover {end} cells of the {n_cells} in adata_sc")
    refusals = [f"rank {k}: {e}" for k, (_, e, _) in enumerate(box) if e]
    if refusals:
        raise ValueError("; ".join(refusals))
    r0, r1 = blocks[dist.get_rank(process_group)]
    return r0, r1, [lab for _, _, lab in box]


def project_genes(adata_map, adata_sc, cluster_label=None, scale=True, *, process_group=None):
    """:338-374 -- adata_map.X^T adata_sc.X over every gene kept, as a (spots x genes) AnnData.  With the mapper kept on
    the device (map_cells_to_space(keep_on_device=True)) it projects through that handle; otherwise, on an sm_90 device,
    through `project` (a sparse adata_sc.X is streamed as CSR, never densified on the host); without one, on the host.

    process_group: `adata_map` is this rank's block of a cell-sharded mapping (map_cells_to_space(process_group=)),
    `adata_sc` the full AnnData, the same on every rank.  A collective: each rank filters the genes of the whole adata_sc
    (so the columns agree), projects adata_sc.X[r0:r1] through its rows and the (spots x genes) partials are summed over
    the group; every rank returns the same AnnData, the projection of every cell.  Refused with ValueError on every rank
    when a rank has no uns["shard_rows"], the blocks do not tile adata_sc's cells in rank order, a rank's obs index is not
    its block of adata_sc.obs.index, or cluster_label is given (clusters mode is never sharded)."""
    adata_sc.var.index = [g.lower() for g in adata_sc.var.index]                 # :353
    adata_sc.var_names_make_unique()                                              # :356
    keep = np.asarray((adata_sc.X != 0).sum(axis=0)).reshape(-1) >= 1             # :359
    if not keep.all():
        adata_sc = adata_sc[:, keep]
    X_sc = adata_sc.X
    if process_group is not None:
        def refusal(r0, r1):
            if cluster_label:
                return "cluster_label projects a clusters-mode mapping, and clusters mode is never sharded"
            if not adata_map.obs.index.equals(adata_sc.obs.index[r0:r1]):
                return f"its mapping's obs index is not rows [{r0}, {r1}) of adata_sc.obs.index"
            return None
        r0, r1, _ = _agree_on_shards(adata_map, process_group, adata_sc.X.shape[0], refusal)
        X_sc = X_sc[r0:r1]
    else:
        if cluster_label:
            adata_sc = mu.adata_to_cluster_expression(adata_sc, cluster_label, scale=scale)
            X_sc = adata_sc.X
        if not adata_map.obs.index.equals(adata_sc.obs.index):
            raise ValueError("The two AnnDatas need to have same `obs` index.")
    mapper = getattr(adata_map, "_tgb200_mapper", None)
    if mapper is not None and process_group is None and mapper.n_cells == X_sc.shape[0]:
        X_space = mapper.project(_dense(X_sc))   # softmax(M)^T X on the device (:368 is a host GEMM)
    else:
        if (dev := _sm90_device(adata_map.X)) is not None:
            X_space = project(adata_map.X, X_sc, device=f"cuda:{dev}")
        else:
            X_space = np.asarray(adata_map.X).T @ _dense(X_sc)
        X_space = mu._sum_over_group(X_space, dev, process_group)
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


def _canonical_csr(X, n_rows):
    """A scipy sparse X -> (int64 indptr, int32 indices, float32 data, n_genes) of canonical CSR: columns strictly
    increasing within each row, duplicates summed (in X's dtype, as toarray() sums them), explicit zeros kept.  The
    structure is checked before scipy touches it; X itself is never modified (a non-canonical input is fixed on a copy)."""
    import scipy.sparse as sp
    csr = X.tocsr()
    if csr.shape[0] != n_rows:
        raise ValueError(f"X has {csr.shape[0]} rows for a mapping of {n_rows} rows")
    n_genes = int(csr.shape[1])
    indptr, indices = np.asarray(csr.indptr), np.asarray(csr.indices)
    nnz = indices.shape[0]
    if indptr.shape != (n_rows + 1,) or csr.data.shape[0] != nnz:
        raise ValueError(f"malformed CSR: indptr of length {indptr.shape[0]} for {n_rows} rows, "
                         f"{nnz} indices and {csr.data.shape[0]} values")
    if indptr[0] != 0 or indptr[-1] != nnz or (np.diff(indptr) < 0).any():
        raise ValueError(f"malformed CSR: indptr must rise from 0 to nnz={nnz}")
    if nnz and (indices.min() < 0 or indices.max() >= n_genes):
        raise ValueError(f"CSR column index outside [0, {n_genes})")
    if n_genes > np.iinfo(np.int32).max - 64:
        raise ValueError(f"{n_genes} genes: more than int32 column indices address")
    row_start = np.zeros(nnz, dtype=bool)
    row_start[indptr[:-1][np.diff(indptr) > 0]] = True
    if not (row_start[1:] | (indices[1:] > indices[:-1])).all():
        if csr is X:
            csr = csr.copy()
        csr = sp.csr_matrix((csr.data, csr.indices, csr.indptr), shape=csr.shape)
        csr.sum_duplicates()                                 # sorts the columns and sums repeats, in X's dtype
    return (np.ascontiguousarray(csr.indptr, dtype=np.int64), np.ascontiguousarray(csr.indices, dtype=np.int32),
            np.ascontiguousarray(csr.data, dtype=np.float32), n_genes)


def project(mapping, X, *, device=None, _block_rows=0):
    """mapping^T X on the device (tgb200_project_map): the (V, n_genes) float32 projection of X through an (N, V) mapping,
    fp32-grade (split-bf16 operands on the tensor cores, chains of 512 cells added in order), identical bits whether X
    comes dense or sparse, from the host or the device.

    `mapping`: a numpy array, or a CUDA tensor (a float32 one with unit column stride is read in place, row stride
    included).  `X`: (N, n_genes) dense numpy array, CUDA tensor, or any scipy sparse matrix -- passed as canonical CSR
    (float32 data, int32 indices, int64 indptr), never densified.  The work runs on the device of a CUDA tensor argument,
    else on `device` (default: torch's current CUDA device), streamed over cell blocks, so neither the mapping nor X has
    to fit in device memory; the result must.  Malformed input raises ValueError before any device work."""
    import scipy.sparse as sp
    import torch
    cuda_map = isinstance(mapping, torch.Tensor) and mapping.is_cuda
    cuda_x = isinstance(X, torch.Tensor) and X.is_cuda
    M = mapping if cuda_map else np.asarray(mapping)
    if M.ndim != 2:
        raise ValueError(f"expected an (N, V) mapping, got shape {tuple(M.shape)}")
    N, V = (int(n) for n in M.shape)
    if sp.issparse(X):
        csr = _canonical_csr(X, N)
        n_genes = csr[3]
    else:
        if not cuda_x:
            X = np.asarray(X)
        if X.ndim != 2 or X.shape[0] != N:
            raise ValueError(f"X has shape {tuple(X.shape)} for a mapping of {N} rows")
        csr, n_genes = None, int(X.shape[1])
    if N == 0 or V == 0 or n_genes == 0:
        return np.zeros((V, n_genes), dtype=np.float32)
    if cuda_map:
        dev = M.device.index
    elif cuda_x:
        dev = X.device.index
    else:
        dev = _require_device("cuda" if device is None else device)
    if cuda_map:
        if M.dtype != torch.float32 or M.stride(1) != 1 or M.stride(0) < V:
            M = M.float().contiguous()
        m_ld = M.stride(0)
    else:
        M = np.ascontiguousarray(M, dtype=np.float32)
        m_ld = V
    if csr is not None:
        indptr, indices, data, _ = csr
        x_args = (None, 0, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data), indices.shape[0])
    else:
        if cuda_x:
            if X.dtype != torch.float32 or X.stride(1) != 1 or X.stride(0) < n_genes:
                X = X.float().contiguous()
            x_ld = X.stride(0)
        else:
            X = np.ascontiguousarray(X, dtype=np.float32)
            x_ld = n_genes
        x_args = (_lib.ptr(X), x_ld, None, None, None, 0)
    out = np.empty((V, n_genes), dtype=np.float32)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    lib = _lib.load()
    _lib.check(lib.tgb200_project_map(_lib.ptr(M), N, V, m_ld, *x_args, n_genes, _lib.ptr(out), int(_block_rows), dev,
                                      stream))
    return out


def _label_columns(series, columns=None):
    """-> (the one-hot columns of tangram/utils.py:105-123 for `series`: its unique values in order of first appearance, a
    NaN included, each row's position among them).  The positions are taken by position, whatever the index.  Given
    `columns` (a list holding every value of `series`), the positions are taken among those instead."""
    values = pd.Series(series).reset_index(drop=True)
    if columns is None:
        columns = pd.unique(values)
    codes = pd.Index(columns).get_indexer(values)
    return columns, values, codes


def _one_hot_codes(series, columns=None):
    """-> (one-hot columns, per-row column for the one-hot product): a NaN label has a column but matches no row there
    (NaN == NaN is false in one_hot_encoding), so its rows add nothing."""
    columns, values, codes = _label_columns(series, columns)
    return columns, np.where(values.isna().to_numpy(), -1, codes)


def _annotation_codes(adata_map, key, process_group):
    """_one_hot_codes of adata_map.obs[key].  With a group (`adata_map` one rank's block of a cell-sharded mapping) this is
    the call's agreement step (_agree_on_shards), and the columns are the whole mapping's: pd.unique of the ranks' labels
    in their order of first appearance, concatenated in rank order.  The blocks are contiguous, so that is the global
    order of first appearance, with one NaN column where the first NaN appears.  The concatenation is taken in the
    column's own dtype, so pd.unique compares the labels as it does on the whole column: in an object Series the float
    NaNs that come back from the gather are not taken as equal, and float labels would get a NaN column per rank."""
    if process_group is None:
        return _one_hot_codes(adata_map.obs[key])
    values = pd.Series(adata_map.obs[key]).reset_index(drop=True)
    _, _, firsts = _agree_on_shards(adata_map, process_group, labels=list(pd.unique(values)))
    columns = list(pd.unique(pd.Series([v for f in firsts for v in f], dtype=values.dtype)))
    return _one_hot_codes(values, columns)


def _mapping_of(adata_map):
    X = adata_map.X
    return X.toarray() if hasattr(X, "toarray") else X


def project_cell_annotations(adata_map, adata_sp, annotation="cell_type", threshold=0.5, *, process_group=None):
    """:126-153 -- transfer `annotation` from the cells onto space: adata_sp.obsm["tangram_ct_pred"] becomes a float64
    (spots x annotations) DataFrame indexed by adata_map.var.index, its columns the annotations in order of first
    appearance, entry [j, t] the mapping probability of spot j summed over the cells annotated t.

    `threshold` has no effect, as in the reference: it filters the cells by adata_map.obs["F_out"] > threshold into a
    variable that is overwritten before use (:144-147), so every cell counts.  The sums are taken on the device in fp64.

    process_group: `adata_map` is this rank's block of a cell-sharded mapping (map_cells_to_space(process_group=)) and
    `adata_sp` the same AnnData on every rank.  A collective: the columns are the labels of every rank's cells in global
    order of first appearance, each rank sums its own rows on the device and the sums are added over the group, so every
    rank writes the frame the unsharded call writes for the whole mapping (to rounding).  Refused with ValueError on every
    rank when a rank has no uns["shard_rows"] or the blocks do not tile the cells in rank order."""
    columns, codes = _annotation_codes(adata_map, annotation, process_group)
    sums, _ = annotate(_mapping_of(adata_map), codes, len(columns))
    sums = mu._sum_over_group(sums, None, process_group)
    adata_sp.obsm["tangram_ct_pred"] = pd.DataFrame(sums.T, index=adata_map.var.index, columns=pd.Index(list(columns)))


def cell_type_mapping(adata_map, cell_types_key="cell_types", *, process_group=None):
    """:820-842 -- adata_map.varm["ct_map"]: the (spots x cell types) sums of project_cell_annotations, min-max
    normalised per cell type (a constant column gives NaN, as in the reference).

    Where adata_map.obs has "F_out" (constrained mode), only the cells with F_out >= 0.5 count, each with its own label.
    The reference raises a shape error there whenever a cell is filtered out (:835 multiplies the filtered mapping by the
    unfiltered one-hot frame); where no cell is filtered out the result is the reference's.  The columns are the labels of
    all cells, so a type whose cells are all filtered out has a zero, and so NaN, column.

    process_group: as in project_cell_annotations; the sums are added over the group before the normalisation, so every
    rank's adata_map.varm["ct_map"] is that of the whole mapping."""
    columns, codes = _annotation_codes(adata_map, cell_types_key, process_group)
    if "F_out" in adata_map.obs.keys():
        codes = np.where(np.asarray(adata_map.obs["F_out"]) >= 0.5, codes, -1)
    sums, _ = annotate(_mapping_of(adata_map), codes, len(columns))
    sums = mu._sum_over_group(sums, None, process_group)
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


def count_cell_annotations(adata_map, adata_sc, adata_sp, annotation="cell_type", threshold=0.5, *,
                           process_group=None):
    """:205-285 -- adata_sp.obsm["tangram_ct_count"]: per spot its coordinates 'x', 'y', its segmented cell count
    'cell_n', its cell ids 'centroids', and per annotation (adata_sc.obs[annotation], in order of first appearance) the
    number of cells whose most probable spot it is.  Where adata_map.obs has "F_out", only the cells with
    F_out > threshold are counted.

    The most probable spot of each counted cell is the device row argmax of the mapping (first spot on ties, as
    np.argmax); the counts are one np.bincount.  Annotations are read by position in adata_sc.obs.

    process_group: `adata_map` is this rank's block of a cell-sharded mapping (map_cells_to_space(process_group=)),
    `adata_sc` and `adata_sp` the same AnnDatas on every rank.  A collective: the columns come from the whole
    adata_sc.obs[annotation], the cell in row i of rows [r0, r1) takes the label at position r0 + i (positions past
    adata_sc's cells are not counted, as without a group), each rank counts its own cells and the int64 counts are added
    over the group, so every rank writes the frame the unsharded call writes for the whole mapping, exactly.  Refused
    with ValueError on every rank when a rank has no uns["shard_rows"] or the blocks do not tile the cells in rank
    order."""
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
    r0 = 0                                              # the global position of this mapping's first cell
    if process_group is not None:
        r0, _, _ = _agree_on_shards(adata_map, process_group)
    columns, _, codes = _label_columns(adata_sc.obs[annotation])
    X = _mapping_of(adata_map)
    N = X.shape[0]
    n = min(N, max(len(codes) - r0, 0))                # cells beyond adata_sc's are not counted (the reference zips)
    labels = np.full(N, -1, dtype=np.int64)
    labels[:n] = codes[r0:r0 + n]
    if "F_out" in adata_map.obs.keys():
        labels[~(np.asarray(adata_map.obs["F_out"]) > threshold)] = -1
    keep = labels >= 0
    _, spot = annotate(X, np.minimum(labels, 0), 1, sums=False, argmax=True)
    counts = np.bincount(spot[keep].astype(np.int64) * len(columns) + labels[keep],
                         minlength=len(df) * len(columns)).reshape(len(df), len(columns))
    counts = mu._sum_over_group(counts, None, process_group)
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


# ---------------------------------------------------------------------------------------------------------------------
# Gene cross-validation (tangram/utils.py:377-758)

def compare_spatial_geneexp(adata_ge, adata_sp, adata_sc=None, genes=None):
    """:377-463 -- per gene the cosine between the projected expression (adata_ge, as project_genes returns it) and the
    measured one (adata_sp): a frame indexed by gene with 'score', 'is_training' (where adata_ge.var or adata_sp.var has
    it), 'sparsity_sp' and, with adata_sc, 'sparsity_sc' and 'sparsity_diff', sorted by score (highest first).
    `genes` (default adata_ge.uns["overlap_genes"]) picks the genes.  As in the reference, the sparsity columns are
    written into adata_sp.var (and adata_sc.var), and the root logger is disabled."""
    logging.getLogger().disabled = True
    if not set(["training_genes", "overlap_genes"]).issubset(set(adata_sp.uns.keys())):
        raise ValueError("Missing tangram parameters. Run `pp_adatas()`.")
    if not set(["training_genes", "overlap_genes"]).issubset(set(adata_ge.uns.keys())):
        raise ValueError("Missing tangram parameters. Use `project_genes()` to get adata_ge.")
    assert list(adata_sp.uns["overlap_genes"]) == list(adata_ge.uns["overlap_genes"])
    overlap_genes = adata_ge.uns["overlap_genes"] if genes is None else genes
    mu.annotate_gene_sparsity(adata_sp)
    X_1 = _mapping_of(adata_ge[:, overlap_genes])
    X_2 = _mapping_of(adata_sp[:, overlap_genes])
    cos_sims = [(v1 @ v2) / (np.linalg.norm(v1) * np.linalg.norm(v2)) for v1, v2 in zip(X_1.T, X_2.T)]
    df_g = pd.DataFrame(cos_sims, overlap_genes, columns=["score"])
    for adata in (adata_ge, adata_sp):
        if "is_training" in adata.var.keys():
            df_g["is_training"] = adata.var.is_training
    df_g["sparsity_sp"] = adata_sp[:, overlap_genes].var.sparsity
    if adata_sc is not None:
        if not set(["training_genes", "overlap_genes"]).issubset(set(adata_sc.uns.keys())):
            raise ValueError("Missing tangram parameters. Run `pp_adatas()`.")
        assert list(adata_sc.uns["overlap_genes"]) == list(adata_sp.uns["overlap_genes"])
        mu.annotate_gene_sparsity(adata_sc)
        df_g = df_g.merge(pd.DataFrame(adata_sc[:, overlap_genes].var["sparsity"]), left_index=True, right_index=True)
        df_g.rename({"sparsity": "sparsity_sc"}, inplace=True, axis="columns")
        df_g["sparsity_diff"] = df_g["sparsity_sp"] - df_g["sparsity_sc"]
    if genes is not None:
        df_g = df_g.loc[genes]
    return df_g.sort_values(by="score", ascending=False)


def _cv_splits(n, cv_mode):
    """(train positions, test positions) of sklearn's LeaveOneOut ('loo') or unshuffled KFold(n_splits=10) ('10fold')
    over n items: KFold's first n % 10 folds hold one item more than the others."""
    if cv_mode == "loo":
        if n < 2:
            raise ValueError(f"Cannot perform LeaveOneOut with n_samples={n}.")
        sizes = [1] * n
    elif cv_mode == "10fold":
        if n < 10:
            raise ValueError(f"Cannot have number of splits n_splits=10 greater than the number of samples: n_samples={n}.")
        sizes = [n // 10 + (1 if f < n % 10 else 0) for f in range(10)]
    else:
        raise ValueError(f'cv_mode must be "loo" or "10fold", got {cv_mode!r}')
    idx, start = np.arange(n), 0
    for size in sizes:
        test = idx[start:start + size]
        yield np.concatenate([idx[:start], idx[start + size:]]), test
        start += size


def cv_data_gen(adata_sc, adata_sp, cv_mode="loo"):
    """:466-500 -- yields (train_genes, test_genes) lists over the training genes of pp_adatas: leave-one-out
    (cv_mode="loo") or ten contiguous folds ("10fold"), as sklearn's LeaveOneOut / KFold(10) split them.  An unknown
    cv_mode raises ValueError (the reference fails there with UnboundLocalError)."""
    if "training_genes" not in adata_sc.uns.keys():
        raise ValueError("Missing tangram parameters. Run `pp_adatas()`.")
    if "training_genes" not in adata_sp.uns.keys():
        raise ValueError("Missing tangram parameters. Run `pp_adatas()`.")
    if not list(adata_sp.uns["training_genes"]) == list(adata_sc.uns["training_genes"]):
        raise ValueError("Unmatched training_genes field in two Anndatas. Run `pp_adatas()`.")
    genes_array = np.array(adata_sp.uns["training_genes"])
    for train_idx, test_idx in _cv_splits(len(genes_array), cv_mode):
        yield list(genes_array[train_idx]), list(genes_array[test_idx])


def cross_val(adata_sc, adata_sp, cluster_label=None, mode="clusters", scale=True, lambda_d=0, lambda_g1=1, lambda_g2=0,
              lambda_r=0, lambda_count=1, lambda_f_reg=1, target_count=None, num_epochs=1000, device="cuda:0",
              learning_rate=0.1, cv_mode="loo", return_gene_pred=False, density_prior=None, random_state=None,
              verbose=False, *, precision="bf16x3", process_group=None):
    """:503-668 -- gene cross-validation: for each fold of cv_data_gen, a mapping trained on the fold's training genes
    (as map_cells_to_space(cv_train_genes=...) trains it) scores the held-out genes with compare_spatial_geneexp.
    Returns cv_dict {"avg_test_score", "avg_train_score"} (nanmean over the folds; a fold's train score is the last
    main_loss of its history), and with cv_mode="loo" and return_gene_pred=True also adata_ge_cv (spots x test genes:
    each gene's projection from the fold that held it out; var "test_score") and test_gene_df (the test genes' rows of
    compare_spatial_geneexp).  verbose prints each fold's scores.

    All folds train on one device handle built once over all training genes: each fold restricts the loss to its
    training genes (a handle masked to S[:, train] computes what a handle built on those columns computes), redraws
    the initial mapping from numpy's global generator exactly as a fresh mapper would (reseeded when random_state is
    truthy), trains num_epochs with a fresh Adam, and projects only the test genes on the device.  `precision` as in
    map_cells_to_space.

    process_group (mode="cells" or "constrained"): the folds' mappings are cell-sharded as in map_cells_to_space -- every
    rank passes the same AnnDatas, trains its block of cells, projects the test genes from its own rows, and the
    projections are summed over the group.  The folds and the gene columns follow rank 0's order of the training genes,
    and every rank returns the same results."""
    logging.getLogger().disabled = True
    logging.getLogger("anndata").disabled = True
    mu._check_shardable(mode, process_group)
    folds = list(cv_data_gen(adata_sc, adata_sp, cv_mode))
    sharding = {}
    if process_group is not None:
        # uns["training_genes"] comes from a set in pp_adatas, so its order (and with it the folds) can differ between
        # processes: every rank takes rank 0's folds, as _prepare_mapping takes rank 0's gene order
        import torch.distributed as dist
        box = [folds]
        dist.broadcast_object_list(box, src=dist.get_global_rank(process_group, 0), group=process_group)
        folds = box[0]
        sharding = dict(process_group=process_group)
        if mode == "cells":
            # the folds draw one after another from numpy's generator: every rank must leave it where the unsharded draw
            # does (a sharded Mapper's draw stops after the rank's last row otherwise)
            sharding["draw_whole_stream"] = True
    adata_ref, genes, S, _, mapper_kw = mu._prepare_mapping(
        adata_sc, adata_sp, None, cluster_label, mode, scale, density_prior, lambda_d, lambda_g1, lambda_g2, lambda_r,
        0, 0, lambda_count, lambda_f_reg, target_count, 0, 0, 0, 0, 0, process_group)
    if mode != "clusters":
        adata_ref = adata_sc
    column = {g: k for k, g in enumerate(genes)}
    test_genes_list, test_pred_list, test_score_list, train_score_list, test_df_list = [], [], [], [], []
    mapper = mu._make_mapper(mode, mapper_kw, device=device, random_state=random_state, precision=precision, **sharding)
    r0, r1 = getattr(mapper, "_rows", (0, S.shape[0]))
    try:
        for fold, (train_genes, test_genes) in enumerate(folds):
            if fold > 0:                      # the constructor made the first fold's draw
                mapper._draw_initial_mapping()
            active = np.zeros(len(genes), dtype=bool)
            active[[column[g] for g in train_genes]] = True
            mapper._set_loss_genes(active)
            mapper._fit(num_epochs, float(learning_rate), None, False, fetch=False)
            train_score = float(mapper.history_matrix[-1, 1])                    # main_loss (:622)
            pred = mu._sum_over_group(mapper.project(S[r0:r1, [column[g] for g in test_genes]]), _device_index(device),
                                      process_group)                              # (spots, test genes)
            var = pd.DataFrame({"is_training": np.zeros(len(test_genes), dtype=bool)}, index=test_genes)
            adata_ge = make_adata(X=pred, obs=adata_sp.obs.copy(), var=var, uns=adata_ref.uns)
            df_g = compare_spatial_geneexp(adata_ge, adata_sp, adata_ref, test_genes)
            test_score = df_g.loc[test_genes]["score"].mean()
            if cv_mode == "loo" and return_gene_pred:
                test_pred_list.append(pred.T)
            test_genes_list.append(test_genes)
            test_score_list.append(test_score)
            train_score_list.append(train_score)
            test_df_list.append(df_g)
            if verbose:
                print("cv set: {}----train score: {:.3f}----test score: {:.3f}".format(fold + 1, train_score, test_score))
    finally:
        mapper.release()

    avg_test_score = np.nanmean(test_score_list)
    avg_train_score = np.nanmean(train_score_list)
    cv_dict = {"avg_test_score": avg_test_score, "avg_train_score": avg_train_score}
    print("cv avg test score {:.3f}".format(avg_test_score))
    print("cv avg train score {:.3f}".format(avg_train_score))
    if cv_mode == "loo" and return_gene_pred:
        test_gene_df = pd.concat(test_df_list, axis=0)
        adata_ge_cv = make_adata(
            X=np.squeeze(test_pred_list).T, obs=adata_sp.obs.copy(),
            var=pd.DataFrame(test_score_list, columns=["test_score"], index=np.squeeze(test_genes_list)))
        return cv_dict, adata_ge_cv, test_gene_df
    return cv_dict


def _auc(x, y):
    """sklearn.metrics.auc: the trapezoidal area under (x, y), x monotonic in either direction."""
    x, y = np.asarray(x).reshape(-1), np.asarray(y).reshape(-1)
    if x.shape[0] != y.shape[0]:
        raise ValueError(f"Found input variables with inconsistent numbers of samples: [{x.shape[0]}, {y.shape[0]}]")
    if x.shape[0] < 2:
        raise ValueError(f"At least 2 points are needed to compute area under curve, but x.shape = {x.shape[0]}")
    direction = 1
    dx = np.diff(x)
    if np.any(dx < 0):
        if np.all(dx <= 0):
            direction = -1
        else:
            raise ValueError("x is neither increasing nor decreasing : {}.".format(x))
    trapezoid = getattr(np, "trapezoid", None) or np.trapz
    return direction * trapezoid(y, x)


def eval_metric(df_all_genes, test_genes=None):
    """:671-758 -- metrics of a compare_spatial_geneexp frame over `test_genes` (default: the genes whose is_training is
    False): ({"avg_test_score", "avg_train_score", "sp_sparsity_score", "auc_score"}, ((fitted xs, ys), (raw test scores,
    raw sparsity_sp))).  auc_score is the area under the quadratic fit of sparsity against score, restricted to the unit
    square, exactly as the reference computes it."""
    if test_genes is not None:
        if not set(test_genes).issubset(set(df_all_genes.index.values)):
            raise ValueError("the input of test_genes should be subset of genes of input dataframe")
        test_genes = np.unique(test_genes)
    else:
        test_genes = list(set(df_all_genes[df_all_genes["is_training"] == False].index.values))  # noqa: E712
    test_gene_scores = df_all_genes.loc[test_genes]["score"]
    test_gene_sparsity_sp = df_all_genes.loc[test_genes]["sparsity_sp"]
    test_score_avg = test_gene_scores.mean()
    train_score_avg = df_all_genes[df_all_genes["is_training"] == True]["score"].mean()  # noqa: E712
    test_score_sps_sp_g2 = np.sum((test_gene_scores * (1 - test_gene_sparsity_sp)) / (1 - test_gene_sparsity_sp).sum())

    xs = list(test_gene_scores)
    ys = list(test_gene_sparsity_sp)
    pol = np.poly1d(np.polyfit(xs, ys, 2))
    pol_xs = np.linspace(0, 1, 10)
    pol_ys = [pol(x) for x in pol_xs]
    if pol_ys[0] > 1:
        pol_ys[0] = 1
    root = None                                   # the first real root in [0, 1] adds the point (root, 0)
    for r in pol.r:
        if np.isreal(r) and r <= 1 and r >= 0:
            root = r
            break
    if root is not None:
        pol_xs = np.append(pol_xs, root)
        pol_ys = np.append(pol_ys, 0)
    # the reference's np.append(pol_xs, 1) / np.append(pol_ys, pol(1)) discard their results: no point (1, pol(1))
    del_idx = [i for i in range(len(pol_xs)) if pol_xs[i] < 0 or pol_ys[i] < 0 or pol_xs[i] > 1 or pol_ys[i] > 1]
    # points are dropped by the position of their value's FIRST occurrence, as the reference's list.index does
    pol_xs = [x for x in pol_xs if list(pol_xs).index(x) not in del_idx]
    pol_ys = [y for y in pol_ys if list(pol_ys).index(y) not in del_idx]
    auc_test_score = np.real(_auc(pol_xs, pol_ys))
    metric_dict = {"avg_test_score": test_score_avg, "avg_train_score": train_score_avg,
                   "sp_sparsity_score": test_score_sps_sp_g2, "auc_score": auc_test_score}
    return metric_dict, ((pol_xs, pol_ys), (xs, ys))
