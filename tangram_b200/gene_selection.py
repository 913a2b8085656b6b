"""Training genes chosen on the GPU, the first step of Tangram's tutorials and its gene_selection/ctg and /hvg:

    tg.rank_genes_groups(ad_sc, groupby="cell_subclass", use_raw=False)     # scanpy's sc.tl.rank_genes_groups (t-test)
    markers = list(np.unique(pd.DataFrame(ad_sc.uns["rank_genes_groups"]["names"]).iloc[0:100, :].melt().value.values))
    tg.pp_adatas(ad_sc, ad_sp, genes=markers)
    markers = tg.ctg(ad_sc, "cell_subclass")                                 # the same with the top 150 of each group
    tg.highly_variable_genes(ad_sc, n_top_genes=4000)                       # scanpy's sc.pp.highly_variable_genes
    genes = tg.hvg(ad_sc)                                                    # its 4000 highly variable genes

Every group's (or batch's) sums, sums of squares and nonzero counts come from one streaming pass over the expression
matrix on the device (`group_stats`, tgb200_group_stats, or tgb200_group_stats_expm1 for the sums of expm1(x)) -- dense,
sparse (as CSR, never densified) or a CUDA tensor read in place -- instead of a mean and variance over X[mask] and
X[~mask] per group on the host.  The Welch t-test, the p-value corrections, the log fold changes and the ranking, and the
dispersions, their binning and normalisation and the selection, are per-gene host arithmetic on those statistics.
scanpy is not needed.
"""
import ctypes
import warnings

import numpy as np
import pandas as pd

from . import _lib
from .engine import _require_device
from .utils import _canonical_csr

_RANGE = 2048                       # cells per summation chain of tgb200_group_stats
_METHODS = ("t-test", "t-test_overestim_var")
_CORR_METHODS = ("benjamini-hochberg", "bonferroni")


def _group_stats_device_bytes(n_genes, n_labels, staging):
    """Least device memory tgb200_group_stats needs: its outputs, the partials of one range's runs, one block of staging."""
    return 24 * n_labels * n_genes + 20 * min(n_labels, _RANGE) * n_genes + staging + 8 * _RANGE + 16 * n_labels


def group_stats(X, labels, n_labels, *, device=None, expm1_scale=None, _block_rows=0):
    """One pass of tgb200_group_stats over the (N, n_genes) expression `X`: -> (sum, sumsq, nnz), each (n_labels,
    n_genes): the float64 sums of x and of x * x, and the int64 count of x != 0 (NaN counting), over the rows labelled t.
    With `expm1_scale` a number, the pass is tgb200_group_stats_expm1: the sums are of y = expm1(expm1_scale * x) and of
    y * y, computed in float64 for every element (scanpy's float32 expm1 overflows to inf above x ~ 88.7; this stays
    finite there), and the count is still of x != 0.

    `labels`: N integers in [-1, n_labels); rows labelled -1 add to nothing.  `X` is read as float32: a dense numpy array,
    any scipy sparse matrix (passed as canonical CSR, never densified) or a CUDA tensor (a float32 one with unit column
    stride is read in place, row stride included).  The sums are fp64 chains over aligned ranges of 2048 cells added in
    range order, so dense and sparse X, host and device data and any block size give identical bits.  The work runs on
    the device of a CUDA tensor X, else on `device` (default: torch's current CUDA device), streamed in cell blocks.
    Malformed input raises ValueError and too little free device memory TangramB200Error, before any device work."""
    import scipy.sparse as sp
    import torch
    n_labels = int(n_labels)
    lab = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
    N = lab.shape[0]
    cuda_x = isinstance(X, torch.Tensor) and X.is_cuda
    if sp.issparse(X):
        if X.shape[0] != N:
            raise ValueError(f"X has {X.shape[0]} rows for {N} labels")
        csr = _canonical_csr(X, N)
        G = csr[3]
    else:
        if not cuda_x:
            X = np.asarray(X)
        if X.ndim != 2 or X.shape[0] != N:
            raise ValueError(f"X has shape {tuple(X.shape)} for {N} labels")
        csr, G = None, int(X.shape[1])
    if n_labels < 1:
        raise ValueError(f"n_labels={n_labels}, must be at least 1")
    if N and (lab.min() < -1 or lab.max() >= n_labels):
        raise ValueError(f"labels must lie in [-1, {n_labels})")
    if N == 0 or G == 0:
        return np.zeros((n_labels, G)), np.zeros((n_labels, G)), np.zeros((n_labels, G), np.int64)
    dev = X.device.index if cuda_x else _require_device("cuda" if device is None else device)
    if csr is not None:
        indptr, indices, data, _ = csr
        range_nnz = np.diff(np.append(indptr[::_RANGE], indptr[-1]))
        staging = 2 * (8 * int(range_nnz.max()) + 8 * (_RANGE + 1))
        x_args = (None, 0, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(data), indices.shape[0])
    else:
        if cuda_x:
            if X.dtype != torch.float32 or X.stride(1) != 1 or X.stride(0) < G:
                X = X.float().contiguous()
            x_ld, staging = X.stride(0), 0
        else:
            X = np.ascontiguousarray(X, dtype=np.float32)
            x_ld, staging = G, 2 * 4 * _RANGE * G
        x_args = (_lib.ptr(X), x_ld, None, None, None, 0)
    need = _group_stats_device_bytes(G, n_labels, staging)
    free, _ = torch.cuda.mem_get_info(dev)
    if need > free:
        raise _lib.TangramB200Error(
            f"group statistics need at least {need / 2**30:.2f} GiB on cuda:{dev} for {G} genes and {n_labels} labels "
            f"({24 * n_labels * G / 2**30:.2f} GiB of it for the result); {free / 2**30:.2f} GiB are free")
    out_s = np.empty((n_labels, G), dtype=np.float64)
    out_q = np.empty((n_labels, G), dtype=np.float64)
    out_n = np.empty((n_labels, G), dtype=np.int64)
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    lib = _lib.load()
    args = (*x_args, N, G, _lib.ptr(lab), n_labels, _lib.ptr(out_s), _lib.ptr(out_q), _lib.ptr(out_n), int(_block_rows),
            dev, stream)
    if expm1_scale is None:
        _lib.check(lib.tgb200_group_stats(*args))
    else:
        _lib.check(lib.tgb200_group_stats_expm1(*args, float(expm1_scale)))
    return out_s, out_q, out_n


def _expression(adata, use_raw, layer):
    """-> (the matrix rank_genes_groups reads, its gene names, whether it is adata.raw)."""
    raw = getattr(adata, "raw", None)
    if layer is not None:
        if use_raw:
            raise ValueError("Cannot specify `layer` and have `use_raw=True`.")
        layers = getattr(adata, "layers", None) or {}
        if layer not in layers:
            raise ValueError(f"layer {layer!r} is not in adata.layers")
        return layers[layer], pd.Index(adata.var_names), False
    if use_raw is None:
        use_raw = raw is not None
    if use_raw:
        if raw is None:
            raise ValueError("use_raw=True, but adata has no raw")
        return raw.X, pd.Index(raw.var_names), True
    return adata.X, pd.Index(adata.var_names), False


def _group_codes(obs, groupby):
    """-> (group names as str: the categories in order, or the sorted unique non-missing values; each cell's group, -1
    where the label is missing)."""
    if groupby not in obs.columns:
        raise ValueError(f"groupby={groupby!r} is not a column of adata.obs")
    col = obs[groupby]
    if isinstance(col.dtype, pd.CategoricalDtype):
        names = [str(c) for c in col.cat.categories]
        codes = col.cat.codes.to_numpy().astype(np.int32)
    else:
        values = col.to_numpy()
        present = ~pd.isna(col).to_numpy()
        uniq = np.unique(values[present])
        names = [str(u) for u in uniq]
        codes = np.full(len(values), -1, dtype=np.int32)
        codes[present] = np.searchsorted(uniq, values[present])
    if len(set(names)) != len(names):
        raise ValueError(f"the groups of {groupby!r} are not distinct as strings: {names}")
    return names, codes


def rank_genes_groups(adata, groupby, *, groups="all", reference="rest", n_genes=None, rankby_abs=False,
                      method="t-test", corr_method="benjamini-hochberg", use_raw=None, layer=None, pts=False,
                      key_added=None, device=None, _block_rows=0):
    """scanpy's sc.tl.rank_genes_groups with the t-test methods: ranks the genes of each group against the rest (or a
    reference group) and writes adata.uns[key_added or "rank_genes_groups"].

    Matrix: adata.layers[layer], else adata.raw.X when use_raw is true (or None and adata.raw exists), else adata.X; read
    as float32 -- dense, any scipy sparse matrix (never densified) or a float32 CUDA tensor (read in place).
    Groups: the categories of obs[groupby] in order, or its sorted unique non-missing values, as str.  A cell with a missing
    label is in no group but in every group's rest.  `groups` ("all" or a list) selects the output groups; the rest of a
    group is every other cell, unselected groups included.  `reference` ("rest" or a group) replaces the rest by that
    group, which is then left out of the output.
    Statistics: one tgb200_group_stats pass gives every group's sum, sum of squares, size and nonzero count; the rest is
    the total minus the group in fp64; mean = sum / n, var = (sumsq / n - mean^2) n / (n - 1).  Scores and p-values are
    Welch's t-test (scipy.stats.ttest_ind_from_stats; "t-test_overestim_var" takes the group's size for the rest's), NaN
    scores become 0 and NaN p-values 1; pvals_adj is Benjamini-Hochberg or Bonferroni over all genes; logfoldchanges are
    log2((expm1(mean_g) + 1e-9) / (expm1(mean_rest) + 1e-9)), in uns["log1p"]["base"] when set.
    Ranking: by descending score (|score| with rankby_abs), the lower gene index first on exactly equal scores -- a stable
    order where scanpy's argpartition may order such ties differently; n_genes=None keeps every gene.
    Output: params, and names / scores (float32) / logfoldchanges (float32) / pvals / pvals_adj as np.rec arrays with one
    field per output group and n_genes rows (pd.DataFrame(uns[key]["names"]) has one column per group); with pts=True,
    pts (and for reference="rest", pts_rest): genes x groups DataFrames of the fraction of cells with x != 0.
    Raises ValueError for an unknown groupby, group or reference, a selected group (or the reference) of fewer than 2
    cells, or an inconsistent use_raw / layer; NotImplementedError for "wilcoxon" and "logreg"."""
    from scipy import stats
    if method in ("wilcoxon", "logreg"):
        raise NotImplementedError(f"method={method!r} is not implemented on the GPU; use 't-test' or "
                                  "'t-test_overestim_var'")
    if method not in _METHODS:
        raise ValueError(f"method={method!r}: expected one of {_METHODS}")
    if corr_method not in _CORR_METHODS:
        raise ValueError(f"corr_method={corr_method!r}: expected one of {_CORR_METHODS}")
    X, var_names, used_raw = _expression(adata, use_raw, layer)
    names, codes = _group_codes(adata.obs, groupby)
    if X.shape[0] != len(codes):
        raise ValueError(f"the expression matrix has {X.shape[0]} rows for {len(codes)} cells")
    if isinstance(groups, str) and groups == "all":
        selected = list(names)
    else:
        selected = [str(g) for g in (groups if not isinstance(groups, str) else [groups])]
    if len(set(selected)) != len(selected):
        raise ValueError(f"groups={selected} names a group twice")
    unknown = [g for g in selected if g not in names]
    if unknown:
        raise ValueError(f"groups {unknown} are not groups of {groupby!r}: {names}")
    if reference != "rest":
        reference = str(reference)
        if reference not in names:
            raise ValueError(f"reference={reference!r} is not a group of {groupby!r}: {names}")
    order = selected + ([reference] if reference != "rest" and reference not in selected else [])
    out_groups = [g for g in selected if g != reference]
    T, G, N = len(names), X.shape[1], len(codes)
    idx = {g: k for k, g in enumerate(names)}
    counts = np.bincount(np.where(codes < 0, T, codes), minlength=T + 1)
    small = [g for g in order if counts[idx[g]] < 2]
    if small:
        raise ValueError(f"groups {small} of {groupby!r} have fewer than 2 cells")
    if n_genes is None or int(n_genes) > G:
        n_genes = G
    n_genes = int(n_genes)
    if n_genes < 0:
        raise ValueError(f"n_genes={n_genes} is negative")

    # one pass: every group's statistics, the cells without a label in an extra bucket so the totals cover every cell
    S, Q, NZ = group_stats(X, np.where(codes < 0, T, codes), T + 1, device=device, _block_rows=_block_rows)
    tot_s, tot_q, tot_nz = S.sum(axis=0), Q.sum(axis=0), NZ.sum(axis=0)
    base = (adata.uns.get("log1p") or {}).get("base")

    def expm1(m):
        return np.expm1(m * np.log(base)) if base is not None else np.expm1(m)

    def mean_var(s, q, n):
        mean = s / n
        return mean, (q / n - mean * mean) * (n / (n - 1))

    if reference != "rest":
        r = idx[reference]
        mean_r, var_r = mean_var(S[r], Q[r], float(counts[r]))
    res = {"names": [], "scores": [], "logfoldchanges": [], "pvals": [], "pvals_adj": []}
    pts_g, pts_r = {}, {}
    with np.errstate(divide="ignore", invalid="ignore"):
        for g in order:
            t = idx[g]
            n_g = float(counts[t])
            if pts:
                pts_g[g] = NZ[t] / n_g
                if reference == "rest":
                    pts_r[g] = (tot_nz - NZ[t]) / float(N - counts[t])
            if g == reference:
                continue
            mean_g, var_g = mean_var(S[t], Q[t], n_g)
            if reference == "rest":
                n_r = float(N - counts[t])
                mean_r, var_r = mean_var(tot_s - S[t], tot_q - Q[t], n_r)
            else:
                n_r = float(counts[idx[reference]])
            n_r_test = n_g if method == "t-test_overestim_var" else n_r
            scores, pvals = stats.ttest_ind_from_stats(mean_g, np.sqrt(var_g), n_g, mean_r, np.sqrt(var_r), n_r_test,
                                                       equal_var=False)
            scores = np.where(np.isnan(scores), 0.0, scores)
            pvals = np.where(np.isnan(pvals), 1.0, pvals)
            if corr_method == "benjamini-hochberg":
                adj = stats.false_discovery_control(pvals, method="bh")
            else:
                adj = np.minimum(pvals * G, 1.0)
            lfc = np.log2((expm1(mean_g) + 1e-9) / (expm1(mean_r) + 1e-9))
            top = np.argsort(-(np.abs(scores) if rankby_abs else scores), kind="stable")[:n_genes]
            res["names"].append(np.asarray(var_names[top], dtype=object))
            res["scores"].append(scores[top].astype(np.float32))
            res["logfoldchanges"].append(lfc[top].astype(np.float32))
            res["pvals"].append(pvals[top].astype(np.float64))
            res["pvals_adj"].append(adj[top].astype(np.float64))

    key = key_added or "rank_genes_groups"
    uns = {"params": {"groupby": groupby, "reference": reference, "method": method, "use_raw": used_raw,
                      "layer": layer, "corr_method": corr_method}}
    dtypes = {"names": "O", "scores": "float32", "logfoldchanges": "float32", "pvals": "float64",
              "pvals_adj": "float64"}
    for field, cols in res.items():
        uns[field] = np.rec.fromarrays(cols if cols else [], dtype=[(g, dtypes[field]) for g in out_groups])
    if pts:
        uns["pts"] = pd.DataFrame(pts_g, index=var_names, columns=order)
        if reference == "rest":
            uns["pts_rest"] = pd.DataFrame(pts_r, index=var_names, columns=order)
    adata.uns[key] = uns


def ctg(adata_sc, cluster_label, n_top=150, *, device=None):
    """The reference's gene_selection/celltype_specific_genes.py::ctg: rank_genes_groups(groupby=cluster_label,
    use_raw=False), then the sorted unique names among the top `n_top` of every group."""
    rank_genes_groups(adata_sc, groupby=cluster_label, use_raw=False, device=device)
    markers_df = pd.DataFrame(adata_sc.uns["rank_genes_groups"]["names"]).iloc[0:n_top, :]
    return list(np.unique(markers_df.melt().value.values))


_HVG_FLAVORS = ("seurat", "cell_ranger")
_MAD_C = 0.6744897501960817         # the standard normal's 0.75 quantile: statsmodels' mad is median(|d - median|) / this


def _hvg_one_batch(s, q, n, flavor, n_bins, n_top_genes, cutoffs):
    """scanpy's single-batch seurat / cell_ranger steps on one batch's per-gene float64 sums of y and y * y over its n
    cells -> (means, dispersions, dispersions_norm, highly_variable)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        mean = s / n
        var = q / n - mean * mean
        if n != 1:                                  # as scanpy: one cell keeps the uncorrected variance
            var *= n / (n - 1)
        mean[mean == 0] = 1e-12
        disp = var / mean
        if flavor == "seurat":
            disp[disp == 0] = np.nan
            disp = np.log(disp)
            mean = np.log1p(mean)
    if flavor == "seurat":
        bins = n_bins
    else:
        bins = np.r_[-np.inf, np.percentile(mean, np.arange(10, 105, 5)), np.inf]
    codes = np.asarray(pd.cut(mean, bins=bins).codes)                        # -1: no bin (a NaN mean)
    avg, dev = np.full(len(mean), np.nan), np.full(len(mean), np.nan)
    for b in np.unique(codes[codes >= 0]):
        in_b = codes == b
        d = disp[in_b]
        if flavor == "seurat":                       # pandas' NaN-skipping mean and std(ddof=1)
            d = d[~np.isnan(d)]
            a = d.mean() if d.size else np.nan
            sd = d.std(ddof=1) if d.size > 1 else np.nan
            if np.isnan(sd):                         # one gene (or none) with a dispersion: normalised to 1
                a, sd = 0.0, a
        else:                                        # pandas' NaN-skipping median; statsmodels' mad propagates NaN
            a = np.median(d[~np.isnan(d)]) if (~np.isnan(d)).any() else np.nan
            sd = np.median(np.abs(d - np.median(d)) / _MAD_C)
        avg[in_b], dev[in_b] = a, sd
    with np.errstate(divide="ignore", invalid="ignore"):
        norm = (disp - avg) / dev
    if n_top_genes is None:
        min_mean, max_mean, min_disp, max_disp = cutoffs
        d = np.nan_to_num(norm)
        hv = (mean > min_mean) & (mean < max_mean) & (d > min_disp) & (d < max_disp)
    else:
        valid = norm[~np.isnan(norm)]
        k = min(n_top_genes, len(norm))
        if k > valid.size:
            warnings.warn("`n_top_genes` > number of normalized dispersions, returning all genes with normalized "
                          "dispersions.", UserWarning, stacklevel=3)
            k = valid.size
        if k == 0:
            hv = np.zeros(len(norm), dtype=bool)
        else:
            cut = np.sort(valid)[::-1][k - 1]
            hv = np.nan_to_num(norm, nan=-np.inf) >= cut
    return mean, disp, norm, hv


def highly_variable_genes(adata, *, layer=None, n_top_genes=None, min_disp=0.5, max_disp=np.inf, min_mean=0.0125,
                          max_mean=3, n_bins=20, flavor="seurat", subset=False, inplace=True, batch_key=None,
                          device=None):
    """scanpy's sc.pp.highly_variable_genes (1.10) with flavor "seurat" or "cell_ranger", on log1p-transformed data.

    Matrix: adata.layers[layer], else adata.X; read as float32 -- dense, any scipy sparse matrix (never densified) or a
    CUDA tensor (read in place).  Batches: with `batch_key`, the categories of obs[batch_key] in order, or its sorted
    unique non-missing values; a cell with a missing batch is in none.  Without it every cell is in one batch.
    Statistics: one device pass (group_stats) gives each batch's per-gene sum and sum of squares -- of expm1(x) for
    "seurat" (expm1(x ln base) with uns["log1p"]["base"]), of x for "cell_ranger" -- and its nonzero counts; mean = S / n
    and var = (Q / n - mean^2) n / (n - 1) (uncorrected for n = 1) in float64.  scanpy's expm1 is float32 and overflows
    to inf above x ~ 88.7; here it is float64 and stays finite.
    Per batch: a zero mean becomes 1e-12 and dispersion = var / mean; "seurat" then takes log(dispersion) (a zero
    dispersion is NaN) and log1p(mean).  Genes are binned by mean -- "seurat": pd.cut into n_bins equal-width bins;
    "cell_ranger": at the 10th, 15th, ..., 100th percentiles -- and dispersions_norm = (dispersion - avg) / dev with avg
    and dev the bin's mean and std ("seurat"; a bin with one gene gets avg 0 and dev its mean) or median and median
    absolute deviation / 0.6745 ("cell_ranger").  Selected: with `n_top_genes`, the genes whose dispersions_norm is at
    least the n-th largest (NaN never; a UserWarning when fewer are not NaN); otherwise NaN counts as 0 and a gene is
    selected when min_mean < mean < max_mean and min_disp < dispersions_norm < max_disp.
    Batched: a gene with no nonzero in a batch is left out of that batch's steps and counts there as means =
    dispersions = dispersions_norm = 0, not selected; each column is the NaN-skipping mean over batches,
    highly_variable_nbatches counts the batches that selected the gene and highly_variable_intersection is whether all
    did.  With `n_top_genes` the first n_top_genes genes by (nbatches, dispersions_norm) descending, NaN last, are
    selected, ties in gene order -- scanpy's unstable sort may order exact ties differently; otherwise the cutoffs apply
    to the averaged values (dispersions_norm with NaN as 0, which is what is stored).
    Output: with inplace, uns["hvg"] = {"flavor": flavor} and var columns highly_variable (bool), means, dispersions
    (float64), dispersions_norm (float32), and with batch_key highly_variable_nbatches (int64) and
    highly_variable_intersection (bool); subset keeps only the selected genes (in place).  With inplace=False the same
    columns are returned as a DataFrame indexed by var_names (only the selected rows with subset) and adata is untouched.
    Raises ValueError for an unknown flavor, batch_key or layer, n_bins < 1 or n_top_genes < 1; NotImplementedError for
    "seurat_v3" and "seurat_v3_paper" (they need skmisc's loess)."""
    if flavor in ("seurat_v3", "seurat_v3_paper"):
        raise NotImplementedError(f"flavor={flavor!r} needs skmisc's loess and is not implemented; use 'seurat' or "
                                  "'cell_ranger'")
    if flavor not in _HVG_FLAVORS:
        raise ValueError(f"flavor={flavor!r}: expected one of {_HVG_FLAVORS}")
    if int(n_bins) < 1:
        raise ValueError(f"n_bins={n_bins}, must be at least 1")
    n_bins = int(n_bins)
    if n_top_genes is not None:
        if int(n_top_genes) < 1:
            raise ValueError(f"n_top_genes={n_top_genes}, must be at least 1")
        n_top_genes = int(n_top_genes)
    X, var_names, _ = _expression(adata, False, layer)
    N, G = X.shape[0], X.shape[1]
    if batch_key is None:
        n_batches, codes = 1, np.zeros(N, dtype=np.int32)
    else:
        if batch_key not in adata.obs.columns:
            raise ValueError(f"batch_key={batch_key!r} is not a column of adata.obs")
        names, codes = _group_codes(adata.obs, batch_key)
        n_batches = len(names)
        if n_batches == 0:
            raise ValueError(f"batch_key={batch_key!r} has no non-missing value")
    if N != len(codes):
        raise ValueError(f"the expression matrix has {N} rows for {len(codes)} cells")
    base = (adata.uns.get("log1p") or {}).get("base")
    scale = (float(np.log(base)) if base is not None else 1.0) if flavor == "seurat" else None
    S, Q, NZ = group_stats(X, codes, n_batches, device=device, expm1_scale=scale)
    sizes = np.bincount(codes[codes >= 0], minlength=n_batches)
    cutoffs = (min_mean, max_mean, min_disp, max_disp)

    if batch_key is None:
        means, disp, norm, hv = _hvg_one_batch(S[0], Q[0], float(sizes[0]), flavor, n_bins, n_top_genes, cutoffs)
    else:
        per = np.zeros((4, n_batches, G))
        for b in range(n_batches):
            keep = NZ[b] > 0
            if keep.any():
                out = _hvg_one_batch(S[b, keep], Q[b, keep], float(sizes[b]), flavor, n_bins, n_top_genes, cutoffs)
                for k in range(4):
                    per[k, b, keep] = out[k]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", category=RuntimeWarning)          # a gene NaN in every batch stays NaN
            means, disp, norm = (np.nanmean(per[k], axis=0) for k in range(3))
        nbatches = per[3].sum(axis=0).astype(np.int64)
        if n_top_genes is not None:
            nan = np.isnan(norm)
            order = np.lexsort((np.arange(G), -np.where(nan, 0.0, norm), nan, -nbatches))
            hv = np.zeros(G, dtype=bool)
            hv[order[:n_top_genes]] = True
        else:
            norm = np.where(np.isnan(norm), 0.0, norm)
            hv = (means > min_mean) & (means < max_mean) & (norm > min_disp) & (norm < max_disp)

    df = pd.DataFrame({"highly_variable": np.asarray(hv, dtype=bool), "means": means, "dispersions": disp,
                       "dispersions_norm": norm.astype(np.float32)}, index=var_names)
    if batch_key is not None:
        df["highly_variable_nbatches"] = nbatches
        df["highly_variable_intersection"] = nbatches == n_batches
    if not inplace:
        return df[df["highly_variable"].to_numpy()] if subset else df
    adata.uns["hvg"] = {"flavor": flavor}
    for col in df.columns:
        adata.var[col] = df[col].to_numpy()
    if subset:
        adata._inplace_subset_var(df["highly_variable"].to_numpy())
    return None


def hvg(adata_sc, n_top_genes=4000, *, device=None):
    """The reference's gene_selection/highly_variable_genes.py::hvg: highly_variable_genes(adata_sc,
    n_top_genes=n_top_genes), then the names of the selected genes in gene order."""
    highly_variable_genes(adata_sc, n_top_genes=n_top_genes, device=device)
    return list(adata_sc.var_names[adata_sc.var["highly_variable"].to_numpy()])
