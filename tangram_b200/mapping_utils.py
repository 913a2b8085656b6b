"""
`map_cells_to_space` with the reference's signature and output contract
(Tangram's tangram/mapping_utils.py:141-428), hosted over the H100 Mapper.
AnnData in, AnnData out (duck-typed: `anndata` is optional).  `pp_adatas` and
`adata_to_cluster_expression` are the small host-side preparations this entry needs
(:20-139).  The spatial terms read the neighbour graph from `adata_sp.obsp`
(scipy CSR); `tg.spatial_neighbors(adata_sp)` builds it on the GPU, as squidpy would.
"""
import logging

import numpy as np
import pandas as pd

from . import mapping_optimizer as mo
from . import spatial_weights as sw
from .adata import make_adata
from .engine import _device_index


def _dense_f32(X):
    if hasattr(X, "toarray"):
        return np.asarray(X.toarray(), dtype=np.float32)
    if isinstance(X, np.ndarray):
        return np.asarray(X, dtype=np.float32)     # the reference calls .toarray() here (:262, latent bug)
    logging.error("AnnData X has unrecognized type: {}".format(type(X)))
    raise NotImplementedError


def annotate_gene_sparsity(adata):
    """tangram/utils.py:46-60: var['sparsity'] = 1 - fraction of non-zero observations."""
    mask = adata.X != 0
    frac = np.asarray(mask.sum(axis=0)).reshape(-1) / adata.n_obs
    adata.var["sparsity"] = 1 - frac


def one_hot_encoding(labels):
    """tangram/utils.py:105-123: one column per unique label, in order of first appearance."""
    labels = pd.Series(labels).reset_index(drop=True)
    return pd.DataFrame({u: (labels == u).astype(int) for u in labels.unique()})


def pp_adatas(adata_sc, adata_sp, genes=None, gene_to_lowercase=True):
    """mapping_utils.py:20-100 (gene intersection + density priors).  The neighbour graph
    (:95-100) is not computed here: build it with tg.spatial_neighbors(adata_sp), or pass it
    in adata_sp.obsp."""
    for ad in (adata_sc, adata_sp):
        # sc.pp.filter_genes(ad, min_cells=1) (:47-48): records var['n_cells'], then drops the all-zero genes IN PLACE --
        # through AnnData._inplace_subset_var, as scanpy does (assigning a differently shaped X / var to a real AnnData raises)
        n_cells = np.asarray((ad.X != 0).sum(axis=0)).reshape(-1)
        ad.var["n_cells"] = n_cells
        keep = n_cells >= 1
        if not keep.all():
            ad._inplace_subset_var(keep)
    if genes is None:
        genes = adata_sc.var.index
    if gene_to_lowercase:
        adata_sc.var.index = [g.lower() for g in adata_sc.var.index]
        adata_sp.var.index = [g.lower() for g in adata_sp.var.index]
        genes = list(g.lower() for g in genes)
    adata_sc.var_names_make_unique()
    adata_sp.var_names_make_unique()
    genes = list(set(genes) & set(adata_sc.var.index) & set(adata_sp.var.index))
    adata_sc.uns["training_genes"] = genes
    adata_sp.uns["training_genes"] = genes
    logging.info("{} training genes are saved in `uns``training_genes` of both single cell and spatial Anndatas.".format(len(genes)))
    overlap = np.sort(list(set(adata_sc.var.index) & set(adata_sp.var.index))).tolist()
    adata_sc.uns["overlap_genes"] = overlap
    adata_sp.uns["overlap_genes"] = overlap
    logging.info("{} overlapped genes are saved in `uns``overlap_genes` of both single cell and spatial Anndatas.".format(len(overlap)))
    n = adata_sp.X.shape[0]
    adata_sp.obs["uniform_density"] = np.ones(n) / n
    counts = np.array(adata_sp.X.sum(axis=1)).squeeze()
    adata_sp.obs["rna_count_based_density"] = counts / np.sum(counts)


def adata_to_cluster_expression(adata, cluster_label, scale=True, add_density=True):
    """mapping_utils.py:103-139: one observation per cluster (sum if scale else mean)."""
    try:
        value_counts = adata.obs[cluster_label].value_counts(normalize=True)
    except KeyError:
        raise ValueError("Provided label must belong to adata.obs.")
    unique_labels = value_counts.index
    new_obs = pd.DataFrame({cluster_label: unique_labels})
    new_obs.index = new_obs.index.astype(str)
    X_new = np.empty((len(unique_labels), adata.shape[1]))
    lab = np.asarray(adata.obs[cluster_label])
    X = adata.X
    for i, l in enumerate(unique_labels):
        rows = X[np.nonzero(lab == l)[0]]
        X_new[i] = np.asarray(rows.sum(axis=0) if scale else rows.mean(axis=0)).reshape(-1)
    ret = make_adata(X=X_new, obs=new_obs, var=adata.var.copy(), uns=adata.uns)
    if add_density:
        ret.obs["cluster_density"] = ret.obs[cluster_label].map(lambda i: value_counts[i])
    return ret


def _validate_mapping_args(mode, cluster_label, lambda_g1, lambda_d, density_prior, target_count, lambda_f_reg, lambda_count):
    """Argument checks of the reference entry point, same order and messages (mapping_utils.py:206-229).
    Returns the effective lambda_d (a density prior switches the density term on, :214-215)."""
    if lambda_g1 == 0:
        raise ValueError("lambda_g1 cannot be 0.")
    if isinstance(density_prior, str) and density_prior not in ("rna_count_based", "uniform"):
        raise ValueError("Invalid input for density_prior.")
    if density_prior is not None and not lambda_d:
        lambda_d = 1
    checks = (
        (lambda_d > 0 and density_prior is None, "When lambda_d is set, please define the density_prior."),
        (mode not in ("clusters", "cells", "constrained"), 'Argument "mode" must be "cells", "clusters" or "constrained'),
        (mode == "clusters" and cluster_label is None, "A cluster_label must be specified if mode is 'clusters'."),
        (mode == "constrained" and not all([target_count, lambda_f_reg, lambda_count]),
         "target_count, lambda_f_reg and lambda_count must be specified if mode is 'constrained'."),
    )
    for failed, message in checks:
        if failed:
            raise ValueError(message)
    return lambda_d


def _prepare_mapping(adata_sc, adata_sp, cv_train_genes, cluster_label, mode, scale, density_prior, lambda_d, lambda_g1,
                     lambda_g2, lambda_r, lambda_l1, lambda_l2, lambda_count, lambda_f_reg, target_count,
                     lambda_neighborhood_g1, lambda_ct_islands, lambda_getis_ord, lambda_moran, lambda_geary,
                     process_group=None):
    """map_cells_to_space's preparation (mapping_utils.py:206-375): argument checks, cluster aggregation, the training
    genes, S, G, the density prior and the spatial operators.  Returns (adata_sc -- aggregated in clusters mode --,
    training_genes, S, G, the keywords of the mode's mapper class apart from device / random_state / precision)."""
    lambda_d = _validate_mapping_args(mode, cluster_label, lambda_g1, lambda_d, density_prior, target_count,
                                      lambda_f_reg, lambda_count)

    if mode == "clusters":
        adata_sc = adata_to_cluster_expression(adata_sc, cluster_label, scale, add_density=True)

    for ad in (adata_sc, adata_sp):                                              # :237-241
        if not set(["training_genes", "overlap_genes"]).issubset(set(ad.uns.keys())):
            raise ValueError("Missing tangram parameters. Run `pp_adatas()`.")
    assert list(adata_sp.uns["training_genes"]) == list(adata_sc.uns["training_genes"])

    if cv_train_genes is None:                                                   # :246-254
        training_genes = adata_sc.uns["training_genes"]
    elif set(cv_train_genes).issubset(set(adata_sc.uns["training_genes"])):
        training_genes = cv_train_genes
    else:
        raise ValueError("Given training genes list should be subset of two AnnDatas.")

    if process_group is not None:
        # pp_adatas builds the gene list through a set (:57-60): its order depends on the process's string hashing, so
        # the ranks agree on rank 0's order before they slice columns
        import torch.distributed as dist
        box = [list(training_genes)]
        dist.broadcast_object_list(box, src=dist.get_global_rank(process_group, 0), group=process_group)
        training_genes = box[0]

    logging.info("Allocate tensors for mapping.")
    S = _dense_f32(adata_sc[:, training_genes].X)                                # :259-275
    G = _dense_f32(adata_sp[:, training_genes].X)
    if not S.any(axis=0).all() or not G.any(axis=0).all():
        raise ValueError("Genes with all zero values detected. Run `pp_adatas()`.")

    d_source = None                                                              # :280-307
    d_str = density_prior
    if type(density_prior) is np.ndarray:
        d_str = "customized"
    if isinstance(density_prior, str) and density_prior == "rna_count_based":
        density_prior = adata_sp.obs["rna_count_based_density"]
    elif isinstance(density_prior, str) and density_prior == "uniform":
        density_prior = adata_sp.obs["uniform_density"]
    if mode == "cells":
        d = density_prior
    if mode == "clusters":
        d_source = np.array(adata_sc.obs["cluster_density"])
    if mode in ["clusters", "constrained"]:                                       # :300-307
        if density_prior is None:
            d = adata_sp.obs["uniform_density"]
            d_str = "uniform"
        else:
            d = density_prior
        if lambda_d is None or lambda_d == 0:
            lambda_d = 1
    d = None if d is None else np.asarray(d, dtype=np.float32)

    voxel_weights, neighborhood_filter, ct_encode, spatial_weights = None, None, None, None   # :317-329
    if mode == "constrained":
        lambda_neighborhood_g1 = lambda_ct_islands = lambda_getis_ord = lambda_moran = lambda_geary = 0   # not used there (:366-375)
    if lambda_neighborhood_g1 > 0:
        voxel_weights = sw.spatial_weights(adata_sp, standardized=True, self_inclusion=True)
    if lambda_ct_islands > 0:
        if cluster_label not in adata_sc.obs.keys():
            raise ValueError("cluster_label must be specified for the cell type island extension.")
        neighborhood_filter = sw.spatial_weights(adata_sp, standardized=False, self_inclusion=False)
        ct_encode = one_hot_encoding(adata_sc.obs[cluster_label]).values
    if lambda_moran > 0 or lambda_geary > 0:
        raise NotImplementedError("lambda_moran / lambda_geary are not supported by tangram_b200")
    if lambda_getis_ord > 0:
        spatial_weights = sw.spatial_weights(adata_sp, standardized=False, self_inclusion=True)

    if mode == "constrained":                                                     # :366-375
        mapper_kw = dict(S=S, G=G, d=d, lambda_d=lambda_d, lambda_g1=lambda_g1, lambda_g2=lambda_g2, lambda_r=lambda_r,
                         lambda_count=lambda_count, lambda_f_reg=lambda_f_reg, target_count=target_count)
    else:
        mapper_kw = dict(
            S=S, G=G, d=d, lambda_d=lambda_d, lambda_g1=lambda_g1, lambda_g2=lambda_g2, lambda_r=lambda_r,
            lambda_l1=lambda_l1, lambda_l2=lambda_l2, d_source=d_source,
            lambda_neighborhood_g1=lambda_neighborhood_g1, voxel_weights=voxel_weights,
            lambda_ct_islands=lambda_ct_islands, neighborhood_filter=neighborhood_filter,
            ct_encode=ct_encode, lambda_getis_ord=lambda_getis_ord, spatial_weights=spatial_weights)
    logging.info("Begin training with {} genes and {} density_prior in {} mode...".format(len(training_genes), d_str, mode))
    return adata_sc, training_genes, S, G, mapper_kw


def _check_shardable(mode, process_group):
    if process_group is not None and mode == "clusters":
        raise ValueError("process_group shards the cells axis: only mode='cells' can be sharded, and mode='constrained' "
                         "(clusters mode has too few rows).")


def _sum_over_group(partial, device, process_group):
    """A sum over this rank's cells (a projection softmax(M)[r0:r1]^T X, per-label sums, counts) -> the sum over the
    group's ranks, the sum over every cell, the same on every rank, in the partial's dtype; unchanged without a group.
    An NCCL group sums on CUDA device `device` (an ordinal; None: torch's current device), any other backend on the
    host."""
    if process_group is None:
        return partial
    import torch
    import torch.distributed as dist
    t = torch.from_numpy(np.ascontiguousarray(partial))
    t = t.cuda(device) if dist.get_backend(process_group) == "nccl" else t
    dist.all_reduce(t, group=process_group)
    return t.cpu().numpy()


def _make_mapper(mode, mapper_kw, **kw):
    """The mode's mapper class, looked up on the module `mo` at call time (a test can stand another class in there)."""
    if mode == "constrained":
        return mo.MapperConstrained(**mapper_kw, **kw)
    return mo.Mapper(**mapper_kw, **kw)


def map_cells_to_space(
    adata_sc, adata_sp, cv_train_genes=None, cluster_label=None, mode="cells", device="cuda:0",
    learning_rate=0.1, num_epochs=1000, scale=True,
    lambda_d=0, lambda_g1=1, lambda_g2=0, lambda_r=0, lambda_l1=0, lambda_l2=0,
    lambda_count=1, lambda_f_reg=1, target_count=None,
    lambda_neighborhood_g1=0, lambda_ct_islands=0, lambda_getis_ord=0, lambda_moran=0, lambda_geary=0,
    random_state=None, verbose=True, density_prior="rna_count_based", precision="bf16x3",
    process_group=None, gather=False, keep_on_device=False, state_memory="device",
):
    """Same contract as the reference (mapping_utils.py:141-428); `device` must be CUDA.  Added keywords:
    precision       "bf16x3" parity-grade on tensor cores (default) | "fp32" FFMA | "bf16" throughput
    process_group   torch.distributed group, one process per GPU (mode='cells' or 'constrained'): every rank passes the SAME
                    adata_sc / adata_sp; the cells are sharded in contiguous blocks (tangram_b200.shard_rows), each rank
                    draws only its rows of the reference's M0 stream (and, in constrained mode, its entries of F0) and
                    trains them, one NCCL exchange per epoch.  Each rank returns the AnnData of ITS cells (obs = that block
                    of adata_sc.obs, with `obs['F_out']` of those cells in constrained mode; `uns['shard_rows']` =
                    (first, last)); the per-gene scores, the history and `uns` are global and identical on every rank.
                    gather=True: rank 0 additionally receives the full mapping (all cells, and the full F_out) and the
                    other ranks return None.
    state_memory    "device" (default) | "host": keep the mapping and Adam's moments in pinned host memory (each rank its
                    own shard), so that a mapping too large for the GPU trains there with bit-identical results; bf16 and
                    bf16x3 only.  "auto": keep as many rows on the device as fit and only the rest in host memory (each
                    rank plans its own shard on its own device)
    keep_on_device  keep the trained mapper (device state ~20 B per mapping element) attached to the result so that
                    project_genes contracts on the GPU; default: release it (`adata_map.X` is all project_genes needs)."""
    _check_shardable(mode, process_group)
    adata_sc, training_genes, S, G, mapper_kw = _prepare_mapping(
        adata_sc, adata_sp, cv_train_genes, cluster_label, mode, scale, density_prior, lambda_d, lambda_g1, lambda_g2,
        lambda_r, lambda_l1, lambda_l2, lambda_count, lambda_f_reg, target_count, lambda_neighborhood_g1,
        lambda_ct_islands, lambda_getis_ord, lambda_moran, lambda_geary, process_group)
    print_each = 100 if verbose else None

    F_out = None
    if state_memory != "device":       # the mapper classes' default; a stand-in class need not know the keyword
        mapper_kw = dict(mapper_kw, state_memory=state_memory)
    mapper = _make_mapper(mode, mapper_kw, device=device, random_state=random_state, precision=precision,
                          process_group=process_group)
    if mode == "constrained":                                                     # :366-389
        mapping_matrix, F_out, training_history = mapper.train(
            learning_rate=learning_rate, num_epochs=num_epochs, print_each=print_each)
    else:
        mapping_matrix, training_history = mapper.train(
            learning_rate=learning_rate, num_epochs=num_epochs, print_each=print_each)

    logging.info("Saving results..")
    r0, r1 = getattr(mapper, "_rows", (0, S.shape[0]))
    obs_map = adata_sc[:, training_genes].obs.copy()
    if process_group is not None:
        obs_map = obs_map.iloc[r0:r1]
    adata_map = make_adata(X=mapping_matrix, obs=obs_map, var=adata_sp[:, training_genes].obs.copy())
    if process_group is not None:
        adata_map.uns["shard_rows"] = (int(r0), int(r1))

    if mode == "constrained":
        adata_map.obs["F_out"] = F_out                                            # :398-399

    # per-gene training score (:401-410): softmax(M)^T S on the device instead of a host GEMM
    G_predicted = _sum_over_group(mapper.project(S[r0:r1]), _device_index(device), process_group)
    num = (G * G_predicted).sum(axis=0)
    den = np.linalg.norm(G, axis=0) * np.linalg.norm(G_predicted, axis=0)
    df_cs = pd.DataFrame(num / den, list(training_genes), columns=["train_score"])
    df_cs = df_cs.sort_values(by="train_score", ascending=False)
    adata_map.uns["train_genes_df"] = df_cs

    annotate_gene_sparsity(adata_sc)                                             # :412-424
    annotate_gene_sparsity(adata_sp)
    adata_map.uns["train_genes_df"]["sparsity_sc"] = adata_sc[:, training_genes].var.sparsity
    adata_map.uns["train_genes_df"]["sparsity_sp"] = adata_sp[:, training_genes].var.sparsity
    adata_map.uns["train_genes_df"]["sparsity_diff"] = (
        adata_sp[:, training_genes].var.sparsity - adata_sc[:, training_genes].var.sparsity)
    adata_map.uns["training_history"] = training_history
    if keep_on_device and process_group is None:
        try:      # M stays resident for project_genes (not part of `uns`: the AnnData stays serialisable); mapper.release() frees it
            adata_map._tgb200_mapper = mapper
        except Exception:  # noqa: BLE001
            mapper.release()
    else:
        mapper.release()
    if process_group is not None and gather:
        adata_map = _gather_mapping(adata_map, adata_sc[:, training_genes].obs.copy(), process_group, device)
    return adata_map


def _gather_mapping(adata_map, obs_all, pg, device):
    """Rank 0 of the group receives every rank's block of rows (gather_object of the host arrays: result packaging, once
    per mapping) and returns the AnnData over all cells, with the full `obs['F_out']` in constrained mode; the other ranks
    return None."""
    import torch.distributed as dist
    rank, world = dist.get_rank(pg), dist.get_world_size(pg)
    parts = [None] * world if rank == 0 else None
    F_out = np.asarray(adata_map.obs["F_out"]) if "F_out" in adata_map.obs.keys() else None
    dist.gather_object((adata_map.uns["shard_rows"], np.asarray(adata_map.X), F_out), parts,
                       dst=dist.get_global_rank(pg, 0), group=pg)
    if rank != 0:
        return None
    parts.sort(key=lambda p: p[0][0])
    full = make_adata(X=np.concatenate([p[1] for p in parts], axis=0), obs=obs_all, var=adata_map.var)
    if F_out is not None:
        full.obs["F_out"] = np.concatenate([p[2] for p in parts])
    full.uns.update({k: v for k, v in adata_map.uns.items() if k != "shard_rows"})
    return full
