"""tangram_b200: H100-native drop-in for Tangram's map_cells_to_space hot path.

    import tangram_b200 as tg
    tg.pp_adatas(ad_sc, ad_sp); ad_map = tg.map_cells_to_space(ad_sc, ad_sp, device="cuda:0")
    ad_ge = tg.project_genes(ad_map, ad_sc)
    X_space = tg.project(ad_map.X, ad_sc.X)          # mapping^T X on the GPU from any mapping; sparse X stays sparse
    tg.project_cell_annotations(ad_map, ad_sp, annotation="cell_type")   # ad_sp.obsm["tangram_ct_pred"]
    cv_dict = tg.cross_val(ad_sc, ad_sp, cluster_label="cell_type", cv_mode="10fold")   # gene cross-validation
    metrics = tg.train_multiple_Mapper(config, data)     # the tuner's trial: five run-to-run agreement metrics
    tg.rank_genes_groups(ad_sc, groupby="cell_type")     # marker genes per group on the GPU; tg.ctg(ad_sc, "cell_type")
    tg.highly_variable_genes(ad_sc, n_top_genes=4000)    # highly variable genes on the GPU; tg.hvg(ad_sc)
    tg.spatial_neighbors(ad_sp, set_diag=False)          # the spatial neighbour graph on the GPU (squidpy's)

One process per GPU (process_group=pg, cells and constrained mode): every rank passes the same AnnDatas and gets its
block of the mapping; project_genes, project_cell_annotations, cell_type_mapping and count_cell_annotations then take that
block with the same process_group= and return (or write) the result of the whole mapping on every rank.  They run on
torch's current CUDA device, so each rank selects its GPU first:
    torch.cuda.set_device(rank)
    ad_map = tg.map_cells_to_space(ad_sc, ad_sp, device=f"cuda:{rank}", process_group=pg)   # this rank's cells
    ad_ge = tg.project_genes(ad_map, ad_sc, process_group=pg)
    tg.count_cell_annotations(ad_map, ad_sc, ad_sp, annotation="cell_type", process_group=pg)
"""
from .mapping_optimizer import Mapper, MapperConstrained  # noqa: F401
from .sharded import shard_rows  # noqa: F401
from .mapping_utils import (  # noqa: F401
    adata_to_cluster_expression, map_cells_to_space, pp_adatas, annotate_gene_sparsity, one_hot_encoding)
from .utils import (  # noqa: F401
    project_genes, project, annotate, project_cell_annotations, cell_type_mapping, count_cell_annotations, create_segment_cell_df,
    deconvolve_cell_annotations, df_to_cell_types, cross_val, cv_data_gen, compare_spatial_geneexp, eval_metric)
from . import mapping_parameter_tuning  # noqa: F401
from .mapping_parameter_tuning import train_multiple_Mapper  # noqa: F401
from .adata import MiniAnnData  # noqa: F401
from .gene_selection import rank_genes_groups, ctg, highly_variable_genes, hvg  # noqa: F401
from .spatial_neighbors import spatial_neighbors  # noqa: F401

__version__ = "0.2.0"
