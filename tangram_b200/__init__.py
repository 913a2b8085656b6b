"""tangram_b200: H100-native drop-in for Tangram's map_cells_to_space hot path.

    import tangram_b200 as tg
    tg.pp_adatas(ad_sc, ad_sp); ad_map = tg.map_cells_to_space(ad_sc, ad_sp, device="cuda:0")
    ad_ge = tg.project_genes(ad_map, ad_sc)
    metrics = tg.train_multiple_Mapper(config, data)     # the tuner's trial: five run-to-run agreement metrics
"""
from .mapping_optimizer import Mapper, MapperConstrained  # noqa: F401
from .sharded import shard_rows  # noqa: F401
from .mapping_utils import (  # noqa: F401
    adata_to_cluster_expression, map_cells_to_space, pp_adatas, annotate_gene_sparsity, one_hot_encoding)
from .utils import project_genes  # noqa: F401
from . import mapping_parameter_tuning  # noqa: F401
from .mapping_parameter_tuning import train_multiple_Mapper  # noqa: F401
from .adata import MiniAnnData  # noqa: F401

__version__ = "0.2.0"
