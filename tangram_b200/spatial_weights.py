"""Sparse restatement of tangram/spatial_weights.py:5-30.  The reference densifies the
~7-nnz/row neighbour graph to V x V (via libpysal / sklearn, absent here); the GPU path
keeps it as scipy CSR end to end (SURVEY.md 8(f) N4)."""
import numpy as np


def spatial_weights(adata_sp, standardized, self_inclusion):
    import scipy.sparse as sp
    if not set(["spatial_connectivities", "spatial_distances"]).issubset(set(adata_sp.obsp.keys())):
        raise ValueError("Missing spatial neighborhood parameters. Run `pp_adatas()` with the spatial information stored in `spatial` in `adata_sp.obsm`.")
    conn = sp.csr_matrix(adata_sp.obsp["spatial_connectivities"])
    if standardized:
        # row-L1-normalised distances (sklearn normalize(norm="l1", axis=1), :16), kept on the
        # connectivity pattern (:17-23)
        g = sp.csr_matrix(adata_sp.obsp["spatial_distances"]).astype(np.float64)
        rs = np.asarray(abs(g).sum(axis=1)).ravel()
        rs[rs == 0] = 1.0
        g = sp.diags(1.0 / rs) @ g
        w = g.multiply(conn != 0).tocsr()
    else:
        w = conn.astype(np.float64)
    if self_inclusion:
        w = w + sp.identity(w.shape[0], format="csr")     # :27-28
    return w.tocsr().astype(np.float32)
