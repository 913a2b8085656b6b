"""The reference's own known-answer test for this path (Tangram's tests/tangram_test.py:67-103):
map_cells_to_space(mode='clusters', cluster_label='subclass_label', random_state=42, num_epochs=500) on
data/test_ad_sc.h5ad x data/test_ad_sp.h5ad must give round(ad_map.X[0,0], 3) == round(e, 3) for nine
hyper-parameter sets.  The inputs (cluster-aggregated S, G, priors) are committed as tests/golden/kat_clusters.npz
(tests/golden/make_kat_fixture.py builds them from the reference's .h5ad files with our HDF5 reader + host logic).
CPU: pins the ORACLE to the reference's published values.  GPU: pins the CUDA path to the same values."""
import os

import numpy as np
import pytest

from oracle.tangram_oracle import OracleMapper

Z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kat_clusters.npz"))
CASES = [tuple(r) for r in Z["cases"]]
H5_SC, H5_SP = "/root/reference/data/test_ad_sc.h5ad", "/root/reference/data/test_ad_sp.h5ad"


def _inputs(case):
    g1, g2, ld, dp, scale, e = case
    dp = int(dp)
    S = Z["S_scale"] if scale else Z["S_mean"]
    # mapping_utils.py:280-307, clusters mode: prior None -> uniform; lambda_d forced to 1 when 0
    d = Z["rna_count_based_density"] if dp == 2 else Z["uniform_density"]
    lam_d = ld if (dp != 0 and ld != 0) else 1.0
    kw = dict(S=S, G=Z["G"], d=d.astype(np.float32), d_source=Z["cluster_density"].astype(np.float32),
              lambda_g1=g1, lambda_g2=g2, lambda_d=lam_d, random_state=42)
    return kw, e


def _check(x00, e):
    assert round(float(x00), 3) == round(float(e), 3)          # the reference's own assertion (:103)
    if e > 1e-4:                                                # the one discriminating case (:77)
        assert abs(x00 - e) < 1e-3 * e
    else:
        assert abs(x00 - e) < 0.15 * e                          # 500 chaotic epochs at the 1e-6 level


def _check_train_score(X_space, kw, hist):
    """The reference's test_train_score_match (tests/tangram_test.py:159-211): the mean per-gene cosine between the
    projected training genes (project_genes, tangram/utils.py:368) and the measured ones (compare_spatial_geneexp,
    tangram/utils.py:412-428) equals the last main_loss of the training history to three decimals."""
    A, B = np.asarray(X_space, dtype=np.float64), np.asarray(kw["G"], dtype=np.float64)
    cos = (A * B).sum(axis=0) / (np.linalg.norm(A, axis=0) * np.linalg.norm(B, axis=0))
    assert abs(cos.mean() * kw["lambda_g1"] - float(hist["main_loss"][-1])) < 5e-4


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_reference_known_answers(case):
    kw, e = _inputs(case)
    out, hist = OracleMapper(**kw).train(500, print_each=None)
    assert out.shape == (18, 9852)
    _check(out[0, 0], e)
    _check_train_score(out.astype(np.float64).T @ kw["S"].astype(np.float64), kw, hist)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
@pytest.mark.parametrize("case", CASES)
def test_cuda_reproduces_reference_known_answers(case, precision):
    from tangram_b200 import Mapper
    kw, e = _inputs(case)
    m = Mapper(device="cuda:0", precision=precision, **kw)
    out, hist = m.train(500, print_each=None)
    _check(out[0, 0], e)
    X_space = m.project(kw["S"])                               # project_genes' GEMM on the device
    assert np.allclose(X_space, out.astype(np.float64).T @ kw["S"].astype(np.float64), rtol=2e-5, atol=1e-7)
    _check_train_score(X_space, kw, hist)


@pytest.mark.skipif(not (os.path.exists(H5_SC) and os.path.exists(H5_SP)), reason="reference data not present (GPU box)")
def test_h5ad_reader_and_host_logic_rebuild_the_fixture():
    """HDF5 mini-reader (tangram_b200/h5mini.py, h5ad.py) + cluster aggregation on the real fixtures."""
    import tangram_b200 as tg
    from tangram_b200.h5ad import read_h5ad
    ad_sc, ad_sp = read_h5ad(H5_SC), read_h5ad(H5_SP)
    assert ad_sc.shape == (26431, 249) and ad_sc.X.nnz == 1133906          # SURVEY.md section 2 row 12
    assert ad_sp.shape == (9852, 249) and ad_sp.X.dtype == np.float32
    assert len(ad_sc.obs["subclass_label"].unique()) == 18
    genes = ad_sc.uns["training_genes"]
    assert len(genes) == 249 and list(genes) == list(ad_sp.uns["training_genes"])
    assert np.array_equal(np.asarray(ad_sp[:, genes].X, dtype=np.float32), Z["G"])
    agg = tg.adata_to_cluster_expression(ad_sc, "subclass_label", scale=True)
    assert np.allclose(np.asarray(agg[:, genes].X, dtype=np.float32), Z["S_scale"])
    assert np.allclose(np.asarray(agg.obs["cluster_density"], dtype=np.float64), Z["cluster_density"])
    # density priors as stored in the fixture's obs (pp_adatas ran on the full gene set before the 249-gene subset)
    assert np.allclose(np.asarray(ad_sp.obs["rna_count_based_density"]), Z["rna_count_based_density"])
    assert abs(float(ad_sp.obs["rna_count_based_density"].sum()) - 1.0) < 1e-9
    assert np.allclose(np.asarray(ad_sp.obs["uniform_density"]), 1.0 / 9852)
