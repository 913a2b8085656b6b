"""Gene cross-validation on the GPU.

The training-gene mask of the loss (tgb200_set_loss_genes): a handle over all genes with mask `a` must compute what a
handle created on S[:, a], G[:, a] computes from the same initial mapping -- history and mapping over 30 steps within
1e-5 (fp32, bf16x3) or the bf16 bounds of the smoke test -- in cells, clusters and constrained mode, with lambda_g2, the
neighbourhood and Getis-Ord terms, inactive genes first, last and in the middle, and through the 2-chunk bf16 pipeline.
dL/dY is exactly 0 on inactive gene columns; an all-ones mask is no mask, bit for bit; validation_terms follow the mask.

cross_val against the reference's golden (tests/golden/cv.npz) in bf16x3 and fp32, against our own per-fold public path
(map_cells_to_space(cv_train_genes=...) + project_genes + compare_spatial_geneexp), and on the reference's real data."""
import contextlib
import io
import os

import numpy as np
import pytest

import tangram_b200 as tg
from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph, synthetic_inputs
from tangram_b200 import _lib
from tangram_b200.mapping_optimizer import Mapper, MapperConstrained
from tests.test_cross_val import CASES, Z, check_against_golden, golden_adatas, golden_kwargs, run_golden

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
STEPS = 30


def _mask(K, where):
    a = np.ones(K, dtype=bool)
    if where == "first":
        a[:3] = False
    elif where == "last":
        a[-2:] = False
    else:
        a[[5, 6, 11, K // 2]] = False
    return a


def _inputs(kind, N=300, V=120, K=40, seed=3):
    inp = synthetic_inputs(N, V, K, seed=seed, clusters=kind == "clusters")
    kw = dict(d=inp["d"], lambda_d=1.0)
    if kind == "clusters":
        kw["d_source"] = inp["d_source"]
    if kind == "spatial":
        conn, dist = grid_graph(V)
        kw.update(lambda_neighborhood_g1=0.8, voxel_weights=spatial_weights_from_graph(conn, dist, True, True),
                  lambda_getis_ord=0.6, spatial_weights=spatial_weights_from_graph(conn, dist, False, True),
                  lambda_g2=0.5)
    if kind == "g2":
        kw["lambda_g2"] = 1.0
    return inp["S"], inp["G"], kw


def _pair(kind, precision, where, N=300):
    S, G, kw = _inputs(kind, N=N)
    a = _mask(S.shape[1], where)
    rng = np.random.default_rng(7)
    M0 = rng.standard_normal((S.shape[0], G.shape[0])).astype(np.float32)
    if kind == "constrained":
        F0 = rng.standard_normal(S.shape[0]).astype(np.float32)
        ckw = dict(d=kw["d"], lambda_d=1.0, lambda_g2=1.0, precision=precision, M0=M0, F0=F0, target_count=100)
        full, sub = MapperConstrained(S, G, **ckw), MapperConstrained(S[:, a], G[:, a], **ckw)
    else:
        full = Mapper(S, G, precision=precision, M0=M0, **kw)
        sub = Mapper(S[:, a], G[:, a], precision=precision, M0=M0, **kw)
    full._set_loss_genes(a)
    return full, sub, a


def _train(m):
    with contextlib.redirect_stdout(io.StringIO()):
        out = m.train(STEPS, print_each=None)
    return out[0], m.history_matrix


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
@pytest.mark.parametrize("kind,where", [("cells", "first"), ("clusters", "last"), ("constrained", "middle"),
                                        ("g2", "middle"), ("spatial", "first")])
def test_masked_handle_equals_subset_handle(kind, where, precision):
    full, sub, a = _pair(kind, precision, where)
    P_full, h_full = _train(full)
    P_sub, h_sub = _train(sub)
    tol_h, tol_P = (1e-3, 2e-2) if precision == "bf16" else (1e-5, 1e-5)
    cols = [c for c in range(12) if not np.isnan(h_sub[:, c]).all()]
    assert np.isnan(h_full[:, [c for c in range(12) if c not in cols]]).all()
    np.testing.assert_allclose(h_full[:, cols], h_sub[:, cols], atol=tol_h, rtol=tol_h)
    assert np.linalg.norm(P_full - P_sub) / np.linalg.norm(P_sub) < tol_P
    if kind != "constrained":
        v_full, v_sub = full.validation_terms(), sub.validation_terms()
        for k in v_sub:
            assert v_full[k] == pytest.approx(v_sub[k], abs=1e-3 if precision == "bf16" else 1e-5), k
    full.release(), sub.release()


def test_masked_bf16_two_chunk_pipeline(monkeypatch):
    monkeypatch.setenv("TGB200_CHUNKS", "2")
    full, sub, a = _pair("cells", "bf16", "middle", N=1024)
    P_full, h_full = _train(full)
    P_sub, h_sub = _train(sub)
    np.testing.assert_allclose(h_full[:, :2], h_sub[:, :2], atol=1e-3)
    assert np.linalg.norm(P_full - P_sub) / np.linalg.norm(P_sub) < 2e-2


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_dY_is_zero_on_inactive_genes(precision):
    full, _, a = _pair("spatial", precision, "middle")
    e = full._engine
    e.step_begin()
    e.step_end(0.1)
    K, V = full.n_genes, full.n_voxels
    dY = e.debug("dY").reshape(V, -1)
    assert (dY[:, :K][:, ~a] == 0).all()
    assert (dY[:, :K][:, a] != 0).any()


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_all_ones_mask_is_no_mask(precision):
    S, G, kw = _inputs("g2")
    M0 = np.random.default_rng(1).standard_normal((S.shape[0], G.shape[0])).astype(np.float32)
    a, b = Mapper(S, G, precision=precision, M0=M0, **kw), Mapper(S, G, precision=precision, M0=M0, **kw)
    a._set_loss_genes(np.ones(S.shape[1], dtype=bool))
    b._set_loss_genes(_mask(S.shape[1], "first"))
    b._set_loss_genes(None)                           # masked, then back to every gene
    Pa, ha = _train(a)
    Pb, hb = _train(b)
    c = Mapper(S, G, precision=precision, M0=M0, **kw)
    Pc, hc = _train(c)
    for P, h in ((Pa, ha), (Pb, hb)):
        assert np.array_equal(P, Pc) and np.array_equal(h, hc, equal_nan=True)


def test_set_loss_genes_errors():
    S, G, kw = _inputs("cells", N=64, V=40, K=12)
    m = Mapper(S, G, precision="fp32", M0=np.zeros((64, 40), np.float32), **kw)
    e = m._engine
    with pytest.raises(_lib.TangramB200Error, match="no gene is active"):
        e.set_loss_genes(np.zeros(12, dtype=bool))
    with pytest.raises(_lib.TangramB200Error, match="expected 0 or 1"):
        e.set_loss_genes(np.full(12, 2, dtype=np.uint8))
    with pytest.raises(ValueError):
        e.set_loss_genes(np.ones(11, dtype=bool))
    e.step_begin()
    with pytest.raises(_lib.TangramB200Error, match="inside a step"):
        e.set_loss_genes(_mask(12, "first"))
    e.step_end(0.1)
    e.set_loss_genes(_mask(12, "first"))
    assert _lib.load().tgb200_set_loss_genes(None, None, None) == -1           # TGB200_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16x3", "fp32"])
@pytest.mark.parametrize("case", CASES)
def test_cross_val_matches_reference_golden(case, precision):
    out, printed = run_golden(case, precision=precision)
    check_against_golden(case, out, printed, 1e-4)


def _per_fold_public_path(case, precision):
    """Per fold: map_cells_to_space(cv_train_genes=...) + project_genes + compare_spatial_geneexp, as the reference's
    cross_val does it; -> (test scores, train scores)."""
    ad_sc, ad_sp = golden_adatas(case)
    kw = golden_kwargs(case)
    cv_mode = kw.pop("cv_mode")
    mode = kw.pop("mode")
    for k in ("return_gene_pred", "verbose"):
        kw.pop(k, None)
    num_epochs = kw.pop("num_epochs")
    kw.setdefault("density_prior", None)             # cross_val's default; map_cells_to_space's is "rna_count_based"
    cluster_label = kw.pop("cluster_label", None)
    ref = tg.adata_to_cluster_expression(ad_sc, cluster_label, True) if mode == "clusters" else ad_sc
    tests, trains = [], []
    for train, test in tg.cv_data_gen(ad_sc, ad_sp, cv_mode):
        ad_map = tg.map_cells_to_space(ad_sc, ad_sp, cv_train_genes=train, mode=mode, num_epochs=num_epochs,
                                       cluster_label=cluster_label, verbose=False, precision=precision, **kw)
        ge = tg.project_genes(ad_map, ad_sc[:, train + test], cluster_label=cluster_label)
        df = tg.compare_spatial_geneexp(ge, ad_sp, ref, train + test)
        tests.append(df.loc[test]["score"].mean())
        trains.append(float(ad_map.uns["training_history"]["main_loss"][-1]))
    return np.array(tests), np.array(trains)


@pytest.mark.parametrize("case", ["clusters_10fold", "cells_10fold", "constrained_10fold"])
def test_cross_val_equals_per_fold_public_path(case, capsys):
    np.random.seed(int(Z[f"{case}_np_seed"]))         # both paths draw every fold's M0 from the same stream
    want_test, want_train = _per_fold_public_path(case, "bf16x3")
    np.random.seed(int(Z[f"{case}_np_seed"]))
    ad_sc, ad_sp = golden_adatas(case)
    out = tg.cross_val(ad_sc, ad_sp, **{**golden_kwargs(case), "verbose": True})
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("cv set")]
    got_train = np.array([float(ln.split("train score: ")[1].split("-")[0]) for ln in lines])
    got_test = np.array([float(ln.split("test score: ")[1]) for ln in lines])
    np.testing.assert_allclose(got_train, want_train, atol=1.01e-3)      # printed to 3 decimals
    np.testing.assert_allclose(got_test, want_test, atol=1.01e-3)
    assert abs(out["avg_test_score"] - np.nanmean(want_test)) < 1e-4
    assert abs(out["avg_train_score"] - np.nanmean(want_train)) < 1e-4


def test_cross_val_reference_data_10fold():
    """The reference's test data, cluster-aggregated (tests/golden/kat_clusters.npz: 18 clusters x 9852 spots x 249
    genes), one pseudo-cell per cluster: 10-fold cross_val completes and equals the per-fold public path."""
    import pandas as pd
    import scipy.sparse as sp
    k = np.load(os.path.join(HERE, "golden", "kat_clusters.npz"))
    S, G = k["S_scale"].astype(np.float32), k["G"].astype(np.float32)
    n, K = S.shape
    genes = [f"gene{i}" for i in range(K)]
    ad_sc = tg.MiniAnnData(X=sp.csr_matrix(S), obs=pd.DataFrame({"cl": [f"c{i}" for i in range(n)]}, index=[f"c{i}" for i in range(n)]),
                           var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=G.copy(), obs=pd.DataFrame(index=[f"s{j}" for j in range(G.shape[0])]), var=pd.DataFrame(index=list(genes)))
    tg.pp_adatas(ad_sc, ad_sp)
    for ad in (ad_sc, ad_sp):
        ad.uns["training_genes"] = sorted(ad.uns["training_genes"])
    epochs = 200
    with contextlib.redirect_stdout(io.StringIO()):
        out = tg.cross_val(ad_sc, ad_sp, cluster_label="cl", mode="clusters", cv_mode="10fold", num_epochs=epochs,
                           random_state=42)
    assert np.isfinite(out["avg_test_score"]) and 0 < out["avg_test_score"] < 1
    tests = []
    for train, test in tg.cv_data_gen(ad_sc, ad_sp, "10fold"):
        ad_map = tg.map_cells_to_space(ad_sc, ad_sp, cv_train_genes=train, mode="clusters", cluster_label="cl",
                                       num_epochs=epochs, random_state=42, verbose=False, density_prior=None)
        ge = tg.project_genes(ad_map, ad_sc[:, train + test], cluster_label="cl")
        tests.append(tg.compare_spatial_geneexp(ge, ad_sp, genes=test)["score"].mean())
    assert abs(out["avg_test_score"] - np.nanmean(tests)) < 1e-4
