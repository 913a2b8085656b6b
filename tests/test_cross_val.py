"""Gene cross-validation on the CPU: the splits of cv_data_gen, compare_spatial_geneexp and eval_metric against the
reference (tests/golden/cv.npz, tests/golden/test_df.csv.gz and, where a Tangram checkout is present, the live reference
functions), and cross_val's orchestration against the reference's golden with an oracle-backed mapper standing in for
the CUDA one: fold order, numpy's generator state after the call, the frames, the prints and the scores."""
import contextlib
import io
import os

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
import torch

import tangram_b200 as tg
from oracle.tangram_oracle import OracleMapper, OracleMapperConstrained
from tangram_b200 import mapping_optimizer as mo
from tangram_b200.adata import MiniAnnData

HERE = os.path.dirname(os.path.abspath(__file__))
Z = np.load(os.path.join(HERE, "golden", "cv.npz"))
CASES = ["clusters_loo", "clusters_10fold", "cells_10fold", "constrained_10fold"]
REF = os.path.join(os.path.dirname(os.path.dirname(HERE)), "reference")


def golden_adatas(case):
    """The golden case's AnnDatas as pp_adatas leaves them (training genes in the stored, sorted order)."""
    S, G, labels = Z[f"{case}_S"], Z[f"{case}_G"], Z[f"{case}_labels"].astype(object)
    N, K = S.shape
    V = G.shape[0]
    genes = [f"g{k:02d}" for k in range(K)]
    ad_sc = MiniAnnData(X=sp.csr_matrix(S), obs=pd.DataFrame({"cell_type": labels}, index=[f"c{i}" for i in range(N)]),
                        var=pd.DataFrame(index=genes))
    ad_sp = MiniAnnData(X=G.copy(), obs=pd.DataFrame(index=[f"s{j}" for j in range(V)]), var=pd.DataFrame(index=list(genes)))
    tg.pp_adatas(ad_sc, ad_sp)
    for ad in (ad_sc, ad_sp):
        ad.uns["training_genes"] = list(genes)
    return ad_sc, ad_sp


def golden_kwargs(case):
    kw = {}
    for key in Z.files:
        if key.startswith(f"{case}_kw_"):
            v = Z[key].item()
            kw[key[len(f"{case}_kw_"):]] = None if v == "None" else v
    if str(Z[f"{case}_mode"]) == "clusters":
        kw["cluster_label"] = "cell_type"
    return dict(mode=str(Z[f"{case}_mode"]), cv_mode=str(Z[f"{case}_cv_mode"]), **kw)


def run_golden(case, **extra):
    """cross_val on the golden case from numpy's seed; -> (output, printed text)."""
    ad_sc, ad_sp = golden_adatas(case)
    np.random.seed(int(Z[f"{case}_np_seed"]))
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        out = tg.cross_val(ad_sc, ad_sp, **golden_kwargs(case), **extra)
    return out, buf.getvalue()


def check_against_golden(case, out, printed, tol):
    """Scores, averages, numpy's generator state, prints and (leave-one-out) frames against the reference's."""
    cv_dict = out[0] if isinstance(out, tuple) else out
    assert abs(cv_dict["avg_test_score"] - Z[f"{case}_avg_test_score"]) < tol
    assert abs(cv_dict["avg_train_score"] - Z[f"{case}_avg_train_score"]) < tol
    state = np.random.get_state()
    assert np.array_equal(state[1], Z[f"{case}_state_key"]) and state[2] == int(Z[f"{case}_state_pos"])
    assert [state[3], state[4]] == list(Z[f"{case}_state_gauss"])
    ref_lines, got_lines = str(Z[f"{case}_printed"]).splitlines(), printed.splitlines()
    assert len(got_lines) == len(ref_lines)
    for g, r in zip(got_lines, ref_lines):         # same text; a printed 3-decimal value may sit on a rounding edge
        assert g.split(":")[0] == r.split(":")[0]
        gv = [float(x) for x in g.replace("-", " ").split() if x.replace(".", "").isdigit() and "." in x]
        rv = [float(x) for x in r.replace("-", " ").split() if x.replace(".", "").isdigit() and "." in x]
        assert np.allclose(gv, rv, atol=1.01e-3), (g, r)
    if isinstance(out, tuple):
        _, ge_cv, df = out
        assert list(ge_cv.var.index) == list(Z[f"{case}_ge_cv_genes"])
        assert list(ge_cv.obs.index) == [f"s{j}" for j in range(Z[f"{case}_G"].shape[0])]
        np.testing.assert_allclose(ge_cv.var["test_score"].to_numpy(), Z[f"{case}_ge_cv_test_score"], atol=tol)
        X = np.asarray(ge_cv.X, dtype=np.float64)
        ref = Z[f"{case}_ge_cv_X"]
        assert X.shape == ref.shape and np.linalg.norm(X - ref) / np.linalg.norm(ref) < tol
        assert list(df.columns) == list(Z[f"{case}_df_columns"])
        assert list(df.index) == list(Z[f"{case}_df_genes"])
        np.testing.assert_allclose(df.to_numpy(np.float64), Z[f"{case}_df_values"], atol=tol)


# ---------------------------------------------------------------------------------------------------------------------
class OracleCVMapper:
    """The surface cross_val drives -- the constructor's draw, _draw_initial_mapping, _set_loss_genes, _fit(fetch=False),
    history_matrix, project, release -- over the CPU oracle: every fit trains a fresh oracle mapper on the active gene
    columns from the drawn initial mapping, which is what a masked handle must compute."""
    constrained = False
    fits = []

    def __init__(self, S, G, d=None, device=None, random_state=None, precision=None, **kw):
        self.S, self.G, self.d, self.kw, self.random_state = S, G, d, kw, random_state
        self.active = np.ones(S.shape[1], dtype=bool)
        self._draw_initial_mapping()

    def _draw_initial_mapping(self):
        if self.random_state:
            np.random.seed(seed=self.random_state)
        N, V = self.S.shape[0], self.G.shape[0]
        if self.constrained:
            np.random.normal(0, 1, (N, V))
        self.M0 = np.random.normal(0, 1, (N, V))
        self.F0 = np.random.normal(0, 1, N) if self.constrained else None

    def _set_loss_genes(self, active):
        self.active = np.asarray(active, dtype=bool)

    def _fit(self, num_epochs, lr, print_each, resume, fetch=True):
        assert not resume and not fetch and print_each is None
        a = self.active
        type(self).fits.append(a.copy())
        with contextlib.redirect_stdout(io.StringIO()):
            if self.constrained:
                o = OracleMapperConstrained(self.S[:, a], self.G[:, a], self.d, M0=self.M0, F0=self.F0, **self.kw)
                o.train(num_epochs, lr, print_each=None)
                main = o.float_history["main_loss"]
            else:
                o = OracleMapper(self.S[:, a], self.G[:, a], d=self.d, M0=self.M0, **self.kw)
                _, h = o.train(num_epochs, lr, print_each=None)
                main = h["main_loss"]
        self.history_matrix = np.full((num_epochs, 16), np.nan, dtype=np.float32)
        self.history_matrix[:, 1] = main
        self.P = torch.softmax(o.M, dim=1).numpy()

    def project(self, X):
        return (self.P.T @ np.asarray(X, dtype=np.float32)).astype(np.float32)

    def release(self):
        pass


class OracleCVMapperConstrained(OracleCVMapper):
    constrained = True


@pytest.mark.parametrize("case", CASES)
def test_cross_val_orchestration_matches_reference(case, monkeypatch):
    monkeypatch.setattr(mo, "Mapper", OracleCVMapper)
    monkeypatch.setattr(mo, "MapperConstrained", OracleCVMapperConstrained)
    OracleCVMapper.fits = []
    out, printed = run_golden(case)
    check_against_golden(case, out, printed, 1e-4)
    # one fit per fold, in cv_data_gen's order, each over its training genes
    genes = list(golden_adatas(case)[1].uns["training_genes"])
    folds = list(tg.cv_data_gen(*golden_adatas(case), cv_mode=str(Z[f"{case}_cv_mode"])))
    assert len(OracleCVMapper.fits) == len(folds)
    for active, (train, _) in zip(OracleCVMapper.fits, folds):
        assert [g for g, on in zip(genes, active) if on] == train
    cv = out[0] if isinstance(out, tuple) else out
    scores = Z[f"{case}_test_scores"]
    assert abs(np.nanmean(scores) - cv["avg_test_score"]) < 1e-4


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [10, 11, 24, 37, 249])
def test_cv_data_gen_equals_sklearn(n):
    from sklearn.model_selection import KFold, LeaveOneOut
    genes = [f"g{i}" for i in range(n)]
    ad = MiniAnnData(X=np.ones((2, n), np.float32), var=pd.DataFrame(index=genes), uns={"training_genes": genes})
    arr = np.array(genes)
    for mode, cv in (("loo", LeaveOneOut()), ("10fold", KFold(n_splits=10))):
        got = list(tg.cv_data_gen(ad, ad, cv_mode=mode))
        want = [(list(arr[a]), list(arr[b])) for a, b in cv.split(arr)]
        assert got == want


def test_cv_data_gen_errors():
    genes = ["a", "b", "c"]
    ad = MiniAnnData(X=np.ones((2, 3), np.float32), uns={"training_genes": genes})
    other = MiniAnnData(X=np.ones((2, 3), np.float32), uns={"training_genes": genes[::-1]})
    bare = MiniAnnData(X=np.ones((2, 3), np.float32))
    with pytest.raises(ValueError, match="Run `pp_adatas\\(\\)`"):
        next(tg.cv_data_gen(bare, ad))
    with pytest.raises(ValueError, match="Run `pp_adatas\\(\\)`"):
        next(tg.cv_data_gen(ad, bare))
    with pytest.raises(ValueError, match="Unmatched training_genes"):
        next(tg.cv_data_gen(ad, other))
    with pytest.raises(ValueError, match="cv_mode"):
        next(tg.cv_data_gen(ad, ad, cv_mode="5fold"))
    with pytest.raises(ValueError, match="n_splits=10"):
        next(tg.cv_data_gen(ad, ad, cv_mode="10fold"))


def _test_df():
    return pd.read_csv(os.path.join(HERE, "golden", "test_df.csv.gz"), index_col=0)


def test_eval_metric_known_answer():
    """The reference's own known answer (its tests/tangram_test.py:214-216) on its data fixture."""
    metrics, ((xs, ys), (raw_x, raw_y)) = tg.eval_metric(_test_df())
    assert metrics["auc_score"] == pytest.approx(0.750597829464878)
    want = Z["eval_test_df"]
    got = [metrics[k] for k in ("avg_test_score", "avg_train_score", "sp_sparsity_score", "auc_score")]
    np.testing.assert_allclose(got, want, rtol=1e-12)
    np.testing.assert_allclose(np.array([xs, ys], dtype=np.float64), Z["eval_test_df_curve"], rtol=1e-12)


def test_eval_metric_auc_and_test_genes():
    from sklearn.metrics import auc
    df = _test_df()
    test = list(df.index[df["is_training"] == False][:300]) + ["igf2"]     # noqa: E712  a training gene, given explicitly
    metrics, ((xs, ys), _) = tg.eval_metric(df, test_genes=test + test[:5])    # duplicates collapse (np.unique)
    assert metrics["auc_score"] == pytest.approx(np.real(auc(xs, ys)), abs=1e-15)
    sub = df.loc[np.unique(test)]
    assert metrics["avg_test_score"] == pytest.approx(sub["score"].mean())
    with pytest.raises(ValueError, match="subset of genes"):
        tg.eval_metric(df, test_genes=["not_a_gene"])


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "tangram")), reason="no Tangram checkout next to this repository")
def test_compare_and_eval_metric_equal_live_reference():
    from tests.golden import make_cv_golden as gen
    ut, _, _ = gen.load_reference()
    rng = np.random.default_rng(5)
    for case in ("cells_10fold", "clusters_loo"):
        S, G = Z[f"{case}_S"], Z[f"{case}_G"]
        genes = [f"g{k:02d}" for k in range(S.shape[1])]
        pred = rng.random((G.shape[0], S.shape[1])).astype(np.float32)
        pred[:, 3] = 0.0                                              # a zero column: NaN score, as in the reference
        out = {}
        for name, f, cls in (("ref", ut.compare_spatial_geneexp, gen.RefAnnData), ("ours", tg.compare_spatial_geneexp, MiniAnnData)):
            ad_sc, ad_sp = gen.make_adatas(S, G, Z[f"{case}_labels"].astype(object), cls)
            var = pd.DataFrame({"is_training": [k % 3 != 0 for k in range(len(genes))]}, index=genes)
            ad_ge = cls(X=pred.copy(), obs=ad_sp.obs.copy(), var=var, uns=ad_sc.uns)
            out[name] = (f(ad_ge, ad_sp), f(ad_ge, ad_sp, ad_sc, genes[5:17]), ad_sp.var["sparsity"].to_numpy())
        for got, want in zip(out["ours"], out["ref"]):
            if isinstance(want, pd.DataFrame):
                pd.testing.assert_frame_equal(got, want, check_exact=True)
            else:
                np.testing.assert_array_equal(got, want)
        df = out["ref"][0].dropna()                 # polyfit does not take the NaN score
        m_ref, c_ref = ut.eval_metric(df)
        m_got, c_got = tg.eval_metric(df)
        assert set(m_ref) == set(m_got)
        for k in m_ref:
            assert m_got[k] == pytest.approx(m_ref[k], rel=1e-12, nan_ok=True)
