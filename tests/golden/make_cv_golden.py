"""
Golden outputs of gene cross-validation (tangram/utils.py: cross_val, compare_spatial_geneexp, eval_metric) from the
REAL reference, run on the CPU (device="cpu").

Needs a Tangram checkout: the one next to this repository, or the one TANGRAM_REFERENCE names (as oracle/build_ref.py):
    python tests/golden/make_cv_golden.py

The unmodified reference utils.py, mapping_utils.py and mapping_optimizer.py are loaded by path as the `tangram` package.
Stubs stand in for what is not installed: `tangram.spatial_weights` is empty (no spatial term is used), and `scanpy` has
`AnnData` = this repository's MiniAnnData (whose dense X also answers the `.toarray()` the reference calls on an
ndarray, mapping_utils.py:262) and `pp.filter_genes`; mapping_utils gets the mapper classes with the density prior
turned from a pandas Series into an array, which torch 2's torch.tensor requires.  The module `utils` sees numpy through a proxy that adds
`np.float = float` (removed from numpy, used at utils.py:622) and records the per-fold score lists cross_val passes to
np.nanmean.  pp_adatas builds the training genes through a set; they are sorted here, so the order does not depend on
string hashing.  Writes tests/golden/cv.npz: per case <c>_* the inputs (cell and spot matrices, labels, gene names), the
arguments, numpy's generator state before and after the call, the per-fold test and train scores, the averages, the
printed text and, for the leave-one-out case, test_gene_df and adata_ge_cv; and eval_metric's answer on the reference's
data/test_df.csv, whose three columns eval_metric reads (score, is_training, sparsity_sp) go to tests/golden/test_df.csv.gz.
"""
import contextlib
import gzip
import importlib.util
import io
import os
import sys
import types

import numpy as np
import pandas as pd
import scipy.sparse as sp
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from tangram_b200.adata import MiniAnnData  # noqa: E402

REF = os.environ.get("TANGRAM_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")

# name: cells, spots, genes, clusters (0: none), mode, cv_mode, keyword arguments of cross_val
CASES = {
    "clusters_loo": dict(N=60, V=300, K=24, T=6, mode="clusters", cv_mode="loo", seed=1,
                         kw=dict(num_epochs=60, random_state=7, return_gene_pred=True, verbose=True)),
    "clusters_10fold": dict(N=80, V=200, K=31, T=6, mode="clusters", cv_mode="10fold", seed=2,
                            kw=dict(num_epochs=60, random_state=None, lambda_g2=1.0, density_prior="rna_count_based")),
    "cells_10fold": dict(N=150, V=90, K=30, T=0, mode="cells", cv_mode="10fold", seed=3,
                         kw=dict(num_epochs=40, random_state=3, lambda_d=1.0, density_prior="uniform", verbose=True)),
    "constrained_10fold": dict(N=120, V=70, K=25, T=0, mode="constrained", cv_mode="10fold", seed=4,
                               kw=dict(num_epochs=40, random_state=5, target_count=60)),
}
NP_SEED = 123          # numpy's global seed before every call (the random_state=None case draws from it)


class _Dense(np.ndarray):
    """An ndarray with the .toarray() the reference calls on dense X."""

    def toarray(self):
        return np.asarray(self)


def _dense(X):
    return X.view(_Dense) if type(X) is np.ndarray else X


class RefAnnData(MiniAnnData):
    @property
    def X(self):
        return self._X

    @X.setter
    def X(self, value):
        self._X = _dense(value)

    def __getitem__(self, key):
        a = MiniAnnData.__getitem__(self, key)
        return RefAnnData(X=a.X, obs=a.obs, var=a.var, uns=a.uns, obsm=a.obsm, obsp=a.obsp, varm=a.varm)

    def copy(self):
        a = MiniAnnData.copy(self)
        return RefAnnData(X=a.X, obs=a.obs, var=a.var, uns=a.uns, obsm=a.obsm, obsp=a.obsp, varm=a.varm)


def _filter_genes(adata, min_cells=1):
    n_cells = np.asarray((adata.X != 0).sum(axis=0)).reshape(-1)
    adata.var["n_cells"] = n_cells
    keep = n_cells >= min_cells
    if not keep.all():
        adata._inplace_subset_var(keep)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    return spec, mod


def load_reference():
    """-> (tangram.utils, tangram.mapping_utils, the list np.nanmean's arguments land in)."""
    pkg = types.ModuleType("tangram")
    pkg.__path__ = []
    sys.modules["tangram"] = pkg
    sys.modules["tangram.spatial_weights"] = types.ModuleType("tangram.spatial_weights")
    sc = types.ModuleType("scanpy")
    sc.AnnData = RefAnnData
    sc.pp = types.SimpleNamespace(filter_genes=_filter_genes)
    sys.modules["scanpy"] = sc
    spec, mo = _load("tangram.mapping_optimizer", os.path.join(REF, "tangram", "mapping_optimizer.py"))
    spec.loader.exec_module(mo)
    ut_spec, ut = _load("tangram.utils", os.path.join(REF, "tangram", "utils.py"))
    mu_spec, mu = _load("tangram.mapping_utils", os.path.join(REF, "tangram", "mapping_utils.py"))
    mu_spec.loader.exec_module(mu)
    ut_spec.loader.exec_module(ut)

    def as_array(cls):            # map_cells_to_space passes the density prior as a pandas Series, which torch 2's
        def make(*args, d=None, **kw):      # torch.tensor no longer takes (mapping_optimizer.py:116, :464)
            return cls(*args, d=None if d is None else np.asarray(d), **kw)
        return make

    mu.mo = types.SimpleNamespace(Mapper=as_array(mo.Mapper), MapperConstrained=as_array(mo.MapperConstrained))
    means = []

    class _Numpy(types.ModuleType):
        def __getattr__(self, name):
            return getattr(np, name)

    proxy = _Numpy("numpy")
    proxy.float = float

    def nanmean(a, *args, **kw):
        means.append(np.array(a, dtype=np.float64))
        return np.nanmean(a, *args, **kw)

    proxy.nanmean = nanmean
    ut.np = proxy
    return ut, mu, means


def inputs(c):
    """Seeded count-like cells x genes and spots x genes, gene names g00.., cluster labels t0.. (every cluster present,
    every gene expressed somewhere)."""
    rng = np.random.default_rng(c["seed"])
    N, V, K, T = c["N"], c["V"], c["K"], c["T"]
    S = np.log1p(rng.poisson(0.8, (N, K))).astype(np.float32)
    G = np.log1p(rng.poisson(1.5, (V, K))).astype(np.float32)
    S[0] += 1.0
    G[0] += 1.0
    labels = np.array([f"t{i % max(T, 1)}" for i in rng.permutation(N)], dtype=object)
    return S, G, labels


def make_adatas(S, G, labels, cls=MiniAnnData):
    """The two AnnDatas after pp_adatas (restated here: the same training genes, sorted; the density priors)."""
    N, K = S.shape
    V = G.shape[0]
    genes = [f"g{k:02d}" for k in range(K)]
    ad_sc = cls(X=sp.csr_matrix(S), obs=pd.DataFrame({"cell_type": labels}, index=[f"c{i}" for i in range(N)]),
                var=pd.DataFrame(index=genes))
    ad_sp = cls(X=G.copy(), obs=pd.DataFrame(index=[f"s{j}" for j in range(V)]), var=pd.DataFrame(index=list(genes)))
    for ad in (ad_sc, ad_sp):
        ad.var["n_cells"] = np.asarray((ad.X != 0).sum(axis=0)).reshape(-1)
        ad.uns["training_genes"] = list(genes)
        ad.uns["overlap_genes"] = list(genes)
    ad_sp.obs["uniform_density"] = np.ones(V) / V
    counts = np.array(ad_sp.X.sum(axis=1)).squeeze()
    ad_sp.obs["rna_count_based_density"] = counts / np.sum(counts)
    return ad_sc, ad_sp


def run_case(ut, means, name, c):
    S, G, labels = inputs(c)
    ad_sc, ad_sp = make_adatas(S, G, labels, RefAnnData)
    kw = dict(c["kw"])
    if c["mode"] == "clusters":
        kw["cluster_label"] = "cell_type"
    np.random.seed(NP_SEED)
    state0 = np.random.get_state()
    means.clear()
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        out = ut.cross_val(ad_sc, ad_sp, mode=c["mode"], cv_mode=c["cv_mode"], device="cpu", **kw)
    state1 = np.random.get_state()
    cv_dict = out[0] if isinstance(out, tuple) else out
    save = {"S": S, "G": G, "labels": labels.astype(str), "mode": np.array(c["mode"]), "cv_mode": np.array(c["cv_mode"]),
            "np_seed": np.array(NP_SEED), "state_key": state1[1], "state_pos": np.array(state1[2]),
            "state_gauss": np.array([state1[3], state1[4]], dtype=np.float64),
            "test_scores": means[0], "train_scores": means[1],
            "avg_test_score": np.array(cv_dict["avg_test_score"]), "avg_train_score": np.array(cv_dict["avg_train_score"]),
            "printed": np.array(buf.getvalue())}
    for k, v in kw.items():
        save["kw_" + k] = np.array("None" if v is None else v)
    if isinstance(out, tuple):
        _, ge_cv, df = out
        save.update(ge_cv_X=np.asarray(ge_cv.X, dtype=np.float64), ge_cv_genes=np.asarray(ge_cv.var.index).astype(str),
                    ge_cv_test_score=ge_cv.var["test_score"].to_numpy(np.float64),
                    df_genes=np.asarray(df.index).astype(str), df_columns=np.array(list(df.columns)),
                    df_values=df.to_numpy(np.float64))
    assert state0[2] != state1[2] or not np.array_equal(state0[1], state1[1])
    print(name, "folds", len(means[0]), "avg test", cv_dict["avg_test_score"], "avg train", cv_dict["avg_train_score"])
    return {f"{name}_{k}": v for k, v in save.items()}


def main():
    ut, _, means = load_reference()
    torch.set_num_threads(1)
    arrays = {}
    for name, c in CASES.items():
        arrays.update(run_case(ut, means, name, c))
    # eval_metric on the reference's own data fixture (its tests pin auc_score = 0.750597829464878)
    df = pd.read_csv(os.path.join(REF, "data", "test_df.csv"), index_col=0)
    used = df[["score", "is_training", "sparsity_sp"]]
    with gzip.open(os.path.join(HERE, "test_df.csv.gz"), "wt", compresslevel=9, newline="") as f:   # noqa: SIM117
        used.to_csv(f, float_format="%.17g")
    df = pd.read_csv(os.path.join(HERE, "test_df.csv.gz"), index_col=0)      # the reduced copy gives the same answer
    metrics, ((xs, ys), _) = ut.eval_metric(df)
    arrays["eval_test_df"] = np.array([metrics[k] for k in ("avg_test_score", "avg_train_score", "sp_sparsity_score",
                                                            "auc_score")], dtype=np.float64)
    arrays["eval_test_df_curve"] = np.array([np.real(xs), np.real(ys)], dtype=np.float64)
    print("eval_metric(test_df.csv)", metrics)
    np.savez_compressed(os.path.join(HERE, "cv.npz"), **arrays)
    print("-> cv.npz", os.path.getsize(os.path.join(HERE, "cv.npz")) // 1024, "KiB")


if __name__ == "__main__":
    main()
