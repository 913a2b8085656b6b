"""cross_val(process_group=) on the CPU: two gloo processes, with the oracle-backed stand-in of tests/test_cross_val.py
sharded by cells in place of the CUDA mapper.  What is tested is the host contract of the sharded cross-validation:

* the folds and the gene columns follow rank 0's order of the training genes, also when the other rank's
  uns["training_genes"] lists them in another order (pp_adatas builds that list through a set);
* each rank projects the test genes from its own rows only, and the projections are summed over the group;
* every rank returns the same cv_dict (and adata_ge_cv / test_gene_df), equal to the unsharded cross_val's.
"""
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

import tangram_b200 as tg
from tangram_b200 import mapping_optimizer as mo
from tangram_b200.sharded import shard_rows
from tests.test_cross_val import OracleCVMapper, golden_adatas, golden_kwargs, Z


class _Sharded:
    """The stand-in's fit runs on every rank over all cells (the oracle does not shard); project() sees only this rank's
    rows, as the sharded Mapper's does, so the result is right only if cross_val sums the ranks' projections."""

    def __init__(self, S, G, d=None, process_group=None, draw_whole_stream=None, **kw):
        rank, world = dist.get_rank(process_group), dist.get_world_size(process_group)
        self._rows = shard_rows(S.shape[0], rank, world)
        # the oracle stand-in always draws every row; what is recorded is whether cross_val asked for the whole stream
        type(self).draw_whole_stream = draw_whole_stream
        super().__init__(S, G, d=d, **kw)

    def project(self, X):
        r0, r1 = self._rows
        assert X.shape[0] == r1 - r0, "a rank projects the rows of its own cells"
        return (self.P[r0:r1].T @ np.asarray(X, dtype=np.float32)).astype(np.float32)


class ShardedCVMapper(_Sharded, OracleCVMapper):
    fits = []


class ShardedCVMapperConstrained(_Sharded, OracleCVMapper):
    constrained = True
    fits = []


def _run(case, cv_mode, random_state, process_group=None, reverse_genes=False):
    """cross_val on the golden case from numpy's seed -> (cv_dict, gene predictions or None, the fits' active masks)."""
    import contextlib
    import io
    ad_sc, ad_sp = golden_adatas(case)
    if reverse_genes:
        for ad in (ad_sc, ad_sp):
            ad.uns["training_genes"] = list(ad.uns["training_genes"])[::-1]
    kw = golden_kwargs(case)
    kw.update(cv_mode=cv_mode, random_state=random_state, return_gene_pred=cv_mode == "loo", verbose=False)
    np.random.seed(int(Z[f"{case}_np_seed"]))
    with contextlib.redirect_stdout(io.StringIO()):
        out = tg.cross_val(ad_sc, ad_sp, process_group=process_group, **kw)
    if isinstance(out, tuple):
        cv, ge, df = out
        pred = dict(X=np.asarray(ge.X), genes=list(ge.var.index), test_score=ge.var["test_score"].to_numpy(),
                    df=df.to_numpy(np.float64), df_genes=list(df.index))
    else:
        cv, pred = out, None
    return dict(cv=cv, pred=pred)


def _worker(rank, world, port, case, cv_mode, random_state, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    mo.Mapper, mo.MapperConstrained = ShardedCVMapper, ShardedCVMapperConstrained
    got = _run(case, cv_mode, random_state, dist.group.WORLD, reverse_genes=rank == 1)
    got["fits"] = [a.copy() for a in ShardedCVMapper.fits + ShardedCVMapperConstrained.fits]
    cls = ShardedCVMapperConstrained if case.startswith("constrained") else ShardedCVMapper
    got["whole_stream"] = cls.draw_whole_stream
    out[rank] = got
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("case,cv_mode,random_state", [("cells_10fold", "10fold", 3), ("cells_10fold", "loo", None),
                                                       ("constrained_10fold", "10fold", 5)])
def test_sharded_cross_val_two_rank_gloo(case, cv_mode, random_state, monkeypatch):
    monkeypatch.setattr(mo, "Mapper", OracleCVMapper)
    monkeypatch.setattr(mo, "MapperConstrained", type("C", (OracleCVMapper,), {"constrained": True}))
    OracleCVMapper.fits = []
    want = _run(case, cv_mode, random_state)
    want_fits = list(OracleCVMapper.fits)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = mp.Manager().dict()
    mp.spawn(_worker, args=(2, port, case, cv_mode, random_state, out), nprocs=2, join=True)
    for r in range(2):
        got = out[r]
        # rank 1 listed the genes in reverse: its folds and columns are rank 0's all the same
        assert len(got["fits"]) == len(want_fits)
        for a, b in zip(got["fits"], want_fits):
            assert np.array_equal(a, b), f"rank {r}: a fold trains other genes than the unsharded fold"
        # cells mode: each fold's draw must leave numpy's generator where the unsharded draw does; a sharded
        # MapperConstrained always draws the whole stream and takes no such keyword
        assert got["whole_stream"] is (True if case.startswith("cells") else None), got["whole_stream"]
        for k in ("avg_test_score", "avg_train_score"):
            assert got["cv"][k] == pytest.approx(want["cv"][k], abs=1e-6), (r, k)
            assert got["cv"][k] == out[0]["cv"][k], f"rank {r} {k} differs from rank 0's"
        if want["pred"] is None:
            assert got["pred"] is None
            continue
        p, w, p0 = got["pred"], want["pred"], out[0]["pred"]
        assert p["genes"] == w["genes"] and p["df_genes"] == w["df_genes"]
        np.testing.assert_allclose(p["X"], w["X"], rtol=1e-5, atol=1e-7)
        np.testing.assert_allclose(p["test_score"], w["test_score"], atol=1e-6)
        np.testing.assert_allclose(p["df"], w["df"], atol=1e-6)
        for k in ("X", "test_score", "df"):
            assert np.array_equal(p[k], p0[k]), f"rank {r} {k} differs from rank 0's"


def test_sharded_cross_val_refuses_clusters_mode():
    ad_sc, ad_sp = golden_adatas("clusters_loo")
    with pytest.raises(ValueError, match="process_group shards the cells axis"):
        tg.cross_val(ad_sc, ad_sp, cluster_label="cell_type", mode="clusters", process_group=object())
