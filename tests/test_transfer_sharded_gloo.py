"""Gene projection and annotation transfer from a cell-sharded mapping, on the CPU: two and three gloo processes, each
holding a block of rows of the golden mappings in tests/golden/annotations.npz, call project_genes,
project_cell_annotations, cell_type_mapping and count_cell_annotations with process_group=.  `annotate` has no CPU path,
so a float64 numpy stand-in takes its place; project_genes runs its host GEMM.

* every rank gets the same results, equal to the reference's golden outputs and to the unsharded calls on the whole
  mapping (the counts and the deconvolved cells exactly, the sums to rounding);
* the blocks are uneven, one of them empty, and the labels are awkward: a label first seen on a later rank, one present
  on rank 1 only, NaN labels first seen on rank 0 or rank 1 (one NaN column all the same), categorical labels, and
  float labels with NaNs on two ranks (numeric cluster ids with missing values);
* a missing uns["shard_rows"] on one rank, overlapping blocks, blocks that miss cells of adata_sc, one rank's obs index
  out of place and cluster_label on one rank are refused with ValueError on every rank, and the group stays usable.
"""
import datetime
import gzip
import os
import pickle
import re
import socket

import numpy as np
import pandas as pd
import pytest
import scipy.sparse as sp
import torch.distributed as dist
import torch.multiprocessing as mp

from tangram_b200 import MiniAnnData, utils
from tangram_b200.sharded import shard_rows
from tests.helpers import GOLDEN_DIR

Z = np.load(os.path.join(GOLDEN_DIR, "annotations.npz"))
with open(os.path.join(GOLDEN_DIR, "annotations_frames.pkl.gz"), "rb") as _f:
    FRAMES = pickle.loads(gzip.decompress(_f.read()))
CASES = ["mixed", "mixed_cat", "mixed_float", "wide", "single", "fout"]
# mixed: T first at row 0, NaN at 5 (also 50, 200), B at 7, Mono at 10, "solo" at 17 only
BLOCKS = {2: {"mixed": [(0, 5), (5, 301)], "mixed_cat": [(0, 9), (9, 301)]},
          3: {"mixed": [(0, 7), (7, 7), (7, 301)], "mixed_cat": [(0, 3), (3, 160), (160, 301)]}}
TRAIN_GENES = ["g1", "g4", "g2-1"]
# mixed_float: the labels of "mixed" as float ids, NaN kept (at rows 5, 50 and 200: on two ranks of every default split)
FLOAT_IDS = {name: 0.5 + k for k, name in enumerate(sorted(set(FRAMES["mixed"]["obs"]["cell_type"].dropna())))}


def case_labels(case, names):
    """Golden label names as the case holds them: the float ids in mixed_float, NaN kept."""
    if not case.endswith("_float"):
        return list(names)
    return [n if pd.isna(n) else FLOAT_IDS[n] for n in names]


def blocks(case, world):
    return BLOCKS[world].get(case) or [shard_rows(Z[f"{case.split('_')[0]}_X"].shape[0], r, world) for r in range(world)]


def annotate_f64(mapping, labels, n_labels, *, sums=True, argmax=False, device=None):
    """utils.annotate in float64 numpy: the per-label sums of the float32 mapping and np.argmax of each labelled row."""
    X = np.asarray(mapping, dtype=np.float32)
    lab = np.asarray(labels).reshape(-1)
    s = np.stack([X[lab == t].astype(np.float64).sum(axis=0) for t in range(n_labels)]) if sums else None
    a = np.where(lab >= 0, X.argmax(axis=1), -1).astype(np.int32) if argmax else None
    return s, a


def sc_expression(N, seed):
    """(N x 24) CSR expression: one all-zero gene, and two gene names that collide once lowercased."""
    rng = np.random.default_rng(seed)
    X = (rng.random((N, 24)) * (rng.random((N, 24)) < 0.3)).astype(np.float32)
    X[:, 5] = 0.0
    genes = [f"G{k}" for k in range(24)]
    genes[3] = "g2"
    return sp.csr_matrix(X), genes


def adatas(case, r0, r1, sharded, dense_sc=False):
    """This rank's AnnDatas for rows [r0, r1) of a golden case: (mapping, spots, adata_sc for the counts, adata_sc for
    project_genes).  `sharded` adds uns["shard_rows"], as map_cells_to_space(process_group=) leaves it."""
    base = case.split("_")[0]
    d, X = FRAMES[base], Z[f"{base}_X"]
    N, V = X.shape
    obs = d["obs"].copy()
    if case.endswith("_cat"):
        labels = obs["cell_type"]
        obs["cell_type"] = pd.Categorical(labels, categories=["zz"] + sorted(set(labels.dropna()))[::-1])
    if case.endswith("_float"):
        obs["cell_type"] = obs["cell_type"].map(FLOAT_IDS)
        assert obs["cell_type"].dtype == np.float64
    uns = {"train_genes_df": pd.DataFrame(index=TRAIN_GENES)}
    if sharded:
        uns["shard_rows"] = (r0, r1)
    ad_map = MiniAnnData(X=X[r0:r1], obs=obs.iloc[r0:r1].copy(), var=d["var"].copy(), uns=uns)
    ad_sp = MiniAnnData(X=np.zeros((V, 1), np.float32), obs=d["var"].copy())
    if "image_features" in d:
        ad_sp.obsm.update(image_features=d["image_features"], spatial=d["spatial"])
        utils.create_segment_cell_df(ad_sp)
    ad_sc = MiniAnnData(X=np.zeros((N, 1), np.float32), obs=obs[["cell_type"]].copy())
    S, genes = sc_expression(N, seed=len(case))
    ad_ge = MiniAnnData(X=S.toarray() if dense_sc else S, obs=pd.DataFrame(index=obs.index),
                        var=pd.DataFrame(index=genes), uns={"overlap_genes": ["g1"]})
    return ad_map, ad_sp, ad_sc, ad_ge


def transfer(case, r0, r1, pg, dense_sc=False):
    """The four calls on rows [r0, r1) of a golden case (with pg=None on the whole mapping) -> their outputs."""
    d = FRAMES[case.split("_")[0]]
    ad_map, ad_sp, ad_sc, ad_ge = adatas(case, r0, r1, pg is not None, dense_sc)
    out = {}
    utils.project_cell_annotations(ad_map, ad_sp, annotation="cell_type", process_group=pg)
    out["pred"] = ad_sp.obsm["tangram_ct_pred"]
    utils.cell_type_mapping(ad_map, cell_types_key="cell_type", process_group=pg)
    out["ct_map"] = ad_map.varm["ct_map"]
    if "image_features" in d:
        for key in [k for k in d if k.startswith("count_")]:
            utils.count_cell_annotations(ad_map, ad_sc, ad_sp, annotation="cell_type", threshold=float(key[6:]),
                                         process_group=pg)
            out[key] = ad_sp.obsm["tangram_ct_count"]
        out["deconv"] = utils.deconvolve_cell_annotations(
            ad_sp, filter_cell_annotation=case_labels(case, d["deconv_filter"])).obs
    ge = utils.project_genes(ad_map, ad_ge, process_group=pg)
    out["ge"] = dict(X=np.asarray(ge.X), obs=ge.obs, var=ge.var, S=ad_ge.X)
    return out


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def init_gloo(rank, world, port):
    """A gloo group whose collectives give up after a minute: a rank left waiting fails the test instead of hanging it."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))


def _calls_worker(rank, world, port, stand_in, out):
    init_gloo(rank, world, port)
    if stand_in:
        utils.annotate = annotate_f64
    got = {}
    for case in CASES:
        r0, r1 = blocks(case, world)[rank]
        got[case] = transfer(case, r0, r1, dist.group.WORLD)
    got["dense_sc"] = transfer("mixed", *blocks("mixed", world)[rank], dist.group.WORLD, dense_sc=True)["ge"]["X"]
    out[rank] = got
    dist.barrier()
    dist.destroy_process_group()


def spawn(worker, world, *args):
    out = mp.Manager().dict()
    mp.spawn(worker, args=(world, free_port(), *args, out), nprocs=world, join=True)
    return [out[r] for r in range(world)]


def close(got, ref, rtol):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape and np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    assert np.all(np.abs(got[ok] - ref[ok]) <= rtol * np.abs(ref[ok])), np.max(np.abs(got[ok] - ref[ok]))


def rel_fro(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def check_ranks_agree(ranks):
    """Every rank's outputs are rank 0's, bit for bit."""
    for r, got in enumerate(ranks[1:], 1):
        for case in CASES:
            for key, v in got[case].items():
                w = ranks[0][case][key]
                if key == "ge":
                    assert np.array_equal(v["X"].view(np.uint32), w["X"].view(np.uint32)), (r, case)
                    pd.testing.assert_frame_equal(v["var"], w["var"])
                    pd.testing.assert_frame_equal(v["obs"], w["obs"])
                else:
                    pd.testing.assert_frame_equal(v, w, check_exact=True, obj=f"rank {r} {case} {key}")


def check_against_golden(case, got, sum_rtol, ct_atol):
    """A rank's annotation outputs against the reference's golden outputs (the counts and deconvolved cells exactly)."""
    base = case.split("_")[0]
    d = FRAMES[base]
    close(got["pred"].to_numpy(), Z[f"{base}_pred"], sum_rtol)
    columns = pd.Index(case_labels(case, d["pred"].columns))
    assert got["pred"].index.equals(d["pred"].index) and got["pred"].columns.equals(columns), case
    assert all(got["pred"].dtypes == np.float64)
    if "ct_map" in d:
        g, r = got["ct_map"].to_numpy(), d["ct_map"].to_numpy()
        assert got["ct_map"].columns.equals(columns)
        assert np.array_equal(np.isnan(g), np.isnan(r)) and np.nanmax(np.abs(g - r)) <= ct_atol, case
    for key in [k for k in d if k.startswith("count_")]:
        ref = d[key].set_axis(list(d[key].columns[:4]) + case_labels(case, d[key].columns[4:]), axis=1)
        pd.testing.assert_frame_equal(got[key], ref, obj=f"{case} {key}")
    if "deconv_obs" in d:
        ref = d["deconv_obs"].assign(cluster=case_labels(case, d["deconv_obs"]["cluster"]))
        pd.testing.assert_frame_equal(got["deconv"], ref, obj=f"{case} deconvolved cells")


def check_genes(got, want, rtol):
    """project_genes on the shards against the call on the whole mapping (and float64), columns and rows included."""
    pd.testing.assert_frame_equal(got["var"], want["var"])
    pd.testing.assert_frame_equal(got["obs"], want["obs"])
    assert list(got["var"].index) == [f"g{k}" if k != 3 else "g2-1" for k in range(24) if k != 5]
    assert got["var"]["is_training"].sum() == 3
    assert rel_fro(got["X"], want["X"]) <= rtol


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_transfer_equals_the_whole_mapping(world, monkeypatch):
    monkeypatch.setattr(utils, "annotate", annotate_f64)
    want = {case: transfer(case, 0, Z[f"{case.split('_')[0]}_X"].shape[0], None) for case in CASES}
    ranks = spawn(_calls_worker, world, True)
    check_ranks_agree(ranks)
    for case in CASES:
        base = case.split("_")[0]
        got, w = ranks[0][case], want[case]
        check_against_golden(case, got, 1e-12, 1e-10)
        check_against_golden(case, w, 1e-12, 1e-10)
        close(got["pred"].to_numpy(), w["pred"].to_numpy(), 1e-13)
        assert got["pred"].columns.equals(w["pred"].columns) and got["pred"].columns.dtype == w["pred"].columns.dtype
        assert got["ct_map"].columns.equals(w["ct_map"].columns)
        g, r = got["ct_map"].to_numpy(), w["ct_map"].to_numpy()
        assert np.array_equal(np.isnan(g), np.isnan(r)) and np.nanmax(np.abs(g - r)) <= 1e-12
        check_genes(got["ge"], w["ge"], 1e-6)
        S = w["ge"]["S"].toarray().astype(np.float64)[:, [k for k in range(24) if k != 5]]
        assert rel_fro(got["ge"]["X"], Z[f"{base}_X"].astype(np.float64).T @ S) <= 1e-6
    assert rel_fro(ranks[0]["dense_sc"], ranks[0]["mixed"]["ge"]["X"]) <= 1e-6
    # the awkward labels are where the docstring says, and land in the reference's columns
    lab = FRAMES["mixed"]["obs"]["cell_type"].to_numpy()
    firsts = [list(pd.unique(pd.Series(lab[r0:r1]))) for r0, r1 in blocks("mixed", world)]
    assert "B" not in firsts[0] and "solo" not in firsts[0] and sum("solo" in f for f in firsts) == 1
    assert [k for k, f in enumerate(firsts) if any(pd.isna(x) for x in f)] == ([1] if world == 2 else [0, 2])
    assert world == 2 or firsts[1] == []
    flt = [list(pd.unique(pd.Series(lab[r0:r1]).map(FLOAT_IDS))) for r0, r1 in blocks("mixed_float", world)]
    assert sum(any(pd.isna(x) for x in f) for f in flt) == 2
    for case in ("mixed", "mixed_cat", "mixed_float"):
        assert sum(pd.isna(c) for c in ranks[0][case]["pred"].columns) == 1


REFUSALS = ["missing", "overlap", "short", "obs", "cluster_label"]


def _refusals_worker(rank, world, port, out):
    init_gloo(rank, world, port)
    utils.annotate = annotate_f64
    pg = dist.group.WORLD
    N = Z["mixed_X"].shape[0]
    got = {}

    def attempt(name, call, ad_sp=None):
        try:
            call()
            got[name] = None
        except ValueError as e:
            got[name] = str(e)
        if ad_sp is not None:
            got[name + " wrote"] = "tangram_ct_pred" in ad_sp.obsm or "tangram_ct_count" in ad_sp.obsm

    for what in REFUSALS:
        if what == "overlap":
            r0, r1 = [(0, 160), (150, N)][rank]
        elif what == "short":
            r0, r1 = [(0, 100), (100, 200)][rank]
        else:
            r0, r1 = shard_rows(N, rank, world)
        ad_map, ad_sp, ad_sc, ad_ge = adatas("mixed", r0, r1, True)
        if what == "missing" and rank == 1:
            del ad_map.uns["shard_rows"]
        if what == "obs" and rank == 1:
            ad_map.obs.index = ad_map.obs.index[::-1]
        kw = dict(cluster_label="cell_type") if what == "cluster_label" and rank == 1 else {}
        attempt(f"{what} project_genes", lambda: utils.project_genes(ad_map, ad_ge, process_group=pg, **kw))
        if what in ("missing", "overlap"):
            attempt(f"{what} project_cell_annotations",
                    lambda: utils.project_cell_annotations(ad_map, ad_sp, process_group=pg), ad_sp)
            attempt(f"{what} cell_type_mapping",
                    lambda: utils.cell_type_mapping(ad_map, cell_types_key="cell_type", process_group=pg))
            attempt(f"{what} count_cell_annotations",
                    lambda: utils.count_cell_annotations(ad_map, ad_sc, ad_sp, process_group=pg), ad_sp)
            got[f"{what} cell_type_mapping wrote"] = "ct_map" in ad_map.varm
    # after every refusal the group still works
    ad_map, ad_sp, _, _ = adatas("mixed", *shard_rows(N, rank, world), True)
    utils.project_cell_annotations(ad_map, ad_sp, process_group=pg)
    got["after"] = ad_sp.obsm["tangram_ct_pred"]
    out[rank] = got
    dist.barrier()
    dist.destroy_process_group()


def test_refusals_raise_on_every_rank():
    ranks = spawn(_refusals_worker, 2)
    expect = {"missing": r"rank\(s\) \[1\] passed a mapping without uns\['shard_rows'\]",
              "overlap": r"do not tile the cells in rank order",
              "short": r"cover 200 cells of the 301 in adata_sc",
              "obs": r"^rank 1: its mapping's obs index is not rows \[151, 301\) of adata_sc\.obs\.index$",
              "cluster_label": r"^rank 1: cluster_label projects a clusters-mode mapping"}
    for got in ranks:
        for name, msg in got.items():
            what = name.split()[0]
            if name.endswith(" wrote"):
                assert msg is False, f"{name} its output before refusing"
            elif name != "after":
                assert msg is not None, f"{name} was not refused"
                assert re.search(expect[what], msg), (name, msg)
        assert set(n.split()[0] for n in got if n != "after") == set(REFUSALS)
    for name in ranks[0]:
        if name != "after":
            assert ranks[0][name] == ranks[1][name], f"{name}: the ranks refused differently"
    close(ranks[0]["after"].to_numpy(), Z["mixed_pred"], 1e-12)
    pd.testing.assert_frame_equal(ranks[1]["after"], ranks[0]["after"], check_exact=True)
