"""Gene projection and annotation transfer after a cell-sharded mapping on two GPUs (NCCL), launched as a torchrun
subprocess like tests/test_sharded_validation_multigpu.py; skipped with fewer than two devices.

map_cells_to_space(process_group=) maps 3001 cells onto 700 spots in cells and in constrained mode; then every rank calls
project_genes, project_cell_annotations, cell_type_mapping and count_cell_annotations (and deconvolve_cell_annotations)
on its shard.  The reference is the same calls without a group on the mapping that map_cells_to_space(gather=True)
returns, whose rows must be the shards' bit for bit.  Bounds: the fp64 sums within 1e-12 relative (the min-max
normalised ct_map within 1e-12), counts and deconvolved cells exact, project_genes within 1e-6 (relative Frobenius).
The results are identical on both ranks.
"""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKER = r'''
import hashlib, os, sys, numpy as np, pandas as pd, torch, torch.distributed as dist
sys.path.insert(0, os.environ["TGB_ROOT"])
from oracle.tangram_oracle import synthetic_inputs
import tangram_b200 as tg
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(rank)
dev = f"cuda:{rank}"
dist.init_process_group("nccl", device_id=torch.device(dev))
pg = dist.group.WORLD

N, V, K = 3001, 700, 120
inp = synthetic_inputs(N, V, K, seed=5)
genes = [f"g{i}" for i in range(K)]
spots = [f"v{i}" for i in range(V)]
rng = np.random.default_rng(3)
labels = np.array(["A", "B", "C", "D", "E", np.nan], dtype=object)[rng.integers(0, 6, N)]
labels[:40] = "A"                          # B..E and NaN are first seen later; "late" only on the last rank
labels[N - 5] = "late"
n_seg = rng.integers(0, 4, V)
n_seg[0] = 2
features = pd.DataFrame({"segmentation_label": n_seg,
                         "segmentation_centroid": [[(float(rng.random()), float(rng.random())) for _ in range(k)]
                                                   for k in n_seg]}, index=spots)
spatial = rng.random((V, 2))


def adatas():
    ad_sc = tg.MiniAnnData(X=inp["S"].copy(), obs=pd.DataFrame({"cell_type": labels}, index=[f"c{i}" for i in range(N)]),
                           var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=inp["G"].copy(), obs=pd.DataFrame(index=spots), var=pd.DataFrame(index=genes))
    tg.pp_adatas(ad_sc, ad_sp)
    return ad_sc, ad_sp


def calls(ad_map, ad_sc, group):
    ad_sp = tg.MiniAnnData(X=np.zeros((V, 1), np.float32), obs=pd.DataFrame(index=spots),
                           obsm={"image_features": features, "spatial": spatial})
    tg.create_segment_cell_df(ad_sp)
    out = {}
    tg.project_cell_annotations(ad_map, ad_sp, annotation="cell_type", process_group=group)
    out["pred"] = ad_sp.obsm["tangram_ct_pred"]
    tg.cell_type_mapping(ad_map, cell_types_key="cell_type", process_group=group)
    out["ct_map"] = ad_map.varm["ct_map"]
    for thr in (0.5, 0.3):
        tg.count_cell_annotations(ad_map, ad_sc, ad_sp, annotation="cell_type", threshold=thr, process_group=group)
        out[f"count_{thr}"] = ad_sp.obsm["tangram_ct_count"]
    out["deconv"] = tg.deconvolve_cell_annotations(ad_sp).obs
    out["ge"] = np.asarray(tg.project_genes(ad_map, ad_sc, process_group=group).X)
    return out


def digest(out):
    h = hashlib.sha256()
    for k in sorted(out):
        v = out[k]
        if isinstance(v, pd.DataFrame):
            h.update(v.to_csv().encode())
            num = v.select_dtypes("number")
            h.update(num.to_numpy(np.float64).tobytes() + repr(list(num.columns)).encode())
        else:
            h.update(v.tobytes())
    return h.hexdigest()


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(np.asarray(b, np.float64)))


for mode, extra in (("cells", {}), ("constrained", dict(target_count=N // 3, lambda_f_reg=1, lambda_count=1))):
    ad_sc, ad_sp = adatas()
    kw = dict(mode=mode, device=dev, num_epochs=20, random_state=7, verbose=False, precision="fp32", process_group=pg,
              **extra)
    part = tg.map_cells_to_space(ad_sc, ad_sp, **kw)
    full = tg.map_cells_to_space(ad_sc, ad_sp, gather=True, **kw)
    r0, r1 = part.uns["shard_rows"]
    shards = [None] * world
    dist.all_gather_object(shards, (r0, r1, np.asarray(part.X),
                                    np.asarray(part.obs["F_out"]) if mode == "constrained" else None))
    got = calls(part, ad_sc, pg)
    digests = [None] * world
    dist.all_gather_object(digests, digest(got))
    assert all(d == digests[0] for d in digests), f"{mode}: the ranks' results differ"
    assert sorted(got["pred"].columns, key=str) == sorted(pd.unique(pd.Series(labels)), key=str)
    if rank == 0:
        for a0, a1, X, F in shards:
            assert np.array_equal(np.asarray(full.X)[a0:a1].view(np.uint32), X.view(np.uint32)), (mode, a0, a1)
            if F is not None:
                assert np.array_equal(np.asarray(full.obs["F_out"])[a0:a1], F), (mode, a0, a1)
        want = calls(full, ad_sc, None)
        for key in ("pred", "ct_map"):
            g, w = got[key], want[key]
            assert g.columns.equals(w.columns) and g.index.equals(w.index), (mode, key)
            g, w = g.to_numpy(), w.to_numpy()
            assert np.array_equal(np.isnan(g), np.isnan(w)), (mode, key)
            ok = ~np.isnan(w)
            err = np.abs(g[ok] - w[ok])
            bound = 1e-12 * (np.abs(w[ok]) if key == "pred" else 1.0)
            assert np.all(err <= bound), (mode, key, float(err.max()))
        for key in ("count_0.5", "count_0.3", "deconv"):
            pd.testing.assert_frame_equal(got[key], want[key], obj=f"{mode} {key}")
        e = rel(got["ge"], want["ge"])
        assert e <= 1e-6, (mode, e)
        print(f"{mode}: {len(got['pred'].columns)} labels, {int(got['count_0.5'].iloc[:, 4:].to_numpy().sum())} cells "
              f"counted, project_genes rel-Frobenius {e:.2e} against the gathered mapping", flush=True)
dist.barrier()
dist.destroy_process_group()
print("SHARDED TRANSFER OK", flush=True)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_sharded_transfer_equals_the_gathered_mapping(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER)
    env = dict(os.environ, TGB_ROOT=ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29547", str(script)]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=1200)
    print(res.stdout[-4000:], res.stderr[-4000:])
    assert res.returncode == 0 and res.stdout.count("SHARDED TRANSFER OK") == 2
