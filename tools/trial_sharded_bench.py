"""The tuner's trial, unsharded on one GPU and sharded over the visible GPUs: wall time of train_multiple_Mapper and its
parts (train_s, project_s with the gene cube's all-reduce, score_s with the agreement's all-reduces), per rank, on
synthetic inputs drawn from a seed.  The unsharded leg runs only where the trial fits on one GPU.  Both legs run the same
configuration from the same generator state, and the report says whether their metrics agree within the trial test's
tolerance (1e-4).  Prints one JSON object; with --out also writes it there.

    python tools/trial_sharded_bench.py [--cells 40000] [--spots 8000] [--genes 1000] [--val 200] [--epochs 100]
                                        [--runs 3] [--world <visible GPUs>] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.tangram_oracle import synthetic_inputs  # noqa: E402
from tangram_b200 import _lib  # noqa: E402
from tangram_b200 import mapping_parameter_tuning as mpt  # noqa: E402

METRICS = ["cell_map_consistency", "cell_map_agreement", "cell_map_certainty", "gene_expr_consistency",
           "gene_expr_correctness"]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return q or torch.cuda.get_device_name(0)


def trial(a, device, process_group=None):
    """One train_multiple_Mapper call on the seeded inputs -> (metrics, parts and wall seconds)."""
    inp = synthetic_inputs(a.cells, a.spots, a.genes, seed=1)
    data = [inp["S"], inp["G"], None, inp["d"], device, None, None, None, None, None,
            list(range(a.genes - a.val)), list(range(a.genes - a.val, a.genes))]
    config = {"num_epochs": a.epochs, "lambda_d": 1.0, "lambda_g2": 0.3, "learning_rate": 0.1}
    np.random.seed(5)
    det = {}
    torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    m = mpt.train_multiple_Mapper(config, data, n_runs=a.runs, details=det, process_group=process_group)
    torch.cuda.synchronize(device)
    wall = time.perf_counter() - t0
    t = {k: round(det[k], 4) for k in ("train_s", "project_s", "score_s")}
    t["wall_s"] = round(wall, 4)
    if "shard_rows" in det:
        t["shard_rows"] = list(det["shard_rows"])
    return m, t


def worker(a):
    """One rank of the sharded leg (under torch.distributed.run)."""
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", device_id=torch.device(f"cuda:{rank}"))
    m, t = trial(a, f"cuda:{rank}", dist.group.WORLD)
    got = [None] * world
    dist.all_gather_object(got, t)
    if rank == 0:
        with open(a.worker_out, "w") as f:
            json.dump({"metrics": m, "ranks": got}, f)
    dist.barrier()
    dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=40000)
    ap.add_argument("--spots", type=int, default=8000)
    ap.add_argument("--genes", type=int, default=1000)
    ap.add_argument("--val", type=int, default=200)
    ap.add_argument("--epochs", type=int, default=100)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--world", type=int, default=0, help="ranks of the sharded leg (default: every visible GPU)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker-out", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker_out:
        worker(a)
        return
    world = a.world or torch.cuda.device_count()
    res = {"card": card(), "gpus": torch.cuda.device_count(), "world": world,
           "shape": {"cells": a.cells, "spots": a.spots, "genes": a.genes, "val_genes": a.val, "epochs": a.epochs,
                     "runs": a.runs}}
    unsharded = None
    try:
        unsharded, res["unsharded"] = trial(a, "cuda:0")
    except _lib.TangramB200Error as e:
        res["unsharded"] = f"does not fit on one GPU: {e}"
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "sharded.json")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
               "--master-addr", "127.0.0.1", "--master-port", "29561", os.path.abspath(__file__), "--worker-out", out]
        cmd += [f"--{k}={getattr(a, k)}" for k in ("cells", "spots", "genes", "val", "epochs", "runs")]
        t0 = time.perf_counter()
        p = subprocess.run(cmd, capture_output=True, text=True)
        launch = time.perf_counter() - t0
        if p.returncode != 0:
            raise SystemExit(f"sharded leg failed:\n{p.stdout[-3000:]}\n{p.stderr[-3000:]}")
        with open(out) as f:
            sharded = json.load(f)
    res["sharded"] = {"ranks": sharded["ranks"], "launch_wall_s": round(launch, 2),
                      "slowest_rank_wall_s": max(r["wall_s"] for r in sharded["ranks"])}
    res["metrics_sharded"] = sharded["metrics"]
    if unsharded is not None:
        res["metrics_unsharded"] = unsharded
        res["max_metric_difference"] = max(abs(unsharded[k] - sharded["metrics"][k]) for k in METRICS)
        res["metrics_agree_within_1e-4"] = res["max_metric_difference"] < 1e-4
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
