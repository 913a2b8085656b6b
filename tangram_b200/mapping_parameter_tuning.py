"""
The hyper-parameter tuner's trial (Tangram's tangram/mapping_parameter_tuning.py:42-139) on the sm_90a (H100) library:
the three run-to-run metrics and `train_multiple_Mapper`, which trains one configuration several times and scores how
well the runs agree.

    pearson_corr(cube)        (R(R-1)/2,) pairwise Pearson correlations of the flattened runs, np.tril_indices order
    vote_entropy(cube)        (N,) normalised entropy of the runs' argmax votes per row
    consensus_entropy(cube)   (N,) normalised entropy of the mean over runs per row

`cube` is an (R, N, V) numpy array or CUDA tensor (or a sequence of R (N, V) ones); all three run on the device in one
streaming pass each (tgb200_agreement), with no N x V scratch and no float64 copy of the cube.  There is no CPU path.

    metrics = train_multiple_Mapper(config, data)     # the five numbers the reference reports to ray.train.report

makes a Ray trainable a one-line wrapper.  The Ray / Optuna driver `mapping_hyperparameter_tuning` itself stays with the
reference.  With `process_group=` (NCCL, one process per GPU) the trial shards the cells of every run over the group, and
`agreement(..., process_group=)` scores a cube whose rows are spread over the ranks.
"""
import ctypes

import numpy as np

from . import _lib
from .engine import _require_device
from .mapping_optimizer import Mapper
from .sharded import shard_rows

_CONFIG_LAMBDAS = ["lambda_d", "lambda_g1", "lambda_g2", "lambda_neighborhood_g1", "lambda_r", "lambda_l1",
                   "lambda_l2", "lambda_ct_islands", "lambda_getis_ord"]     # :97
# device bytes per mapping element one Mapper handle holds at most (M, m, v, operands, a projection's P planes)
_HANDLE_BYTES_PER_ELEMENT = 28


def _runs_on_device(cube, device):
    """(R, N, V) ndarray / CUDA tensor / sequence of (N, V) -> (list of R CUDA tensors with unit column stride and equal
    row stride, device ordinal).  Host data is copied to the device once, as float32."""
    import torch
    if isinstance(cube, torch.Tensor) and cube.is_cuda:
        dev = cube.device.index
        runs = list(cube.unbind(0)) if cube.dim() == 3 else None
    elif isinstance(cube, (list, tuple)) and cube and all(isinstance(c, torch.Tensor) and c.is_cuda for c in cube):
        dev = cube[0].device.index
        runs = list(cube)
    else:
        dev = _require_device("cuda" if device is None else device)
        arr = np.asarray(cube if not isinstance(cube, (list, tuple)) else np.stack([np.asarray(c) for c in cube]))
        if arr.ndim != 3:
            raise ValueError(f"expected an (R, N, V) cube, got shape {arr.shape}")
        runs = list(torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float32)).to(f"cuda:{dev}").unbind(0))
    if runs is None or any(r.dim() != 2 for r in runs):
        raise ValueError("expected an (R, N, V) cube or a sequence of R (N, V) arrays")
    shape = tuple(runs[0].shape)
    out = []
    for r in runs:
        if tuple(r.shape) != shape or r.device.index != dev:
            raise ValueError("all runs must have the same shape and device")
        r = r.float()
        if r.stride(1) != 1 or (shape[0] > 1 and r.stride(0) != runs[0].stride(0)) or r.stride(0) < shape[1]:
            r = r.contiguous()
        out.append(r)
    if len({r.stride(0) for r in out}) > 1:
        out = [r.contiguous() for r in out]
    return out, dev


def agreement(cube, *, pearson=True, vote=False, consensus=False, device=None, process_group=None):
    """One pass of tgb200_agreement over the R runs of `cube`: -> (pearson (R(R-1)/2,) float64 or None,
    vote entropy (N,) float32 or None, consensus entropy (N,) float32 or None).  `device` places host data (default:
    the current CUDA device); device data is read where it lives.

    process_group: `cube` holds this rank's rows of a cube whose rows are spread over the group's ranks (the same R and
    V everywhere, any number of rows each).  A collective: the ranks' shift samples and Pearson sums are summed over the
    group (tgb200_agreement_sample / _partials / _pearson), so every rank gets the same Pearson values, those of the
    whole cube; the entropies are this rank's rows.  With one rank the result is tgb200_agreement's, bit for bit."""
    import torch
    runs, dev = _runs_on_device(cube, device)
    R = len(runs)
    rows, cols = runs[0].shape
    lib = _lib.load()
    ptrs = (_lib._P * R)(*[r.data_ptr() for r in runs])
    p = np.empty(R * (R - 1) // 2, dtype=np.float64) if pearson else None
    v = np.empty(rows, dtype=np.float32) if vote else None
    c = np.empty(rows, dtype=np.float32) if consensus else None
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    if process_group is None:
        _lib.check(lib.tgb200_agreement(ptrs, R, rows, cols, runs[0].stride(0), _lib.ptr(p), _lib.ptr(v),
                                        _lib.ptr(c), dev, stream))
        return p, v, c
    import torch.distributed as dist
    ld = runs[0].stride(0)

    def all_reduce(t):
        """in-place sum over the group: on the device for NCCL, on the host for other backends"""
        if dist.get_backend(process_group) == "nccl":
            dist.all_reduce(t, group=process_group)
            return t
        h = t.cpu()
        dist.all_reduce(h, group=process_group)
        return h.to(t.device)

    f64 = dict(dtype=torch.float64, device=f"cuda:{dev}")
    # [R sample sums, sample size, rows]: the shared shift and the global row count from one all-reduce
    sample = torch.empty(R + 2, **f64)
    _lib.check(lib.tgb200_agreement_sample(ptrs, R, rows, cols, ld, _lib.ptr(sample), dev, stream))
    sample[R + 1] = rows
    sample = all_reduce(sample).cpu().numpy()
    shift = sample[:R] / sample[R]        # what k_agreement_shift divides on the device: the same bits for one rank
    rows_global = int(sample[R + 1])
    sums = torch.empty(R + R * (R + 1) // 2, **f64)
    _lib.check(lib.tgb200_agreement_partials(ptrs, R, rows, cols, ld, _lib.ptr(shift), _lib.ptr(sums), _lib.ptr(v),
                                             _lib.ptr(c), dev, stream))
    sums = all_reduce(sums)
    if pearson:
        _lib.check(lib.tgb200_agreement_pearson(_lib.ptr(sums), R, rows_global, cols, _lib.ptr(p), dev, stream))
    return p, v, c


def pearson_corr(cube, *, device=None):
    """:42-53 -- all pairwise Pearson correlations of the R flattened runs, (R(R-1)/2,) float64 in np.tril_indices(R, -1)
    order, as np.corrcoef computes them (fp64 sums)."""
    return agreement(cube, device=device)[0]


def vote_entropy(pred_probs_cube, *, device=None):
    """:55-69 -- per row, the entropy of the runs' argmax votes normalised by log(V): (N,).  The votes are np.argmax's:
    the first column on ties, a NaN counting as the maximum (the first NaN wins), column 0 for an all -inf row.  NaN on
    every row when V == 1, as the reference's division by log(1) = 0 gives."""
    return agreement(pred_probs_cube, pearson=False, vote=True, device=device)[1]


def consensus_entropy(pred_probs_cube, *, device=None):
    """:71-82 -- per row, the entropy of the mean over runs (renormalised, 0 log 0 = 0) normalised by log(V): (N,).
    NaN for a row whose mean holds a NaN or an infinity or sums to 0, and on every row when V == 1."""
    return agreement(pred_probs_cube, pearson=False, consensus=True, device=device)[2]


def train_multiple_Mapper(config, data, *, n_runs=3, precision="bf16x3", details=None, process_group=None):
    """:86-139 -- train the configuration `config` n_runs times (random_state = 0, 1, 2, ...) on `data`, the reference's
    12-entry list [S, G, d_source, d, device, print_each, voxel_weights, ct_encode, neighborhood_filter, spatial_weights,
    train_genes_idx, val_genes_idx], and return the five metrics the reference reports:
        cell_map_consistency   mean pairwise Pearson correlation of the mappings
        cell_map_agreement     1 - mean vote entropy of the mappings
        cell_map_certainty     1 - mean consensus entropy of the mappings
        gene_expr_consistency  mean pairwise Pearson correlation of the projected validation genes
        gene_expr_correctness  mean over runs of the final validation gene score (val_gene_sim after the last update)
    As in the reference, run 0 is unseeded (random_state=0 is falsy, mapping_optimizer.py:148) and continues numpy's
    global generator.  The mappings stay on the device (an R x N x V cube), the validation genes are projected there,
    and each run's handle is released before the next starts.  `details`, if a dict, receives the device cubes
    ("cell_cube" R x N x V, "gene_cube" R x V x n_val), the per-run "val_gene_sim" and the seconds spent in "train_s",
    "project_s" and "score_s".

    process_group: a torch.distributed NCCL group, one process per GPU, shards the cells as Mapper(process_group=) does.
    Every rank passes the same `data` with its own device in data[4], and every rank must enter with the same state of
    numpy's global generator (run 0 draws from it; nothing broadcasts it): each rank then leaves it where the unsharded
    trial leaves it.  Each rank holds an R x N_r x V cube of its rows shard_rows(N, rank, world) (the memory check
    counts those rows only); the validation genes projected from a rank's rows are summed over the group, so every rank
    holds the whole gene cube; the cell metrics come from agreement(process_group=) and from the entropies summed over
    the group.  Every rank returns the same five metrics.  `details` also receives "shard_rows" (r0, r1), and
    "cell_cube" is the rank's own rows.  A non-NCCL group and n_runs > 8 are refused before any training."""
    import time

    import torch
    (S, G, d_source, d, device, print_each, voxel_weights, ct_encode, neighborhood_filter, spatial_weights,
     train_genes_idx, val_genes_idx) = data
    if process_group is not None:
        import torch.distributed as dist
        if n_runs > 8:
            raise ValueError(f"a sharded trial scores at most 8 runs (the agreement pass takes 1..8), got n_runs={n_runs}")
        if dist.get_backend(process_group) != "nccl":
            raise ValueError("a sharded trial needs an NCCL process group: each run's final validation of the sharded "
                             "mapping sums its forward on the group's NCCL communicator, which a non-NCCL group lacks")
    dev = _require_device(device)
    hyperparameters = {"d_source": d_source}
    for param in _CONFIG_LAMBDAS:
        if param in config:
            hyperparameters[param] = config[param]
    learning_rate = config.get("learning_rate", 0.1)
    num_epochs = config.get("num_epochs", 1000)

    S = np.asarray(S, dtype=np.float32)
    N, V = S.shape[0], np.shape(G)[0]
    r0, r1 = (0, N) if process_group is None else shard_rows(N, dist.get_rank(process_group),
                                                                 dist.get_world_size(process_group))
    N_r = r1 - r0
    S_val = np.ascontiguousarray(S[r0:r1, val_genes_idx] if val_genes_idx is not None else S[r0:r1])
    n_val = S_val.shape[1]
    k_train = len(train_genes_idx) if train_genes_idx is not None else S.shape[1]
    cube_bytes = 4 * n_runs * N_r * V + 4 * n_runs * V * n_val
    handle_bytes = _HANDLE_BYTES_PER_ELEMENT * N_r * V + 16 * (N_r + V) * (k_train + n_val)
    free, _ = torch.cuda.mem_get_info(dev)
    if cube_bytes + handle_bytes > free:
        raise _lib.TangramB200Error(
            f"train_multiple_Mapper needs about {(cube_bytes + handle_bytes) / 2**30:.1f} GiB on cuda:{dev} "
            f"({n_runs} mappings of {N_r} x {V} = {cube_bytes / 2**30:.1f} GiB, plus one mapper of "
            f"{handle_bytes / 2**30:.1f} GiB); {free / 2**30:.1f} GiB are free")

    sharding = {} if process_group is None else dict(process_group=process_group, draw_whole_stream=True)
    t_train = t_proj = 0.0
    cell_cube = torch.empty((n_runs, N_r, V), dtype=torch.float32, device=f"cuda:{dev}")
    gene_cube = torch.empty((n_runs, V, n_val), dtype=torch.float32, device=f"cuda:{dev}")   # (S_val^T P)^T
    val_gene_scores = []
    for run in range(n_runs):
        t0 = time.perf_counter()
        mapper = Mapper(S=S, G=G, d=d, train_genes_idx=train_genes_idx, val_genes_idx=val_genes_idx,
                        voxel_weights=voxel_weights, neighborhood_filter=neighborhood_filter, ct_encode=ct_encode,
                        spatial_weights=spatial_weights, device=f"cuda:{dev}", random_state=run, precision=precision,
                        **hyperparameters, **sharding)
        try:
            # the reference validates after every update (val_each=1) and keeps only the last score: one evaluation
            # after the final update is the same number (sharded: a collective over the group)
            mapper.train(num_epochs, learning_rate=learning_rate, print_each=print_each, out=cell_cube[run])
            val_gene_scores.append(mapper.validation_terms()["val_gene_sim"])
            t1 = time.perf_counter()
            # :134 -- S[:, val]^T @ mapping, stored transposed: Pearson over flattened runs does not see the order
            mapper.project(S_val, out=gene_cube[run])
            if process_group is not None:
                dist.all_reduce(gene_cube[run], group=process_group)     # the projection of every cell
                torch.cuda.current_stream(dev).synchronize()
            t2 = time.perf_counter()
        finally:
            mapper.release()
        t_train += t1 - t0
        t_proj += t2 - t1

    t0 = time.perf_counter()
    cell_p, cell_v, cell_c = agreement(cell_cube, vote=True, consensus=True, process_group=process_group)
    gene_p = agreement(gene_cube)[0]
    if process_group is None:
        vote_mean, cons_mean = cell_v.astype(np.float64).mean(), cell_c.astype(np.float64).mean()
    else:
        # sum over every rank's rows / n_cells_global: with one rank, the operation .mean() performs
        sums = torch.tensor([cell_v.astype(np.float64).sum(), cell_c.astype(np.float64).sum()], dtype=torch.float64,
                            device=f"cuda:{dev}")
        dist.all_reduce(sums, group=process_group)
        vote_mean, cons_mean = sums.cpu().numpy() / N
    t_score = time.perf_counter() - t0
    if isinstance(details, dict):
        details.update(cell_cube=cell_cube, gene_cube=gene_cube, val_gene_sim=val_gene_scores, train_s=t_train,
                       project_s=t_proj, score_s=t_score)
        if process_group is not None:
            details["shard_rows"] = (r0, r1)
    return {"cell_map_consistency": float(cell_p.mean()),
            "cell_map_agreement": float(1 - vote_mean),
            "cell_map_certainty": float(1 - cons_mean),
            "gene_expr_consistency": float(gene_p.mean()),
            "gene_expr_correctness": float(np.mean(val_gene_scores))}
