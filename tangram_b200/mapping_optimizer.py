"""
Drop-in replacement for the reference optimizer class `Mapper`
(Tangram's tangram/mapping_optimizer.py:14-408), running on the sm_90a (H100) C-ABI
library (include/tangram_b200.h) through `tangram_b200.engine.Engine`.  Same constructor keywords,
same `train()` signature, same return types and history conventions.  There is no CPU path: `device` must be a
CUDA device with compute capability 9.0.

Additions (keyword-only, all optional):
  precision   "bf16x3" (default: parity-grade fp32 results on wgmma tensor cores -- every operand is split into three
              bf16 planes and the six significant partial products are accumulated in fp32) |
              "fp32" (FFMA contractions, the cross-check) | "bf16" (plain bf16 operands: throughput mode)
  M0          explicit initial mapping (ndarray N x V); default is the reference draw, made on the device bit for bit
              (legacy_rng), leaving numpy's global generator where the host draw leaves it
  process_group / shard  cell-sharded multi-GPU operation (one process per GPU): every rank passes the
              full S (/ M0) and keeps rows shard_rows(N, rank, world); with a NCCL process group the handle gets its own
              NCCL communicator (tgb200_comm_init_rank) and the per-iteration exchange runs inside tgb200_run;
              MapperConstrained takes both with the same meaning (full S, M0 and F0 on every rank)
  n_cells_global         pre-sharded variant (Mapper only): S, M0, d_source, ct_encode already hold only this rank's rows
  train(..., resume=True)  continue with the Adam state of the previous train() call (the reference -- and the default
              here -- builds a fresh optimizer in every train() call, mapping_optimizer.py:373)
  train(..., out=tensor)   write softmax(M) into a CUDA tensor instead of returning a host array
  validation_terms(), project(X, out=None), state() / load_state(...)
"""
import numpy as np

from . import _lib, legacy_rng
from .engine import Engine, _device_index
from .sharded import shard_rows, sharded_steps

_HIST_KEYS = ["total_loss", "main_loss", "vg_reg", "kl_reg", "entropy_reg"]
_VAL_KEYS = ["val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy"]
# (history column, printed name) in the reference's print order (mapping_optimizer.py:273-298)
_PRINT_TERMS = [
    (1, "Gene-voxel score"), (2, "Voxel-gene score"), (3, "Cell densities reg"), (4, "Entropy reg"),
    (5, "L1 reg"), (6, "L2 reg"), (7, "Spatial weighted score"), (8, "Cell type islands penalty"),
    (9, "Getis-Ord score"),
]


class _ResultBuffer:
    """Where softmax(M) lands (mapping_optimizer.py:406-408).  A fresh 4 GB numpy array is a million page faults and a
    staged pageable copy (~0.7 s at 100k x 10k); so for large results a host thread faults the pages in and page-locks
    them WHILE the iterations run (tgb200_host_pin), and the final device->host copy is one DMA at link speed.  Results
    under 1 GB (where faulting + registering costs more than the staged copy it saves, and where many ranks of one node would
    all be registering at once), or a failed registration (locked-memory limit), simply use the pageable path."""
    MIN_BYTES = 1 << 30

    def __init__(self, lib, shape, device):
        self.arr = np.empty(shape, dtype=np.float32)
        self._lib, self._pinned, self._thread = lib, False, None
        if self.arr.nbytes >= self.MIN_BYTES:
            import threading
            self._thread = threading.Thread(target=self._pin, args=(int(device),), daemon=True)
            self._thread.start()

    def _pin(self, device):
        import os
        threads = max(1, min(8, (os.cpu_count() or 2) // 2))
        self._pinned = self._lib.tgb200_host_pin(_lib.ptr(self.arr), self.arr.nbytes, threads, device) == 0

    def ready(self):
        if self._thread is not None:
            self._thread.join()
            self._thread = None
        return self.arr

    def release(self):
        self.ready()
        if self._pinned:
            self._lib.tgb200_host_unpin(_lib.ptr(self.arr))
            self._pinned = False


def legacy_normal_rows(random_state, n_rows, n_cols, r0, r1, block_rows=4096):
    """Rows [r0, r1) of the reference's initial draw `np.random.normal(0, 1, (n_rows, n_cols))` (mapping_optimizer.py:
    148-150: legacy MT19937, seeded only if `random_state` is truthy) WITHOUT materialising the other rows: the legacy
    generator has no skip-ahead (polar Box-Muller with rejection), so the stream is consumed block by block and only this
    rank's rows are kept -- same bits as the full draw, O(block) extra memory instead of 8 bytes x n_rows x n_cols."""
    if random_state:
        np.random.seed(seed=random_state)
    out = np.empty((r1 - r0, n_cols), dtype=np.float32)
    for b0 in range(0, r1, block_rows):          # rows past r1 are never needed: stop there
        b1 = min(b0 + block_rows, r1)
        blk = np.random.normal(0, 1, (b1 - b0, n_cols))
        lo, hi = max(b0, r0), b1
        if hi > lo:
            out[lo - r0:hi - r0] = blk[lo - b0:hi - b0]
    return out


def discard_normal_rows(n_rows, n_cols, block_rows=4096):
    """Advance numpy's legacy global generator past `np.random.normal(0, 1, (n_rows, n_cols))` block by block, without
    holding the draw: the legacy normals are consumed one at a time (the cached second value of a pair included), so the
    generator ends in the same state as after the full draw."""
    for b0 in range(0, n_rows, block_rows):
        np.random.normal(0, 1, (min(block_rows, n_rows - b0), n_cols))


def _validation_period(val_each):
    """train(val_each=) -> the period of Engine.set_validation (0: no validation).  The reference validates the epochs t with
    t % val_each == 0 (mapping_optimizer.py:398), which for a negative integer are those of -val_each; 0 fails there as
    here."""
    if val_each is None:
        return 0
    every = int(val_each)
    if every != val_each:
        raise ValueError(f"val_each must be an integer, got {val_each!r}")
    if every == 0:
        raise ZeroDivisionError("val_each = 0: integer modulo by zero")
    return abs(every)


def format_terms(terms):
    """The reference's print line (mapping_optimizer.py:300-307, :555-562) from (name, value) pairs; NaN terms are left
    out."""
    msg = ["{}: {:.3f}".format(name, value) for name, value in terms if not np.isnan(value)]
    return str(msg).replace("[", "").replace("]", "").replace("'", "")


class _EngineMapper:
    """What Mapper and MapperConstrained share: an Engine (`_engine`) of n_cells x n_voxels, the cell-sharded setup and
    loop, the epoch-chunk schedule, the history fetch and the result buffer."""

    def _select_rows(self, n_rows_given, n_cells_global, shard, process_group, presharded=False):
        """Cell-sharded operation: the block [r0, r1) of the n_cells_global cells this rank keeps -- all given rows for a
        pre-sharded caller, else `shard`, else this rank's block of `process_group` (shard_rows), else every cell.  Sets
        _rows, _pg, _sharded and returns (r0, r1)."""
        self._pg = process_group
        self._rows = (0, n_rows_given)
        if presharded:
            pass
        elif shard is not None:
            self._rows = (int(shard[0]), int(shard[1]))
            if not 0 <= self._rows[0] < self._rows[1] <= n_cells_global:
                raise ValueError(f"shard {tuple(shard)} is not a non-empty block of rows of [0, {n_cells_global})")
        elif process_group is not None:
            import torch.distributed as dist
            r, w = dist.get_rank(process_group), dist.get_world_size(process_group)
            self._rows = shard_rows(n_cells_global, r, w)
        r0, r1 = self._rows
        self._sharded = (r1 - r0) != n_cells_global
        self._own_comm = False
        return r0, r1

    def _init_comm(self, pg):
        """NCCL group: lend the handle the process-level communicator of this group (tangram_b200.sharded.nccl_comm_for_group,
        created once) so that tgb200_run issues the per-iteration exchange itself.  Non-NCCL groups (gloo in the CPU tests)
        keep the host-driven exchange of tangram_b200.sharded."""
        from .sharded import nccl_comm_for_group
        got = nccl_comm_for_group(pg, self._cfg.device)
        if got is None:
            return
        self._engine.set_comm(*got)
        self._own_comm = True

    def release(self):
        """Free the device state now (M, m, v, operands: ~20 bytes per mapping element) instead of at garbage collection."""
        self._engine.close()

    def kernel_launches(self):
        return self._engine.kernel_launches()

    def project(self, X, out=None):
        """softmax(M)^T @ X on the device (project_genes' GEMM, tangram/utils.py:368) -> (n_voxels, n_cols) float32
        ndarray; or, with `out` (a contiguous float32 CUDA tensor of that shape on this mapper's device), written there."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        if X.shape[0] != self.n_cells:
            raise ValueError("X must have one row per cell")
        if out is None:
            out = np.empty((self.n_voxels, X.shape[1]), dtype=np.float32)
        else:
            self._check_out(out, (self.n_voxels, X.shape[1]))
        return self._engine.project(X, out)

    def _check_out(self, out, shape):
        import torch
        if not (isinstance(out, torch.Tensor) and out.is_cuda and out.device.index == self._cfg.device):
            raise TypeError(f"out must be a CUDA tensor on cuda:{self._cfg.device}")
        if out.dtype != torch.float32 or tuple(out.shape) != shape or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous float32 tensor of shape {shape}")

    def _run(self, n_steps, lr):
        if not self._sharded or self._own_comm:
            self._engine.run(n_steps, lr)    # sharded: the NCCL exchange is inside
            return
        from types import SimpleNamespace

        import torch
        import torch.distributed as dist
        e, stream = self._engine, torch.cuda.current_stream(self._cfg.device).cuda_stream
        # the engine protocol of tangram_b200.sharded, issued on torch's current stream
        on_stream = SimpleNamespace(exchange_tensor=e.exchange_tensor, step_begin=lambda: e.step_begin(stream),
                                    step_end=lambda lr_: e.step_end(lr_, stream))
        sharded_steps(on_stream, n_steps, lr,
                      lambda t: dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self._pg))   # the one exchange per step

    def _set_loss_genes(self, active):
        """Cross-validation fold: the loss sees only the genes flagged in `active` (n_genes booleans; None = all), as a
        mapper built on S[:, active], G[:, active] would (Engine.set_loss_genes)."""
        self._engine.set_loss_genes(active)

    def _fit(self, num_epochs, lr, print_each, resume, out=None, val_each=None, val_history=None, fetch=True):
        """num_epochs updates (a fresh Adam unless `resume`), run in chunks that end where the reference prints.  With
        `val_each`, the epochs t with t % val_each == 0 are validated on the device inside those chunks
        (Engine.set_validation) and their four values are appended to the lists of `val_history`.  Sets history_matrix to
        this call's rows and returns softmax(M), in `out` or a host array; with fetch=False (cross-validation scores genes
        with project() and needs no mapping on the host) it returns None."""
        every = _validation_period(val_each)
        if not resume:
            self._engine.reset_adam()
        first = self._engine.history_len()
        result = None
        if out is not None:
            self._check_out(out, (self.n_cells, self.n_voxels))
        elif fetch:
            result = _ResultBuffer(_lib.load(), (self.n_cells, self.n_voxels), self._cfg.device)
        validating = False
        try:
            if every:
                self._engine.set_validation(every)
                validating = True
            t = 0
            while t < num_epochs:
                if print_each:
                    chunk = min(num_epochs - t, print_each - (t % print_each))
                else:
                    chunk = num_epochs - t
                self._run(chunk, lr)
                if print_each and t % print_each == 0:
                    print(format_terms(self._print_terms(self._engine.history(first + t, 1)[0])))
                t += chunk
            self.history_matrix = self._engine.history(first, num_epochs)
            if every:
                for c, key in enumerate(_VAL_KEYS, start=_lib.HIST_VAL_TOTAL):
                    val_history[key].extend(float(x) for x in self.history_matrix[::every, c])
            if out is None and result is None:
                return None
            return self._engine.get_mapping(out if out is not None else result.ready())
        finally:
            if validating:
                self._engine.set_validation(0)
            if result is not None:
                result.release()


class Mapper(_EngineMapper):
    def __init__(
        self,
        S,
        G,
        train_genes_idx=None,
        val_genes_idx=None,
        d=None,
        d_source=None,
        lambda_g1=1.0,
        lambda_d=0,
        lambda_g2=0,
        lambda_r=0,
        lambda_l1=0,
        lambda_l2=0,
        lambda_neighborhood_g1=0,
        voxel_weights=None,
        lambda_getis_ord=0,
        lambda_geary=0,
        lambda_moran=0,
        neighborhood_filter=None,
        ct_encode=None,
        lambda_ct_islands=0,
        spatial_weights=None,
        device="cuda:0",
        adata_map=None,
        random_state=None,
        *,
        precision="bf16x3",
        M0=None,
        process_group=None,
        shard=None,
        n_cells_global=None,
    ):
        if lambda_geary > 0 or lambda_moran > 0:
            # mapping_optimizer.py:173-185: not on the accelerated path (Geary builds V x V x K)
            raise NotImplementedError("lambda_moran / lambda_geary are not supported by tangram_b200")
        if adata_map is not None:
            raise NotImplementedError  # the reference raises here too (:151-153)
        if precision not in _lib.PREC:
            raise ValueError(f"precision must be one of {list(_lib.PREC)}")
        self.device = device
        self.random_state = random_state
        self.precision = precision

        S = np.asarray(S, dtype=np.float32)
        G = np.asarray(G, dtype=np.float32)
        if train_genes_idx is not None:      # :87-92 (val subset is never read, :321-322)
            S = S[:, train_genes_idx]
            G = G[:, train_genes_idx]
        S = np.ascontiguousarray(S)
        G = np.ascontiguousarray(G)
        if S.shape[1] != G.shape[1]:
            raise ValueError("S and G must have the same number of genes")
        n_rows_given, n_voxels, n_genes = S.shape[0], G.shape[0], S.shape[1]
        presharded = n_cells_global is not None
        n_cells_global = int(n_cells_global) if presharded else n_rows_given
        if n_cells_global < n_rows_given:
            raise ValueError(f"n_cells_global={n_cells_global} is smaller than the {n_rows_given} rows of S given")

        self.target_density_enabled = d is not None
        self.source_density_enabled = d_source is not None
        density_mode = _lib.DENSITY_NONE
        if self.target_density_enabled:
            density_mode = _lib.DENSITY_SOURCE if self.source_density_enabled else _lib.DENSITY_CELLS
        if ct_encode is not None:
            ct_encode = np.ascontiguousarray(np.asarray(ct_encode, dtype=np.float32))
        n_types = ct_encode.shape[1] if (ct_encode is not None and lambda_ct_islands > 0) else 0

        if M0 is not None:
            M0 = np.asarray(M0)
            if M0.shape != (n_rows_given, n_voxels):
                raise ValueError("M0 has the wrong shape")

        # cell-sharded operation: this rank keeps rows [r0, r1)
        r0, r1 = self._select_rows(n_rows_given, n_cells_global, shard, process_group, presharded)
        self._presharded = presharded
        if M0 is not None:
            M0 = M0[r0:r1]

        e = self._engine = Engine(
            r1 - r0, n_voxels, n_genes, n_types=n_types, n_cells_global=n_cells_global, device=_device_index(device),
            precision=precision, density_mode=density_mode, lambda_g1=lambda_g1, lambda_d=lambda_d,
            lambda_g2=lambda_g2, lambda_r=lambda_r, lambda_l1=lambda_l1, lambda_l2=lambda_l2,
            lambda_neighborhood_g1=lambda_neighborhood_g1, lambda_ct_islands=lambda_ct_islands,
            lambda_getis_ord=lambda_getis_ord)
        self._cfg = e.cfg
        self.n_cells, self.n_voxels, self.n_genes = r1 - r0, n_voxels, n_genes

        e.set_expression(np.ascontiguousarray(S[r0:r1]), G)
        if self.target_density_enabled:
            ds = None
            if self.source_density_enabled:
                ds = np.ascontiguousarray(np.asarray(d_source, dtype=np.float32)[r0:r1])
            e.set_density(np.ascontiguousarray(np.asarray(d, dtype=np.float32)), ds)
        graphs = []
        if lambda_neighborhood_g1 > 0:
            graphs.append((_lib.GRAPH_VOXEL_WEIGHTS, voxel_weights, "voxel_weights"))
        if lambda_ct_islands > 0:
            graphs.append((_lib.GRAPH_NEIGHBORHOOD_FILTER, neighborhood_filter, "neighborhood_filter"))
        if lambda_getis_ord > 0:
            graphs.append((_lib.GRAPH_SPATIAL_WEIGHTS, spatial_weights, "spatial_weights"))
        for which, mat, name in graphs:
            if mat is None:
                raise ValueError(f"{name} is required by the enabled lambda")
            e.set_graph(which, mat)
        if lambda_ct_islands > 0:
            if ct_encode is None:
                raise ValueError("ct_encode is required when lambda_ct_islands > 0")
            e.set_ct_encode(np.ascontiguousarray(ct_encode[r0:r1]))
        if M0 is None:
            self._draw_initial_mapping()
        else:
            e.set_mapping(np.ascontiguousarray(M0, dtype=np.float32))
            del M0
        if self._sharded and process_group is not None:
            self._init_comm(process_group)

    def _draw_initial_mapping(self):
        """The reference's initial mapping (:147-157): np.random.normal(0, 1, (N, V)) from numpy's legacy global generator,
        seeded first only if random_state is truthy, cast to float32.  A rank of a sharded run draws the same stream and
        keeps only its rows (pre-sharded callers get a per-rank draw).  The draw runs on the device (legacy_rng) unless
        this numpy's arithmetic differs from the device formula; either way the generator ends where the host draw leaves
        it.  Resets the Adam state and the history."""
        r0, r1 = self._rows
        if not self._presharded and legacy_rng.device_draw_supported():
            if self.random_state:
                np.random.seed(seed=self.random_state)
            legacy_rng.draw_global(self._engine, 0, r0, r1 * self.n_voxels)   # the generator ends after row r1
        else:
            M0 = legacy_normal_rows(self.random_state, r1, self.n_voxels, r0, r1)
            self._engine.set_mapping(np.ascontiguousarray(M0, dtype=np.float32))

    # ------------------------------------------------------------------------------
    @staticmethod
    def _print_terms(row):
        return [(name, row[c]) for c, name in _PRINT_TERMS]

    def train(self, num_epochs, learning_rate=0.1, print_each=100, val_each=None, *, resume=False, out=None):
        """mapping_optimizer.py:358-408.  Returns (softmax(M) as (N, V) f32 ndarray, history).
        Every call starts a fresh Adam (zero moments, t = 1) like the reference's `torch.optim.Adam([self.M])` at :373;
        `resume=True` keeps the optimizer state of the previous call instead.
        `out`: a contiguous float32 CUDA tensor of shape (N, V) on this mapper's device; softmax(M) is written there
        (device to device, no host copy) and `out` is returned in place of the ndarray."""
        import logging
        if print_each:
            logging.info(f"Printing scores every {print_each} epochs.")
        val_history = {key: [] for key in _VAL_KEYS}
        output = self._fit(num_epochs, float(learning_rate), print_each, resume, out, val_each, val_history)
        rows = self.history_matrix
        training_history = {"total_loss": [np.array(x, dtype=np.float32) for x in rows[:, 0]]}   # 0-d ndarrays (:390)
        for c, key in enumerate(_HIST_KEYS[1:], start=1):
            training_history[key] = [float(x) for x in rows[:, c]]
        training_history.update(val_history)
        return output, training_history

    # --- extras beyond the reference surface -------------------------------------------
    def validation_terms(self):
        """The reference's validation scores (_val_loss_fn, mapping_optimizer.py:311-356) of the current mapping:
        {val_total_loss, val_gene_sim, val_sp_sparsity_weighted_sim, val_entropy} as floats."""
        return {k: float(x) for k, x in zip(_VAL_KEYS, self._engine.validation_terms())}

    def state(self):
        """(M, m, v, step): checkpoint of the optimizer (the reference stubs resume, :151-153)."""
        M = np.empty((self.n_cells, self.n_voxels), dtype=np.float32)
        m = np.empty_like(M)
        v = np.empty_like(M)
        return M, m, v, self._engine.get_state(M, m, v)

    def load_state(self, M, m, v, step):
        M, m, v = (np.ascontiguousarray(x, dtype=np.float32) for x in (M, m, v))
        self._engine.set_state(M, m, v, step)

    def _debug(self, name):
        """Diagnostics: internal device buffer by name (see tgb200_debug_buffer)."""
        return self._engine.debug(name)


class MapperConstrained(_EngineMapper):
    """Drop-in for the reference `MapperConstrained` (mapping_optimizer.py:411-639): same constructor keywords,
    `train()` returns `(mapping, F_out, training_history)` with the reference's history conventions (all values are
    strings, :630).  The per-cell filter rides the same kernels: S_f = sigmoid(F) o S is the operand of all three
    contractions, dL/df_i is the row-dot the backward pass needs anyway, and F gets its own small Adam kernel.

    Cell-sharded like Mapper (`process_group=` / `shard=`): every rank passes the full S (and M0, F0) and keeps a block of
    cells -- its rows of M and S, its entries of F and the Adam state of both.  The filter's global sums (sum f and the
    f-regulariser) travel in the tail of the one exchange per epoch, so every rank sees the global loss; `train()` returns
    this rank's mapping rows and F_out entries, with the global history."""
    _KEYS = ["total_loss", "main_loss", "vg_reg", "kl_reg", "entropy_reg", "count_reg", "lambda_f_reg"]
    _PRINT_NAMES = ["Score", "VG reg", "KL reg", "Entropy reg", "Count reg", "Lambda f reg"]          # :555-562

    def __init__(self, S, G, d, lambda_d=1, lambda_g1=1, lambda_g2=1, lambda_r=0, lambda_count=1, lambda_f_reg=1,
                 target_count=None, device="cuda:0", adata_map=None, random_state=None, *, precision="bf16x3",
                 M0=None, F0=None, process_group=None, shard=None):
        if adata_map is not None:
            raise NotImplementedError      # the reference raises here too (:476-477)
        if precision not in _lib.PREC:
            raise ValueError(f"precision must be one of {list(_lib.PREC)}")
        self.random_state = random_state
        S = np.ascontiguousarray(np.asarray(S, dtype=np.float32))
        G = np.ascontiguousarray(np.asarray(G, dtype=np.float32))
        n_cells, n_voxels, n_genes = S.shape[0], G.shape[0], S.shape[1]
        if M0 is not None and F0 is not None:
            M0, F0 = np.asarray(M0), np.asarray(F0)
            if M0.shape != (n_cells, n_voxels) or F0.shape != (n_cells,):
                raise ValueError("M0 / F0 have the wrong shape")
        # cell-sharded operation: this rank keeps cells [r0, r1)
        r0, r1 = self._select_rows(n_cells, n_cells, shard, process_group)
        self.target_density_enabled = d is not None
        e = self._engine = Engine(
            r1 - r0, n_voxels, n_genes, n_cells_global=n_cells, device=_device_index(device), precision=precision,
            density_mode=_lib.DENSITY_CELLS if self.target_density_enabled else _lib.DENSITY_NONE,
            lambda_g1=lambda_g1, lambda_d=lambda_d, lambda_g2=lambda_g2, lambda_r=lambda_r, constrained=True,
            lambda_count=lambda_count, lambda_f_reg=lambda_f_reg,
            target_count=float(n_voxels if target_count is None else target_count))      # :480-483
        self._cfg = e.cfg
        self.n_cells, self.n_voxels, self.n_genes = r1 - r0, n_voxels, n_genes
        self._n_cells_global = n_cells
        e.set_expression(np.ascontiguousarray(S[r0:r1]), G)
        if self.target_density_enabled:
            e.set_density(np.ascontiguousarray(np.asarray(d, dtype=np.float32)))
        if M0 is None or F0 is None:
            self._draw_initial_mapping()
        else:
            e.set_mapping(np.ascontiguousarray(M0[r0:r1], dtype=np.float32))
            e.set_filter(np.ascontiguousarray(F0[r0:r1], dtype=np.float32))
        if self._sharded and process_group is not None:
            self._init_comm(process_group)

    def _draw_initial_mapping(self):
        """The reference's initial M and F (:472-493) from numpy's legacy global generator, seeded first only if
        random_state is truthy: M is drawn twice (the second draw is used), F after it.  M is drawn on the device when
        this numpy's arithmetic matches the device formula (the first N x V normals are skipped), F on the host.  A rank
        of a sharded run keeps rows [r0, r1) of the second draw and F[r0:r1]; on every rank the generator ends where the
        unsharded draw leaves it.  Resets the Adam state (of M and F) and the history."""
        n_cells, n_voxels = self._n_cells_global, self.n_voxels
        r0, r1 = self._rows
        if self.random_state:
            np.random.seed(seed=self.random_state)
        if legacy_rng.device_draw_supported():
            legacy_rng.draw_global(self._engine, n_cells * n_voxels, r0, 2 * n_cells * n_voxels)
        else:
            discard_normal_rows(n_cells, n_voxels)                       # the first draw, discarded (:475)
            M0 = legacy_normal_rows(None, n_cells, n_voxels, r0, r1)     # rows [r0, r1) of the second (:485)
            discard_normal_rows(n_cells - r1, n_voxels)
            self._engine.set_mapping(np.ascontiguousarray(M0, dtype=np.float32))
        F0 = np.random.normal(0, 1, n_cells)                                # :490
        self._engine.set_filter(np.ascontiguousarray(F0[r0:r1], dtype=np.float32))

    def _print_terms(self, row):
        return zip(self._PRINT_NAMES, self._values_from_row(row))

    def train(self, num_epochs, learning_rate=0.1, print_each=100, *, resume=False):
        """mapping_optimizer.py:589-639.  A fresh Adam over [M, F] per call (:607) unless resume=True."""
        output = self._fit(num_epochs, float(learning_rate), print_each, resume)
        hist = {k: [] for k in self._KEYS}
        for r in self.history_matrix:
            hist["total_loss"].append("tensor({:.4f}, grad_fn=<AddBackward0>)".format(float(r[0])))     # str(tensor), :630
            for k, v in zip(self._KEYS[1:], self._values_from_row(r)):
                hist[k].append(str(v))
        F_out = np.empty(self.n_cells, dtype=np.float32)
        self._engine.get_filter(sigmoid=F_out)
        return output, F_out, hist

    @staticmethod
    def _values_from_row(r):
        """(main_loss, vg_reg, kl_reg, entropy_reg, count_reg, lambda_f_reg) with the reference's sign/NaN conventions."""
        ent = -float(r[4])            # the reference logs +sum(P log P) here (:526, :540)
        return (float(r[1]), float(r[2]), float(r[3]), ent, float(r[10]), float(r[11]))

    def filter_logits(self):
        F = np.empty(self.n_cells, dtype=np.float32)
        self._engine.get_filter(logits=F)
        return F

    def state(self):
        M = np.empty((self.n_cells, self.n_voxels), dtype=np.float32)
        step = self._engine.get_state(M)
        return M, self.filter_logits(), step
