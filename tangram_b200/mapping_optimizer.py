"""
Drop-in replacement for the reference optimizer class `Mapper`
(Tangram's tangram/mapping_optimizer.py:14-408), running on the sm_90a (H100) C-ABI
library (include/tangram_b200.h).  Same constructor keywords, same `train()` signature,
same return types and history conventions.  There is no CPU path: `device` must be a
CUDA device with compute capability 9.0.

Additions (keyword-only, all optional):
  precision   "bf16x3" (default: parity-grade fp32 results on wgmma tensor cores -- every operand is split into three
              bf16 planes and the six significant partial products are accumulated in fp32) |
              "fp32" (FFMA contractions, the cross-check) | "bf16" (plain bf16 operands: throughput mode)
  M0          explicit initial mapping (ndarray N x V); default is the reference draw
  process_group / shard  cell-sharded multi-GPU operation (one process per GPU): every rank passes the
              full S (/ M0) and keeps rows shard_rows(N, rank, world); with a NCCL process group the handle gets its own
              NCCL communicator (tgb200_comm_init_rank) and the per-iteration exchange runs inside tgb200_run
  n_cells_global         pre-sharded variant: S, M0, d_source, ct_encode already hold only this rank's rows
  train(..., resume=True)  continue with the Adam state of the previous train() call (the reference -- and the default
              here -- builds a fresh optimizer in every train() call, mapping_optimizer.py:373)
"""
import ctypes

import numpy as np

from . import _lib
from .sharded import shard_rows, sharded_steps

_HIST_KEYS = ["total_loss", "main_loss", "vg_reg", "kl_reg", "entropy_reg"]
_VAL_KEYS = ["val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy"]
# (history column, printed name) in the reference's print order (mapping_optimizer.py:273-298)
_PRINT_TERMS = [
    (1, "Gene-voxel score"), (2, "Voxel-gene score"), (3, "Cell densities reg"), (4, "Entropy reg"),
    (5, "L1 reg"), (6, "L2 reg"), (7, "Spatial weighted score"), (8, "Cell type islands penalty"),
    (9, "Getis-Ord score"),
]


def _device_index(device):
    """'cuda', 'cuda:1', torch.device -> ordinal.  'cpu' is refused: no CPU fallback."""
    s = str(device)
    if s.startswith("cuda"):
        return int(s.split(":")[1]) if ":" in s else 0
    raise ValueError(
        f"tangram_b200.Mapper runs on H100 GPUs only (device={device!r}); "
        "use the reference implementation for device='cpu'")


def _to_csr(mat, n):
    """dense ndarray (what the reference passes, mapping_utils.py:319-329) or scipy sparse -> CSR triplet."""
    import scipy.sparse as sp
    if mat is None:
        return None
    if hasattr(mat, "detach"):
        mat = mat.detach().cpu().numpy()
    csr = mat.tocsr() if sp.issparse(mat) else sp.csr_matrix(np.asarray(mat))
    if csr.shape != (n, n):
        raise ValueError(f"spatial operator has shape {csr.shape}, expected {(n, n)}")
    csr.sort_indices()
    return (np.ascontiguousarray(csr.indptr, dtype=np.int32),
            np.ascontiguousarray(csr.indices, dtype=np.int32),
            np.ascontiguousarray(csr.data, dtype=np.float32))


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


def format_terms(row):
    """The reference's print line (mapping_optimizer.py:300-307) from one history row."""
    msg = ["{}: {:.3f}".format(name, row[c]) for c, name in _PRINT_TERMS if not np.isnan(row[c])]
    return str(msg).replace("[", "").replace("]", "").replace("'", "")


class Mapper:
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
        self._lib = _lib.load()
        self._h = None
        self._pg = process_group

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
        self._rows = (0, n_rows_given)
        if presharded:
            pass
        elif shard is not None:
            self._rows = (int(shard[0]), int(shard[1]))
        elif process_group is not None:
            import torch.distributed as dist
            r, w = dist.get_rank(process_group), dist.get_world_size(process_group)
            self._rows = shard_rows(n_cells_global, r, w)
        r0, r1 = self._rows
        sharded = (r1 - r0) != n_cells_global
        # initial mapping: legacy numpy RNG, float64 draw, f32 cast; seeded only if truthy (:147-157).  A rank of a
        # sharded run draws the same stream and keeps only its rows (pre-sharded callers pass M0 or get a per-rank draw).
        if M0 is None:
            M0 = legacy_normal_rows(self.random_state, n_rows_given, n_voxels, r0, r1)
        else:
            M0 = M0[r0:r1]

        cfg = _lib.Config()
        cfg.struct_size = ctypes.sizeof(_lib.Config)
        cfg.device = _device_index(device)
        cfg.n_cells, cfg.n_voxels, cfg.n_genes, cfg.n_types = r1 - r0, n_voxels, n_genes, n_types
        cfg.n_cells_global = n_cells_global
        cfg.precision = _lib.PREC[precision]
        cfg.density_mode = density_mode
        cfg.lambda_g1, cfg.lambda_d, cfg.lambda_g2 = lambda_g1, lambda_d, lambda_g2
        cfg.lambda_r, cfg.lambda_l1, cfg.lambda_l2 = lambda_r, lambda_l1, lambda_l2
        cfg.lambda_neighborhood_g1 = lambda_neighborhood_g1
        cfg.lambda_ct_islands = lambda_ct_islands
        cfg.lambda_getis_ord = lambda_getis_ord
        cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps = 0.9, 0.999, 1e-8   # torch.optim.Adam defaults (:373)
        h = ctypes.c_void_p()
        _lib.check(self._lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)))
        self._h = h
        self._cfg = cfg
        self._sharded = sharded
        self.n_cells, self.n_voxels, self.n_genes = r1 - r0, n_voxels, n_genes

        L = self._lib
        _lib.check(L.tgb200_set_expression(h, _lib.ptr(np.ascontiguousarray(S[r0:r1])), _lib.ptr(G), None))
        if self.target_density_enabled:
            dd = np.ascontiguousarray(np.asarray(d, dtype=np.float32))
            ds = None
            if self.source_density_enabled:
                ds = np.ascontiguousarray(np.asarray(d_source, dtype=np.float32)[r0:r1])
            _lib.check(L.tgb200_set_density(h, _lib.ptr(dd), _lib.ptr(ds), None))
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
            indptr, indices, vals = _to_csr(mat, n_voxels)
            _lib.check(L.tgb200_set_graph(h, which, _lib.ptr(indptr), _lib.ptr(indices), _lib.ptr(vals),
                                          len(vals), None))
        if lambda_ct_islands > 0:
            if ct_encode is None:
                raise ValueError("ct_encode is required when lambda_ct_islands > 0")
            _lib.check(L.tgb200_set_ct_encode(h, _lib.ptr(np.ascontiguousarray(ct_encode[r0:r1])), None))
        M0 = np.ascontiguousarray(M0, dtype=np.float32)
        _lib.check(L.tgb200_set_mapping(h, _lib.ptr(M0), None))
        del M0
        self._own_comm = False
        if sharded and process_group is not None:
            self._init_comm(process_group)

    def _init_comm(self, pg):
        """NCCL group: lend the handle the process-level communicator of this group (tangram_b200.sharded.nccl_comm_for_group,
        created once) so that tgb200_run issues the per-iteration exchange itself.  Non-NCCL groups (gloo in the CPU tests)
        keep the host-driven exchange of tangram_b200.sharded."""
        from .sharded import nccl_comm_for_group
        got = nccl_comm_for_group(pg, self._cfg.device)
        if got is None:
            return
        comm, rank, world = got
        _lib.check(self._lib.tgb200_set_comm(self._h, comm, rank, world))
        self._own_comm = True

    # ------------------------------------------------------------------------------
    def release(self):
        """Free the device state now (M, m, v, operands: ~20 bytes per mapping element) instead of at garbage collection."""
        if self._h is not None:
            self._lib.tgb200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass

    def _history_rows(self, first, count):
        out = np.empty((count, _lib.HIST_COLS), dtype=np.float32)
        if count:
            _lib.check(self._lib.tgb200_get_history(self._h, first, count, _lib.ptr(out), None))
        return out

    def _exchange_tensor(self):
        """torch view of the device exchange buffer (for torch.distributed.all_reduce)."""
        import torch
        p = ctypes.c_void_p()
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_exchange_buffer(self._h, ctypes.byref(p), ctypes.byref(n)))

        class _Wrap:
            __cuda_array_interface__ = {
                "shape": (n.value,), "typestr": "<f4", "data": (p.value, False), "version": 3, "strides": None}
        return torch.as_tensor(_Wrap(), device=f"cuda:{self._cfg.device}")

    def _run(self, n_steps, lr):
        if n_steps <= 0:
            return
        if not self._sharded or self._own_comm:
            _lib.check(self._lib.tgb200_run(self._h, n_steps, lr, None))    # sharded: the NCCL exchange is inside
            return
        import torch
        import torch.distributed as dist
        mapper, stream = self, ctypes.c_void_p(torch.cuda.current_stream(self._cfg.device).cuda_stream)

        class _Eng:   # the engine protocol of tangram_b200.sharded over the C-ABI handle
            def exchange_tensor(self):
                return mapper._exchange_tensor()

            def step_begin(self):
                _lib.check(mapper._lib.tgb200_step_begin(mapper._h, stream))

            def step_end(self, lr_):
                _lib.check(mapper._lib.tgb200_step_end(mapper._h, lr_, stream))

        sharded_steps(_Eng(), n_steps, lr,
                      lambda t: dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self._pg))   # the one exchange per step

    def train(self, num_epochs, learning_rate=0.1, print_each=100, val_each=None, *, resume=False):
        """mapping_optimizer.py:358-408.  Returns (softmax(M) as (N, V) f32 ndarray, history).
        Every call starts a fresh Adam (zero moments, t = 1) like the reference's `torch.optim.Adam([self.M])` at :373;
        `resume=True` keeps the optimizer state of the previous call instead."""
        import logging
        if print_each:
            logging.info(f"Printing scores every {print_each} epochs.")
        if not resume:
            _lib.check(self._lib.tgb200_reset_adam(self._h, None))
        training_history = {key: [] for key in _HIST_KEYS + _VAL_KEYS}
        first = ctypes.c_int64()
        _lib.check(self._lib.tgb200_history_len(self._h, ctypes.byref(first)))
        first = first.value
        lr = float(learning_rate)
        result = _ResultBuffer(self._lib, (self.n_cells, self.n_voxels), self._cfg.device)
        try:
            return self._train_loop(num_epochs, lr, print_each, val_each, first, training_history, result)
        finally:
            result.release()

    def _train_loop(self, num_epochs, lr, print_each, val_each, first, training_history, result):
        t = 0
        while t < num_epochs:
            if val_each is not None:
                chunk = 1
            elif print_each:
                chunk = min(num_epochs - t, print_each - (t % print_each))
            else:
                chunk = num_epochs - t
            self._run(chunk, lr)
            if print_each and t % print_each == 0:
                print(format_terms(self._history_rows(first + t, 1)[0]))
            if val_each is not None and t % val_each == 0:
                vals = np.zeros(4, dtype=np.float32)
                _lib.check(self._lib.tgb200_validation_terms(self._h, _lib.ptr(vals), None))
                for k, x in zip(_VAL_KEYS, vals):
                    training_history[k].append(float(x))
            t += chunk

        rows = self._history_rows(first, num_epochs)
        training_history["total_loss"] = [np.array(x, dtype=np.float32) for x in rows[:, 0]]   # 0-d ndarrays (:390)
        for c, key in enumerate(_HIST_KEYS[1:], start=1):
            training_history[key] = [float(x) for x in rows[:, c]]
        self.history_matrix = rows
        output = result.ready()
        _lib.check(self._lib.tgb200_get_mapping(self._h, _lib.ptr(output), None))
        return output, training_history

    # --- extras beyond the reference surface -------------------------------------------
    def state(self):
        """(M, m, v, step): checkpoint of the optimizer (the reference stubs resume, :151-153)."""
        M = np.empty((self.n_cells, self.n_voxels), dtype=np.float32)
        m = np.empty_like(M)
        v = np.empty_like(M)
        step = ctypes.c_int64()
        _lib.check(self._lib.tgb200_get_state(self._h, _lib.ptr(M), _lib.ptr(m), _lib.ptr(v), ctypes.byref(step), None))
        return M, m, v, step.value

    def load_state(self, M, m, v, step):
        M, m, v = (np.ascontiguousarray(x, dtype=np.float32) for x in (M, m, v))
        _lib.check(self._lib.tgb200_set_state(self._h, _lib.ptr(M), _lib.ptr(m), _lib.ptr(v), int(step), None))

    def project(self, X):
        """softmax(M)^T @ X on the device (project_genes' GEMM, tangram/utils.py:368)."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        if X.shape[0] != self.n_cells:
            raise ValueError("X must have one row per cell")
        out = np.empty((self.n_voxels, X.shape[1]), dtype=np.float32)
        _lib.check(self._lib.tgb200_project(self._h, _lib.ptr(X), X.shape[1], _lib.ptr(out), None))
        return out

    def _debug(self, name):
        """Diagnostics: internal device buffer by name (see tgb200_debug_buffer)."""
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_debug_buffer(self._h, name.encode(), None, 0, ctypes.byref(n)))
        out = np.empty(max(n.value, 4), dtype=np.float32)
        _lib.check(self._lib.tgb200_debug_buffer(self._h, name.encode(), _lib.ptr(out), out.size, ctypes.byref(n)))
        return out[:n.value]

    def kernel_launches(self):
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_kernel_launches(self._h, ctypes.byref(n)))
        return n.value


class MapperConstrained:
    """Drop-in for the reference `MapperConstrained` (mapping_optimizer.py:411-639): same constructor keywords,
    `train()` returns `(mapping, F_out, training_history)` with the reference's history conventions (all values are
    strings, :630).  The per-cell filter rides the same kernels: S_f = sigmoid(F) o S is the operand of all three
    contractions, dL/df_i is the row-dot the backward pass needs anyway, and F gets its own small Adam kernel."""

    def __init__(self, S, G, d, lambda_d=1, lambda_g1=1, lambda_g2=1, lambda_r=0, lambda_count=1, lambda_f_reg=1,
                 target_count=None, device="cuda:0", adata_map=None, random_state=None, *, precision="bf16x3",
                 M0=None, F0=None):
        if adata_map is not None:
            raise NotImplementedError      # the reference raises here too (:476-477)
        if precision not in _lib.PREC:
            raise ValueError(f"precision must be one of {list(_lib.PREC)}")
        self._lib = _lib.load()
        self._h = None
        self.random_state = random_state
        S = np.ascontiguousarray(np.asarray(S, dtype=np.float32))
        G = np.ascontiguousarray(np.asarray(G, dtype=np.float32))
        n_cells, n_voxels, n_genes = S.shape[0], G.shape[0], S.shape[1]
        self.target_density_enabled = d is not None
        if M0 is None or F0 is None:
            # :472-493 -- M is drawn twice (the second draw is used), F after it, legacy numpy RNG
            if self.random_state:
                np.random.seed(seed=self.random_state)
            np.random.normal(0, 1, (n_cells, n_voxels))
            M0 = np.random.normal(0, 1, (n_cells, n_voxels))
            F0 = np.random.normal(0, 1, n_cells)
        cfg = _lib.Config()
        cfg.struct_size = ctypes.sizeof(_lib.Config)
        cfg.device = _device_index(device)
        cfg.n_cells, cfg.n_voxels, cfg.n_genes, cfg.n_types = n_cells, n_voxels, n_genes, 0
        cfg.n_cells_global = n_cells
        cfg.precision = _lib.PREC[precision]
        cfg.density_mode = _lib.DENSITY_CELLS if self.target_density_enabled else _lib.DENSITY_NONE
        cfg.lambda_g1, cfg.lambda_d, cfg.lambda_g2, cfg.lambda_r = lambda_g1, lambda_d, lambda_g2, lambda_r
        cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps = 0.9, 0.999, 1e-8
        cfg.constrained = 1
        cfg.lambda_count, cfg.lambda_f_reg = lambda_count, lambda_f_reg
        cfg.target_count = float(n_voxels if target_count is None else target_count)      # :480-483
        self._lam = dict(g1=lambda_g1, d=lambda_d, g2=lambda_g2, r=lambda_r, c=lambda_count, f=lambda_f_reg)
        h = ctypes.c_void_p()
        _lib.check(self._lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(h)))
        self._h, self._cfg = h, cfg
        self.n_cells, self.n_voxels, self.n_genes = n_cells, n_voxels, n_genes
        L = self._lib
        _lib.check(L.tgb200_set_expression(h, _lib.ptr(S), _lib.ptr(G), None))
        if self.target_density_enabled:
            dd = np.ascontiguousarray(np.asarray(d, dtype=np.float32))
            _lib.check(L.tgb200_set_density(h, _lib.ptr(dd), None, None))
        _lib.check(L.tgb200_set_mapping(h, _lib.ptr(np.ascontiguousarray(M0, dtype=np.float32)), None))
        _lib.check(L.tgb200_set_filter(h, _lib.ptr(np.ascontiguousarray(F0, dtype=np.float32)), None))

    def __del__(self):
        try:
            if self._h is not None:
                self._lib.tgb200_destroy(self._h)
                self._h = None
        except Exception:  # noqa: BLE001
            pass

    @staticmethod
    def _print_line(vals):
        names = ["Score", "VG reg", "KL reg", "Entropy reg", "Count reg", "Lambda f reg"]          # :555-562
        msg = ["{}: {:.3f}".format(n, v) for n, v in zip(names, vals) if not np.isnan(v)]
        return str(msg).replace("[", "").replace("]", "").replace("'", "")

    def train(self, num_epochs, learning_rate=0.1, print_each=100, *, resume=False):
        """mapping_optimizer.py:589-639.  A fresh Adam over [M, F] per call (:607) unless resume=True."""
        keys = ["total_loss", "main_loss", "vg_reg", "kl_reg", "entropy_reg", "count_reg", "lambda_f_reg"]
        if not resume:
            _lib.check(self._lib.tgb200_reset_adam(self._h, None))
        first = ctypes.c_int64()
        _lib.check(self._lib.tgb200_history_len(self._h, ctypes.byref(first)))
        first = first.value
        result = _ResultBuffer(self._lib, (self.n_cells, self.n_voxels), self._cfg.device)
        try:
            return self._train_loop(num_epochs, learning_rate, print_each, first, keys, result)
        finally:
            result.release()

    def _train_loop(self, num_epochs, learning_rate, print_each, first, keys, result):
        t = 0
        while t < num_epochs:
            chunk = min(num_epochs - t, print_each - (t % print_each)) if print_each else num_epochs - t
            _lib.check(self._lib.tgb200_run(self._h, chunk, float(learning_rate), None))
            if print_each and t % print_each == 0:
                print(self._print_line(self._row_values(first + t)))
            t += chunk
        rows = np.empty((num_epochs, _lib.HIST_COLS), dtype=np.float32)
        if num_epochs:
            _lib.check(self._lib.tgb200_get_history(self._h, first, num_epochs, _lib.ptr(rows), None))
        self.history_matrix = rows
        hist = {k: [] for k in keys}
        for r in rows:
            vals = self._values_from_row(r)
            hist["total_loss"].append("tensor({:.4f}, grad_fn=<AddBackward0>)".format(float(r[0])))     # str(tensor), :630
            for k, v in zip(keys[1:], vals):
                hist[k].append(str(v))
        output = result.ready()
        _lib.check(self._lib.tgb200_get_mapping(self._h, _lib.ptr(output), None))
        F_out = np.empty(self.n_cells, dtype=np.float32)
        _lib.check(self._lib.tgb200_get_filter(self._h, None, _lib.ptr(F_out), None))
        return output, F_out, hist

    def _values_from_row(self, r):
        """(main_loss, vg_reg, kl_reg, entropy_reg, count_reg, lambda_f_reg) with the reference's sign/NaN conventions."""
        ent = -float(r[4])            # the reference logs +sum(P log P) here (:526, :540)
        return (float(r[1]), float(r[2]), float(r[3]), ent, float(r[10]), float(r[11]))

    def _row_values(self, idx):
        row = np.empty((1, _lib.HIST_COLS), dtype=np.float32)
        _lib.check(self._lib.tgb200_get_history(self._h, idx, 1, _lib.ptr(row), None))
        return self._values_from_row(row[0])

    def filter_logits(self):
        F = np.empty(self.n_cells, dtype=np.float32)
        _lib.check(self._lib.tgb200_get_filter(self._h, _lib.ptr(F), None, None))
        return F

    def state(self):
        M = np.empty((self.n_cells, self.n_voxels), dtype=np.float32)
        step = ctypes.c_int64()
        _lib.check(self._lib.tgb200_get_state(self._h, _lib.ptr(M), None, None, ctypes.byref(step), None))
        return M, self.filter_logits(), step.value


MapperConstrained.release = Mapper.release
MapperConstrained.project = Mapper.project
MapperConstrained.kernel_launches = Mapper.kernel_launches
