"""The one Python owner of a C-ABI handle (include/tangram_b200.h): every call that takes a `tgb200_mapper*` goes through
`Engine`.  `Mapper` and `MapperConstrained` (the reference-shaped front ends) and the tuner build on it; callers that
manage their own buffers (bench.py, multi-GPU drivers) use it directly."""
import ctypes

import numpy as np

from . import _lib


def _device_index(device):
    """Mapper's device: 'cuda' (device 0), 'cuda:1', torch.device -> ordinal.  'cpu' is refused: no CPU fallback."""
    s = str(device)
    if s.startswith("cuda"):
        return int(s.split(":")[1]) if ":" in s else 0
    raise ValueError(
        f"tangram_b200.Mapper runs on H100 GPUs only (device={device!r}); "
        "use the reference implementation for device='cpu'")


def _require_device(device):
    """The tuner's and annotation helpers' device: -> ordinal of a visible CUDA device ('cuda' is torch's current one),
    or TangramB200Error: there is no CPU fallback."""
    import torch
    s = str(device)
    if not s.startswith("cuda"):
        raise _lib.TangramB200Error(f"tangram_b200 runs on H100 GPUs only (device={device!r}); no CPU fallback")
    if not torch.cuda.is_available():
        raise _lib.TangramB200Error("no CUDA device visible: tangram_b200 has no CPU fallback")
    return int(s.split(":")[1]) if ":" in s else torch.cuda.current_device()


def _csr(mat, n):
    """n x n spatial operator -- dense ndarray (what the reference passes, mapping_utils.py:319-329), torch tensor or
    scipy sparse -> CSR triplet (int32 indptr, int32 indices, float32 values) with sorted indices."""
    import scipy.sparse as sp
    if hasattr(mat, "detach"):
        mat = mat.detach().cpu().numpy()
    csr = mat.tocsr() if sp.issparse(mat) else sp.csr_matrix(np.asarray(mat))
    if csr.shape != (n, n):
        raise ValueError(f"spatial operator has shape {csr.shape}, expected {(n, n)}")
    csr.sort_indices()
    return (np.ascontiguousarray(csr.indptr, dtype=np.int32),
            np.ascontiguousarray(csr.indices, dtype=np.int32),
            np.ascontiguousarray(csr.data, dtype=np.float32))


# state_memory="host": bytes per mapping element (on the device, in pinned host memory).  The device keeps the contraction
# operands: bf16 P and dq in bf16 mode; three P planes and the fp32 dP in bf16x3 mode.  The host keeps M, m (bf16 in bf16
# mode) and v.
HOST_STATE_BYTES_PER_ELEMENT = {"bf16": (4, 10), "bf16x3": (10, 12)}


def host_memory_available():
    """MemAvailable of /proc/meminfo in bytes (None where the file or the field is missing)."""
    try:
        with open("/proc/meminfo") as f:
            for line in f:
                if line.startswith("MemAvailable:"):
                    return int(line.split()[1]) * 1024
    except OSError:
        return None
    return None


def check_state_memory(state_memory, precision):
    """Validate Engine's `state_memory` argument for `precision`."""
    if state_memory not in _lib.STATE_MEMORY:
        raise ValueError(f"state_memory must be one of {list(_lib.STATE_MEMORY)}, got {state_memory!r}")
    if state_memory != "device" and precision not in HOST_STATE_BYTES_PER_ELEMENT:
        raise ValueError(f"state_memory={state_memory!r} needs precision 'bf16' or 'bf16x3', not {precision!r}: fp32 fuses Adam "
                         "into its FFMA contraction's epilogue, which reads the optimizer state of every row on the device")


def check_host_state_fits(n_cells, n_voxels, n_genes, precision, device, host_available=None, device_free=None):
    """Before a state_memory="host" handle is allocated: raise TangramB200Error when the pinned host state would not fit in
    MemAvailable, or the device part (the contraction operands, estimated as the tuner estimates a handle) would not fit
    in the device's free memory.  `host_available` / `device_free` (bytes) default to /proc/meminfo and
    torch.cuda.mem_get_info."""
    dev_b, host_b = HOST_STATE_BYTES_PER_ELEMENT[precision]
    elems = n_cells * (-(-n_voxels // 64) * 64)
    need_host = host_b * elems
    if host_available is None:
        host_available = host_memory_available()
    if host_available is not None and need_host > host_available:
        raise _lib.TangramB200Error(
            f"state_memory='host' needs about {need_host / 2**30:.1f} GiB of pinned host memory for M, m and v of "
            f"{n_cells} x {n_voxels} ({host_b} B per element in {precision} mode); MemAvailable is "
            f"{host_available / 2**30:.1f} GiB")
    need_dev = dev_b * elems + 16 * (n_cells + n_voxels) * n_genes
    if device_free is None:
        import torch
        device_free, _ = torch.cuda.mem_get_info(device)
    if need_dev > device_free:
        raise _lib.TangramB200Error(
            f"state_memory='host' still needs about {need_dev / 2**30:.1f} GiB on cuda:{device} for the contraction "
            f"operands of {n_cells} x {n_voxels} ({dev_b} B per element in {precision} mode, plus the expression "
            f"operands); {device_free / 2**30:.1f} GiB are free")


def plan_state(cfg, device_free):
    """tgb200_plan_state: where a handle of `cfg` (_lib.Config) keeps its state with `device_free` bytes free on its
    device -- the split tgb200_create makes (TGB200_STATE_RESIDENT_ROWS / TGB200_STATE_BLOCK_ROWS included)."""
    plan = _lib.StatePlan()
    _lib.check(_lib.load().tgb200_plan_state(ctypes.byref(cfg), int(device_free), ctypes.byref(plan)))
    return plan


def check_auto_state_fits(cfg, host_available=None, device_free=None):
    """Before a state_memory="auto" handle is allocated: plan its split as tgb200_create will, and raise
    TangramB200Error when the host rows would not fit in MemAvailable or not even the operands, the ring and the reserve
    fit on the device.  `host_available` / `device_free` (bytes) default to /proc/meminfo and torch.cuda.mem_get_info.
    Returns the plan."""
    if device_free is None:
        import torch
        device_free, _ = torch.cuda.mem_get_info(cfg.device)
    plan = plan_state(cfg, device_free)
    n, v = cfg.n_cells, cfg.n_voxels
    if plan.host_bytes:
        if host_available is None:
            host_available = host_memory_available()
        if host_available is not None and plan.host_bytes > host_available:
            raise _lib.TangramB200Error(
                f"state_memory='auto' keeps {plan.resident_rows} of {n} rows on cuda:{cfg.device} and needs "
                f"{plan.host_bytes / 2**30:.1f} GiB of pinned host memory for the other {n - plan.resident_rows} rows of "
                f"M, m and v ({n} x {v}); MemAvailable is {host_available / 2**30:.1f} GiB")
    need_dev = plan.device_bytes + plan.reserve_bytes
    if need_dev > device_free:
        raise _lib.TangramB200Error(
            f"state_memory='auto' needs {need_dev / 2**30:.1f} GiB on cuda:{cfg.device} for {n} x {v} with "
            f"{plan.resident_rows} rows resident ({plan.device_bytes / 2**30:.1f} GiB of operands, resident rows and "
            f"ring, {plan.reserve_bytes / 2**30:.1f} GiB kept free); {device_free / 2**30:.1f} GiB are free")
    return plan


class Engine:
    """Config fields not given default to 0, except lambda_g1 (1) and lambda_d (1 when there is a density).
    state_memory="host" keeps M and Adam's moments in pinned host memory (TGB200_STATE_HOST), after checking that both
    the host and the device side fit.  state_memory="auto" keeps as many rows on the device as fit and only the rest in
    pinned host memory (TGB200_STATE_AUTO), after checking the library's plan of that split."""

    def __init__(self, n_cells, n_voxels, n_genes, *, n_types=0, n_cells_global=None, device=0,
                 precision="fp32", density_mode=_lib.DENSITY_CELLS, constrained=False, state_memory="device",
                 **lambdas):
        check_state_memory(state_memory, precision)
        self._lib = _lib.load()
        if state_memory == "host":
            check_host_state_fits(n_cells, n_voxels, n_genes, precision, device)
        cfg = _lib.Config()
        cfg.struct_size = ctypes.sizeof(_lib.Config)
        cfg.device = device
        cfg.n_cells, cfg.n_voxels, cfg.n_genes, cfg.n_types = n_cells, n_voxels, n_genes, n_types
        cfg.n_cells_global = n_cells_global or n_cells
        cfg.precision = _lib.PREC[precision]
        cfg.density_mode = density_mode
        cfg.lambda_g1 = lambdas.pop("lambda_g1", 1.0)
        cfg.lambda_d = lambdas.pop("lambda_d", 1.0 if density_mode != _lib.DENSITY_NONE else 0.0)
        for k in ("lambda_g2", "lambda_r", "lambda_l1", "lambda_l2", "lambda_neighborhood_g1",
                  "lambda_ct_islands", "lambda_getis_ord", "lambda_count", "lambda_f_reg", "target_count"):
            setattr(cfg, k, lambdas.pop(k, 0.0))
        if lambdas:
            raise TypeError(f"unknown arguments {sorted(lambdas)}")
        cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps = 0.9, 0.999, 1e-8      # torch.optim.Adam defaults
        cfg.constrained = int(constrained)
        cfg.state_memory = _lib.STATE_MEMORY[state_memory]
        if state_memory == "auto":
            check_auto_state_fits(cfg)
        self.cfg = cfg
        self._h = ctypes.c_void_p()
        _lib.check(self._lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(self._h)))

    def close(self):
        """Free the handle's state now (M, m, v, operands: ~20 bytes per mapping element) instead of at garbage collection."""
        if self._h:
            self._lib.tgb200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass

    @staticmethod
    def _s(stream):
        return ctypes.c_void_p(stream) if stream else None

    def set_expression(self, S, G, stream=None):
        _lib.check(self._lib.tgb200_set_expression(self._h, _lib.ptr(S), _lib.ptr(G), self._s(stream)))

    def set_density(self, d, d_source=None, stream=None):
        _lib.check(self._lib.tgb200_set_density(self._h, _lib.ptr(d), _lib.ptr(d_source), self._s(stream)))

    def set_ct_encode(self, E, stream=None):
        _lib.check(self._lib.tgb200_set_ct_encode(self._h, _lib.ptr(E), self._s(stream)))

    def set_graph(self, which, mat, stream=None):
        """`mat`: the n_voxels x n_voxels operator, dense, torch or scipy sparse."""
        ip, ix, vv = _csr(mat, self.cfg.n_voxels)
        _lib.check(self._lib.tgb200_set_graph(self._h, which, _lib.ptr(ip), _lib.ptr(ix), _lib.ptr(vv), len(vv),
                                              self._s(stream)))

    def set_mapping(self, M0, stream=None):
        _lib.check(self._lib.tgb200_set_mapping(self._h, _lib.ptr(M0), self._s(stream)))

    def init_mapping_normal(self, seed, stream=None, first_row=0):
        _lib.check(self._lib.tgb200_init_mapping_normal_rows(self._h, seed, first_row, self._s(stream)))

    def init_mapping_legacy(self, state, skip=0, first_row=0, end_normal=None, stream=None):
        """The reference draw np.random.normal(0, 1, ...) from the numpy generator state `state` (get_state() tuple):
        rows [first_row, first_row + n_cells) of a draw that starts `skip` normals into the stream.  Returns (the state
        after end_normal normals, default the end of these rows, as np.random.set_state takes it; values recomputed on
        the host)."""
        if end_normal is None:
            end_normal = skip + (first_row + self.cfg.n_cells) * self.cfg.n_voxels
        start, end, n_fixed = _lib.MtState.from_numpy(state), _lib.MtState(), ctypes.c_int64()
        _lib.check(self._lib.tgb200_init_mapping_legacy(self._h, ctypes.byref(start), int(skip), int(first_row),
                                                        int(end_normal), ctypes.byref(end), ctypes.byref(n_fixed),
                                                        self._s(stream)))
        return end.to_numpy(), n_fixed.value

    def set_filter(self, F0, stream=None):
        """Constrained mode: initial filter logits (n_cells)."""
        _lib.check(self._lib.tgb200_set_filter(self._h, _lib.ptr(F0), self._s(stream)))

    def get_filter(self, logits=None, sigmoid=None, stream=None):
        """Constrained mode: copy the filter logits F and/or sigmoid(F) (n_cells each; None skips) out of the handle."""
        _lib.check(self._lib.tgb200_get_filter(self._h, _lib.ptr(logits), _lib.ptr(sigmoid), self._s(stream)))

    def set_loss_genes(self, active=None, stream=None):
        """Restrict the loss to the genes flagged in `active` (n_genes booleans or 0/1 values; None = every gene).  The
        handle then computes what a handle created on S[:, active], G[:, active] computes from the same mapping; the
        mapping, the Adam state and the history are kept (tgb200_set_loss_genes)."""
        a = None
        if active is not None:
            a = np.asarray(active)
            if a.shape != (self.cfg.n_genes,):
                raise ValueError(f"active has shape {a.shape}, expected ({self.cfg.n_genes},)")
            a = np.ascontiguousarray(a, dtype=np.uint8)
        _lib.check(self._lib.tgb200_set_loss_genes(self._h, _lib.ptr(a), self._s(stream)))

    def set_validation(self, every, stream=None):
        """Validate every `every`-th epoch (counted from this call; 0 = off) inside run() / step_end(): _val_loss_fn's four
        values of the updated mapping go to history columns HIST_VAL_* of the epoch's row (tgb200_set_validation)."""
        _lib.check(self._lib.tgb200_set_validation(self._h, int(every), self._s(stream)))

    def reset_adam(self, stream=None):
        _lib.check(self._lib.tgb200_reset_adam(self._h, self._s(stream)))

    def run(self, n_steps, lr=0.1, stream=None):
        _lib.check(self._lib.tgb200_run(self._h, n_steps, lr, self._s(stream)))

    def step_begin(self, stream=None):
        _lib.check(self._lib.tgb200_step_begin(self._h, self._s(stream)))

    def step_end(self, lr=0.1, stream=None):
        _lib.check(self._lib.tgb200_step_end(self._h, lr, self._s(stream)))

    def set_comm(self, comm, rank, world):
        """Lend the handle an existing ncclComm_t (tangram_b200.sharded.nccl_comm_for_group); the caller keeps ownership."""
        _lib.check(self._lib.tgb200_set_comm(self._h, comm, rank, world))

    def exchange_tensor(self):
        """torch view of the device exchange buffer (for torch.distributed.all_reduce)."""
        import torch
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        _lib.check(self._lib.tgb200_exchange_buffer(self._h, ctypes.byref(p), ctypes.byref(n)))

        class _Wrap:
            __cuda_array_interface__ = {"shape": (n.value,), "typestr": "<f4", "data": (p.value, False),
                                        "version": 3, "strides": None}
        return torch.as_tensor(_Wrap(), device=f"cuda:{self.cfg.device}")

    def history_len(self):
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_history_len(self._h, ctypes.byref(n)))
        return n.value

    def history(self, first=0, count=None):
        """Rows [first, first + count) of the loss history (default: to the end), (count, HIST_COLS) float32."""
        if count is None:
            count = self.history_len() - first
        out = np.empty((count, _lib.HIST_COLS), dtype=np.float32)
        if count:
            _lib.check(self._lib.tgb200_get_history(self._h, first, count, _lib.ptr(out), None))
        return out

    def validation_terms(self, stream=None):
        """(val_total_loss, val_gene_sim, val_sp_sparsity_weighted_sim, val_entropy) of the current mapping, float32."""
        out = np.zeros(4, dtype=np.float32)
        _lib.check(self._lib.tgb200_validation_terms(self._h, _lib.ptr(out), self._s(stream)))
        return out

    def get_mapping(self, out, stream=None):
        _lib.check(self._lib.tgb200_get_mapping(self._h, _lib.ptr(out), self._s(stream)))
        return out

    def project(self, X, out, stream=None):
        """out (voxels x n_cols, f32) = softmax(M)^T X; X is (cells x n_cols) f32, host or device memory.  The same bits as
        utils.project(get_mapping(), X), in every precision."""
        n_cols = int(X.shape[1])
        _lib.check(self._lib.tgb200_project(self._h, _lib.ptr(X), n_cols, _lib.ptr(out), self._s(stream)))
        return out

    def get_state(self, M=None, m=None, v=None, stream=None):
        """Copy M / m / v (n_cells x n_voxels f32, host or device buffers; None skips) out of the handle; returns the step count."""
        step = ctypes.c_int64()
        _lib.check(self._lib.tgb200_get_state(self._h, _lib.ptr(M), _lib.ptr(m), _lib.ptr(v), ctypes.byref(step), self._s(stream)))
        return step.value

    def set_state(self, M, m, v, step, stream=None):
        _lib.check(self._lib.tgb200_set_state(self._h, _lib.ptr(M), _lib.ptr(m), _lib.ptr(v), int(step), self._s(stream)))

    def debug(self, name):
        """Internal device buffer by name (tgb200_debug_buffer) as a host array."""
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_debug_buffer(self._h, name.encode(), None, 0, ctypes.byref(n)))
        out = np.empty(max(n.value, 4), dtype=np.float32)
        _lib.check(self._lib.tgb200_debug_buffer(self._h, name.encode(), _lib.ptr(out), out.size, ctypes.byref(n)))
        return out[:n.value]

    def resident_rows(self):
        """Rows [0, R) of M and Adam's moments are in device memory, the rest in pinned host memory."""
        n = ctypes.c_int32()
        _lib.check(self._lib.tgb200_resident_rows(self._h, ctypes.byref(n)))
        return n.value

    def kernel_launches(self):
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_kernel_launches(self._h, ctypes.byref(n)))
        return n.value

    def profile_step(self, lr=0.1, stream=None, cap=64):
        names = (ctypes.c_char_p * cap)()
        ms = (ctypes.c_float * cap)()
        n = ctypes.c_int32()
        _lib.check(self._lib.tgb200_profile_step(self._h, lr, self._s(stream), names, ms, cap, ctypes.byref(n)))
        return [(names[i].decode(), float(ms[i])) for i in range(n.value)]

    def timeline(self, enable, cap=4096):
        """tgb200_debug_timeline: enable=True starts recording; enable=False returns [(name, stream, end_ms)]."""
        if enable:
            _lib.check(self._lib.tgb200_debug_timeline(self._h, 1, None, None, None, 0, None))
            return None
        names = (ctypes.c_char_p * cap)()
        streams = (ctypes.c_int32 * cap)()
        ms = (ctypes.c_float * cap)()
        n = ctypes.c_int32()
        _lib.check(self._lib.tgb200_debug_timeline(self._h, 0, names, streams, ms, cap, ctypes.byref(n)))
        return [(names[i].decode(), int(streams[i]), float(ms[i])) for i in range(n.value)]

    def algorithmic_cost(self):
        b, f = ctypes.c_double(), ctypes.c_double()
        _lib.check(self._lib.tgb200_algorithmic_cost(self._h, ctypes.byref(b), ctypes.byref(f)))
        return b.value, f.value
