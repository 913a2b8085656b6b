"""Thin object wrapper over the C-ABI handle (include/tangram_b200.h) for callers that
manage their own buffers (bench.py, multi-GPU drivers).  `Mapper` is the reference-shaped
front end; this is the explicit one."""
import ctypes

import numpy as np

from . import _lib


class Engine:
    def __init__(self, n_cells, n_voxels, n_genes, *, n_types=0, n_cells_global=None, device=0,
                 precision="fp32", density_mode=_lib.DENSITY_CELLS, **lambdas):
        self._lib = _lib.load()
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
                  "lambda_ct_islands", "lambda_getis_ord"):
            setattr(cfg, k, lambdas.pop(k, 0.0))
        if lambdas:
            raise TypeError(f"unknown arguments {sorted(lambdas)}")
        cfg.adam_beta1, cfg.adam_beta2, cfg.adam_eps = 0.9, 0.999, 1e-8
        self.cfg = cfg
        self._h = ctypes.c_void_p()
        _lib.check(self._lib.tgb200_create(ctypes.byref(cfg), ctypes.byref(self._h)))

    def close(self):
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

    def set_graph(self, which, csr, stream=None):
        csr = csr.tocsr()
        csr.sort_indices()
        ip = np.ascontiguousarray(csr.indptr, dtype=np.int32)
        ix = np.ascontiguousarray(csr.indices, dtype=np.int32)
        vv = np.ascontiguousarray(csr.data, dtype=np.float32)
        _lib.check(self._lib.tgb200_set_graph(self._h, which, _lib.ptr(ip), _lib.ptr(ix), _lib.ptr(vv), len(vv),
                                              self._s(stream)))

    def set_mapping(self, M0, stream=None):
        _lib.check(self._lib.tgb200_set_mapping(self._h, _lib.ptr(M0), self._s(stream)))

    def init_mapping_normal(self, seed, stream=None, first_row=0):
        _lib.check(self._lib.tgb200_init_mapping_normal_rows(self._h, seed, first_row, self._s(stream)))

    def init_mapping_legacy(self, state, skip=0, first_row=0, end_normal=None, stream=None):
        """The reference draw np.random.normal(0, 1, ...) from the numpy generator state `state` (get_state() tuple):
        rows [first_row, first_row + n_cells) of a draw that starts `skip` normals into the stream.  Returns (the state
        after end_normal normals, default the end of these rows; values recomputed on the host)."""
        from . import legacy_rng
        if end_normal is None:
            end_normal = skip + (first_row + self.cfg.n_cells) * self.cfg.n_voxels
        return legacy_rng.init_mapping(self._lib, self._h, state, skip, first_row, end_normal, self._s(stream))

    def run(self, n_steps, lr=0.1, stream=None):
        _lib.check(self._lib.tgb200_run(self._h, n_steps, lr, self._s(stream)))

    def step_begin(self, stream=None):
        _lib.check(self._lib.tgb200_step_begin(self._h, self._s(stream)))

    def step_end(self, lr=0.1, stream=None):
        _lib.check(self._lib.tgb200_step_end(self._h, lr, self._s(stream)))

    def comm_init(self, rank, world, broadcast):
        """Own NCCL communicator for the cell-sharded tgb200_run: rank 0 creates the 128-byte id (tgb200_comm_unique_id),
        `broadcast(uint8 ndarray) -> ndarray` carries it to every rank by any means, every rank joins."""
        uid = np.zeros(128, dtype=np.uint8)
        if rank == 0:
            _lib.check(self._lib.tgb200_comm_unique_id(_lib.ptr(uid), uid.nbytes))
        uid = np.ascontiguousarray(broadcast(uid), dtype=np.uint8)
        _lib.check(self._lib.tgb200_comm_init_rank(self._h, _lib.ptr(uid), rank, world))

    def set_comm(self, comm, rank, world):
        """Lend the handle an existing ncclComm_t (tangram_b200.sharded.nccl_comm_for_group); the caller keeps ownership."""
        _lib.check(self._lib.tgb200_set_comm(self._h, comm, rank, world))

    def exchange_tensor(self):
        import torch
        p, n = ctypes.c_void_p(), ctypes.c_int64()
        _lib.check(self._lib.tgb200_exchange_buffer(self._h, ctypes.byref(p), ctypes.byref(n)))

        class _Wrap:
            __cuda_array_interface__ = {"shape": (n.value,), "typestr": "<f4", "data": (p.value, False),
                                        "version": 3, "strides": None}
        return torch.as_tensor(_Wrap(), device=f"cuda:{self.cfg.device}")

    def history(self):
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_history_len(self._h, ctypes.byref(n)))
        out = np.empty((n.value, _lib.HIST_COLS), dtype=np.float32)
        if n.value:
            _lib.check(self._lib.tgb200_get_history(self._h, 0, n.value, _lib.ptr(out), None))
        return out

    def get_mapping(self, out, stream=None):
        _lib.check(self._lib.tgb200_get_mapping(self._h, _lib.ptr(out), self._s(stream)))
        return out

    def project(self, X, out, stream=None):
        """out (voxels x n_cols, f32) = softmax(M)^T X; X is (cells x n_cols) f32, host or device memory."""
        n_cols = int(X.shape[1])
        _lib.check(self._lib.tgb200_project(self._h, _lib.ptr(X), n_cols, _lib.ptr(out), self._s(stream)))
        return out

    def get_state(self, M=None, m=None, v=None, stream=None):
        """Copy M / m / v (n_cells x n_voxels f32, host or device buffers; None skips) out of the handle; returns the step count."""
        step = ctypes.c_int64()
        _lib.check(self._lib.tgb200_get_state(self._h, _lib.ptr(M), _lib.ptr(m), _lib.ptr(v), ctypes.byref(step), self._s(stream)))
        return step.value

    def debug(self, name):
        """Internal device buffer by name (tgb200_debug_buffer) as a host array."""
        n = ctypes.c_int64()
        _lib.check(self._lib.tgb200_debug_buffer(self._h, name.encode(), None, 0, ctypes.byref(n)))
        out = np.empty(max(n.value, 4), dtype=np.float32)
        _lib.check(self._lib.tgb200_debug_buffer(self._h, name.encode(), _lib.ptr(out), out.size, ctypes.byref(n)))
        return out[:n.value]

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
