/*
 * tangram_b200 -- C-ABI of the H100-native (sm_90a) `map_cells_to_space` hot path.
 *
 * This is the drop-in boundary for ONE path of broadinstitute/Tangram: the optimizer in
 * tangram/mapping_optimizer.py (class Mapper).  Each entry point cites the reference
 * interface it replaces (file:line in the reference tree).  The library is plain C ABI:
 * opaque handle, raw pointers and sizes, int status codes, no C++ / torch types, no
 * exceptions, no exit().  Pointer arguments documented "host or device" are copied with
 * cudaMemcpyDefault (UVA), mirroring the reference, which copies every input
 * (`torch.tensor(ndarray)`, mapping_optimizer.py:83-157).
 *
 * Every function returns 0 on success or a negative tgb200_status; the message for the
 * calling thread's last failure is available from tgb200_last_error().
 *
 * `stream` arguments are `cudaStream_t` passed as void* (NULL = legacy default stream).
 */
#ifndef TANGRAM_B200_H_
#define TANGRAM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define TGB200_API __attribute__((visibility("default")))
#else
#define TGB200_API
#endif

typedef struct tgb200_mapper tgb200_mapper; /* opaque; replaces a `Mapper` instance */

typedef enum tgb200_status {
  TGB200_OK = 0,
  TGB200_ERR_INVALID = -1,   /* bad argument / bad config                              */
  TGB200_ERR_CUDA = -2,      /* CUDA runtime / driver error (message has the detail)   */
  TGB200_ERR_STATE = -3,     /* call order violated (e.g. run before set_expression)   */
  TGB200_ERR_UNSUPPORTED = -4, /* term outside the hot-path scope (Moran / Geary)      */
  TGB200_ERR_NO_DEVICE = -5  /* no sm_90 device: there is NO CPU fallback              */
} tgb200_status;

/* Arithmetic of the two contractions (softmax(M)^T S and S dY^T). */
typedef enum tgb200_precision {
  TGB200_PREC_FP32 = 0,  /* fp32 FFMA contraction: parity mode (reference is fp32, TF32 off) */
  TGB200_PREC_BF16 = 1,  /* bf16 operands on wgmma tensor cores, fp32 accumulate in registers */
  TGB200_PREC_BF16X3 = 2 /* parity mode on tensor cores: each fp32 operand = 3 bf16 planes, 6 partial products */
} tgb200_precision;

/* mapping_optimizer.py:212-221: which density term is active. */
typedef enum tgb200_density_mode {
  TGB200_DENSITY_NONE = 0,   /* d is None                       (:220-221)            */
  TGB200_DENSITY_CELLS = 1,  /* d_pred = log(P.sum(0)/N)        (:217)                */
  TGB200_DENSITY_SOURCE = 2  /* d_pred = log(d_source @ P)      (:215, clusters mode) */
} tgb200_density_mode;

/* Sparse V x V operators (CSR) that replace the reference's dense V x V matrices. */
typedef enum tgb200_graph {
  TGB200_GRAPH_VOXEL_WEIGHTS = 0,       /* Mapper(voxel_weights=)        :125-127, used :235-236 */
  TGB200_GRAPH_NEIGHBORHOOD_FILTER = 1, /* Mapper(neighborhood_filter=)  :130-132, used :244     */
  TGB200_GRAPH_SPATIAL_WEIGHTS = 2      /* Mapper(spatial_weights=)      :139-141, used :171     */
} tgb200_graph;

/* Columns of one history row (one row per epoch; loss BEFORE that epoch's update,
 * mapping_optimizer.py:383-392).  Terms whose lambda is 0 are NaN, as in the reference
 * (:208-263: x / lambda with lambda == 0). */
enum {
  TGB200_HIST_TOTAL = 0,   /* total_loss            :266-270 */
  TGB200_HIST_MAIN = 1,    /* main_loss  (gv/l_g1)  :208     */
  TGB200_HIST_VG = 2,      /* vg_reg                :209     */
  TGB200_HIST_KL = 3,      /* kl_reg                :219     */
  TGB200_HIST_ENTROPY = 4, /* entropy_reg           :225     */
  TGB200_HIST_L1 = 5,      /* l1_reg                :229     */
  TGB200_HIST_L2 = 6,      /* l2_reg                :231     */
  TGB200_HIST_NEIGHBORHOOD = 7, /* gv_neighborhood_sim :237  */
  TGB200_HIST_CT_ISLANDS = 8,   /* ct_island_penalty   :246  */
  TGB200_HIST_GETIS_ORD = 9,    /* getis_ord_sim       :257  */
  TGB200_HIST_COUNT = 10,       /* count_reg     (MapperConstrained :543) */
  TGB200_HIST_F_REG = 11,       /* lambda_f_reg  (MapperConstrained :544) */
  TGB200_HIST_COLS = 16
};

/* Replaces the keyword arguments of Mapper.__init__ (mapping_optimizer.py:19-45). */
typedef struct tgb200_config {
  int32_t struct_size;     /* = sizeof(tgb200_config); ABI guard                              */
  int32_t device;          /* CUDA device ordinal                                             */
  int32_t n_cells;         /* rows of M / S held by THIS handle (S.shape[0], :150)            */
  int32_t n_voxels;        /* G.shape[0]                                                      */
  int32_t n_genes;         /* training genes (S.shape[1] == G.shape[1])                       */
  int32_t n_types;         /* ct_encode.shape[1], 0 if unused (:134-136)                      */
  int64_t n_cells_global;  /* total cells over all ranks (== n_cells when not sharded)        */
  int32_t precision;       /* tgb200_precision                                                */
  int32_t density_mode;    /* tgb200_density_mode                                             */
  float lambda_g1;         /* :27  */
  float lambda_d;          /* :28  */
  float lambda_g2;         /* :29  */
  float lambda_r;          /* :30  */
  float lambda_l1;         /* :31  */
  float lambda_l2;         /* :32  */
  float lambda_neighborhood_g1; /* :33 */
  float lambda_ct_islands; /* :40  */
  float lambda_getis_ord;  /* :35  */
  float adam_beta1;        /* torch.optim.Adam defaults used at :373 -> 0.9   */
  float adam_beta2;        /* 0.999 */
  float adam_eps;          /* 1e-8  */
  /* MapperConstrained (mapping_optimizer.py:411-639): a per-cell sigmoid filter F is learned next to M */
  int32_t constrained;     /* 1 = constrained mode (then density_mode must be NONE or CELLS) */
  float lambda_count;      /* :426 */
  float lambda_f_reg;      /* :427 */
  float target_count;      /* :428, :480-483 */
} tgb200_config;

/* ---- lifetime -------------------------------------------------------------------- */

/* Mapper.__init__ (:19-157) minus the data: allocates device state for the given shape. */
TGB200_API int tgb200_create(const tgb200_config* cfg, tgb200_mapper** out);
TGB200_API int tgb200_destroy(tgb200_mapper* h);

/* ---- inputs (copied; caller keeps ownership) ---------------------------------------- */

/* S (n_cells x n_genes) and G (n_voxels x n_genes), row-major f32, host or device.
 * Replaces :83-92 (self.S / self.G / S_train / G_train). */
TGB200_API int tgb200_set_expression(tgb200_mapper* h, const float* S, const float* G, void* stream);
/* d (n_voxels) and optional d_source (n_cells), :114-120.  NULL = absent. */
TGB200_API int tgb200_set_density(tgb200_mapper* h, const float* d, const float* d_source, void* stream);
/* ct_encode (n_cells x n_types) one-hot, :134-136. */
TGB200_API int tgb200_set_ct_encode(tgb200_mapper* h, const float* ct_encode, void* stream);
/* One V x V operator as CSR with HOST pointers (int32 indptr[V+1], indices[nnz], f32 values[nnz]).
 * Replaces the dense matrices at :125-141 (built by tangram/spatial_weights.py:5-30). */
TGB200_API int tgb200_set_graph(tgb200_mapper* h, int which, const int32_t* indptr,
                                const int32_t* indices, const float* values, int64_t nnz, void* stream);

/* Initial mapping M0 (n_cells x n_voxels f32, host or device): the float32 cast of the
 * reference's host draw at :147-157.  Resets the Adam state and the step counter. */
TGB200_API int tgb200_set_mapping(tgb200_mapper* h, const float* M0, void* stream);
/* Device-side N(0,1) init (Philox) for throughput runs; NOT bit-compatible with :150. */
TGB200_API int tgb200_init_mapping_normal(tgb200_mapper* h, uint64_t seed, void* stream);
/* Same for a cell-sharded handle: `first_row` is the global index of this handle's first cell, so the draw of a
 * cell does not depend on how the cells are sharded over ranks (tgb200_init_mapping_normal == first_row 0). */
TGB200_API int tgb200_init_mapping_normal_rows(tgb200_mapper* h, uint64_t seed, int64_t first_row, void* stream);

/* A fresh optimizer on the current mapping: what every Mapper.train call does when it builds torch.optim.Adam([M])
 * anew (:373, :607) -- zero moments, bias correction restarts at t = 1.  M, F, the history and its length are kept. */
TGB200_API int tgb200_reset_adam(tgb200_mapper* h, void* stream);

/* Constrained mode: initial filter logits F0 (n_cells, host or device; the reference draws them at :490).
 * Resets the filter's Adam state. */
TGB200_API int tgb200_set_filter(tgb200_mapper* h, const float* F0, void* stream);
/* Filter logits F and/or sigmoid(F) (n_cells each, host or device; NULL to skip).  Replaces :638. */
TGB200_API int tgb200_get_filter(tgb200_mapper* h, float* F_out, float* f_out, void* stream);

/* ---- the hot loop ------------------------------------------------------------------ */

/* Mapper.train's loop body x n_steps (:382-396): loss, backward, Adam.  No host syncs;
 * per-epoch scalars go to a device-side history buffer. */
TGB200_API int tgb200_run(tgb200_mapper* h, int32_t n_steps, float learning_rate, void* stream);

/* Cell-sharded operation (one handle per rank): step_begin computes this rank's partial
 * sums; the caller all-reduces (sum) the exchange buffer across ranks (NCCL); step_end
 * finishes the iteration.  tgb200_run == step_begin + step_end when not sharded, and step_begin + NCCL all-reduce +
 * step_end on a sharded handle that has a communicator (below). */
TGB200_API int tgb200_step_begin(tgb200_mapper* h, void* stream);
TGB200_API int tgb200_exchange_buffer(tgb200_mapper* h, float** device_ptr, int64_t* n_floats);
TGB200_API int tgb200_step_end(tgb200_mapper* h, float learning_rate, void* stream);

/* Cell-sharded operation without the caller in the loop: give the handle the NCCL communicator of the ranks that share
 * the voxels (one rank per GPU, each holding a contiguous block of cells; n_cells_global = the total) and tgb200_run
 * issues the per-iteration exchange itself, on its own streams, overlapped with the update of the previous iteration.
 * The reference has no multi-device path at all (one torch.device, mapping_utils.py:310); this replaces a user-level
 * loop around Mapper.train.  NCCL is bound at run time (libnccl.so.2 via dlopen: the instance already loaded in the
 * process, e.g. PyTorch's, else the system one).
 *   tgb200_comm_unique_id   rank 0: 128 opaque bytes (ncclGetUniqueId) to hand to every rank by any means
 *   tgb200_comm_init_rank   every rank: ncclCommInitRank on the handle's device; the handle owns the communicator
 *   tgb200_set_comm         alternatively borrow an existing ncclComm_t (NULL detaches); the caller keeps ownership and must
 *                           detach or destroy the handle before destroying that communicator
 * When a communicator arrives the exchange buffer is moved into ncclMemAlloc memory and registered with it (ncclCommRegister,
 * NCCL >= 2.19; silently skipped otherwise), so that the in-place all-reduce runs as an in-switch NVLS reduction on user
 * buffers; pointers obtained earlier from tgb200_exchange_buffer are invalid afterwards. */
TGB200_API int tgb200_comm_unique_id(void* id_out_128_bytes, int64_t capacity);
TGB200_API int tgb200_comm_init_rank(tgb200_mapper* h, const void* unique_id_128_bytes, int32_t rank, int32_t world);
TGB200_API int tgb200_set_comm(tgb200_mapper* h, void* nccl_comm, int32_t rank, int32_t world);
/* A communicator that outlives handles (ncclCommInitRank on `device`; costs a second or more at 8 ranks): create it once per
 * process and group of ranks, lend it to every handle with tgb200_set_comm, destroy it when no handle uses it any more. */
TGB200_API int tgb200_comm_create(const void* unique_id_128_bytes, int32_t rank, int32_t world, int32_t device, void** comm_out);
TGB200_API int tgb200_comm_destroy(void* nccl_comm);

/* ---- outputs ----------------------------------------------------------------------- */

/* Number of epochs recorded so far. */
TGB200_API int tgb200_history_len(tgb200_mapper* h, int64_t* n);
/* Rows [first, first+count) of the history, TGB200_HIST_COLS floats each, to HOST memory.
 * Replaces the per-iteration .tolist() syncs at :208-263 / :390-392. */
TGB200_API int tgb200_get_history(tgb200_mapper* h, int64_t first, int64_t count, float* out_host, void* stream);
/* softmax(M, dim=1) as n_cells x n_voxels f32 (host or device).  Replaces :406-408. */
TGB200_API int tgb200_get_mapping(tgb200_mapper* h, float* out, void* stream);
/* _val_loss_fn (:311-356): out[4] = expression_sim, gv_sim, sp_sparsity_weighted_gv_sim, entropy (HOST). */
TGB200_API int tgb200_validation_terms(tgb200_mapper* h, float* out4_host, void* stream);
/* project_genes' GEMM (tangram/utils.py:368): out (n_voxels x n_cols) = softmax(M)^T X,
 * X (n_cells x n_cols) row-major f32, host or device; fp32 accumulate. */
TGB200_API int tgb200_project(tgb200_mapper* h, const float* X, int64_t n_cols, float* out, void* stream);

/* Checkpoint / resume (the reference stubs this: `raise NotImplemented`, :151-153).
 * Any pointer may be NULL to skip it.  M, m, v: n_cells x n_voxels f32, host or device. */
TGB200_API int tgb200_get_state(tgb200_mapper* h, float* M, float* m, float* v, int64_t* step, void* stream);
TGB200_API int tgb200_set_state(tgb200_mapper* h, const float* M, const float* m, const float* v, int64_t step, void* stream);

/* ---- introspection ----------------------------------------------------------------- */

/* Kernels launched by this handle since creation (for bench.py's gpu_launches). */
TGB200_API int tgb200_kernel_launches(tgb200_mapper* h, int64_t* n);
/* Runs ONE full iteration with CUDA events around each kernel on `stream`;
 * fills names[i] (static strings) / ms[i] for up to `cap` kernels, *n = count. */
TGB200_API int tgb200_profile_step(tgb200_mapper* h, float learning_rate, void* stream,
                                   const char** names, float* ms, int32_t cap, int32_t* n);
/* Algorithmic bytes and flops of one iteration for this handle's shape (DESIGN.md). */
TGB200_API int tgb200_algorithmic_cost(tgb200_mapper* h, double* hbm_bytes, double* flops);

/* Diagnostics: copy an internal device buffer to HOST memory after a step.  name: "Y" (V x Ke),
 * "dY" (V x Ke), "rdot" (n_cells), "Sx" (n_cells x Ke), "shape" (Ke, ld, fwd_splits, r_parts).
 * out_host may be NULL to query the size (*n). */
TGB200_API int tgb200_debug_buffer(tgb200_mapper* h, const char* name, float* out_host, int64_t cap, int64_t* n);

/* Diagnostics: enable != 0 starts recording a CUDA event after every launch on the stream it went to; enable == 0 stops
 * and returns, per launch, its name, stream (0 caller, 1 the handle's contraction stream, 2 its update stream) and
 * completion time in ms relative to the first one -- the only way to see the two-stream pipeline without a tracer. */
TGB200_API int tgb200_debug_timeline(tgb200_mapper* h, int32_t enable, const char** names, int32_t* streams, float* end_ms,
                                     int32_t cap, int32_t* n);

/* Host-binding helpers for the result of Mapper.train (softmax(M).cpu().numpy(), mapping_optimizer.py:406-408): fault in and
 * page-lock a caller-owned host buffer so that tgb200_get_mapping's device->host copy runs as one DMA at link speed.  Meant to
 * be called from a host thread WHILE the iterations run (the pages are touched by `threads` worker threads, then registered
 * with the CUDA driver on `device`); tgb200_host_unpin before the buffer is freed.  Both are optional: an unpinned buffer works, slower. */
TGB200_API int tgb200_host_pin(void* buf, int64_t bytes, int32_t threads, int32_t device);
TGB200_API int tgb200_host_unpin(void* buf);

TGB200_API const char* tgb200_last_error(void);
TGB200_API const char* tgb200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TANGRAM_B200_H_ */
