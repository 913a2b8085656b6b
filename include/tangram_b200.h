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
  /* _val_loss_fn (:311-356) of the mapping AFTER that epoch's update, on the rows tgb200_set_validation selects; NaN on the
   * other rows while validation is on, 0 on every row while it is off */
  TGB200_HIST_VAL_TOTAL = 12,      /* val_total_loss               :328 */
  TGB200_HIST_VAL_GENE_SIM = 13,   /* val_gene_sim                 :326 */
  TGB200_HIST_VAL_SPARSITY = 14,   /* val_sp_sparsity_weighted_sim :329-331 */
  TGB200_HIST_VAL_ENTROPY = 15,    /* val_entropy                  :333 */
  TGB200_HIST_COLS = 16
};

/* Replaces the keyword arguments of Mapper.__init__ (mapping_optimizer.py:19-45). */
typedef struct tgb200_config {
  int32_t struct_size;     /* = sizeof(tgb200_config); ABI guard (the size without state_memory is accepted too) */
  int32_t device;          /* CUDA device ordinal                                             */
  int32_t n_cells;         /* rows of M / S held by THIS handle (S.shape[0], :150)            */
  int32_t n_voxels;        /* G.shape[0]                                                      */
  int32_t n_genes;         /* training genes (S.shape[1] == G.shape[1])                       */
  int32_t n_types;         /* ct_encode.shape[1], 0 if unused (:134-136)                      */
  int64_t n_cells_global;  /* total cells over all ranks (== n_cells when not sharded; <= 0: n_cells; below n_cells: invalid) */
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
  int32_t state_memory;    /* tgb200_state_memory: where M and Adam's moments live (0: on the device) */
} tgb200_config;

/* Placement of the optimizer state M, m (bf16 mode: mb) and v.  TGB200_STATE_HOST keeps them in pinned host memory
 * (cudaHostAlloc).  Every pass that reads or writes them -- the row pass (also that of get_mapping, the projection and the
 * validation) and the streaming update in both modes -- walks them in row blocks through a ring of two device slots: the
 * copy-in of block b+1 and the copy-out of block b-1 run on the copy engines while block b's kernel runs, and in bf16 mode
 * the blocks nest inside the cell chunks of the pipeline.  The slots are sized from free device memory (at most 128 MiB in
 * all; the environment variable TGB200_STATE_BLOCK_ROWS sets the rows per block).  The draws, the zeroing and the state
 * get / set reach the host state directly.  The device then holds about 4 B per mapping element in bf16 mode and 10 B in
 * bf16x3 mode (the contraction operands) instead of 14 B and 22 B; the host holds 10 B (bf16) or 12 B (bf16x3).  The
 * kernels run their resident arithmetic on the staged rows, so results are bit-identical to TGB200_STATE_DEVICE.  fp32
 * mode fuses Adam into its FFMA contraction's epilogue and is refused with TGB200_ERR_UNSUPPORTED.
 * TGB200_STATE_AUTO keeps as many rows on the device as fit and only the rest in host memory: tgb200_create plans the
 * split with tgb200_plan_state on the device's free memory.  When every row fits, the handle is a TGB200_STATE_DEVICE
 * handle (same allocations, kernels and launches; no pinned memory, ring or copy streams).  Otherwise rows [0, R) of M,
 * m / mb and v live in device memory and rows [R, N) in pinned host memory; every pass over a row range launches its
 * resident rows directly, in pieces between the staged blocks, so the ring's copies run under the resident rows' kernels.
 * The environment variable TGB200_STATE_RESIDENT_ROWS forces R.  Results are bit-identical to the other placements;
 * fp32 is refused as for TGB200_STATE_HOST. */
typedef enum tgb200_state_memory {
  TGB200_STATE_DEVICE = 0,
  TGB200_STATE_HOST = 1,
  TGB200_STATE_AUTO = 2
} tgb200_state_memory;

/* Where a handle of `cfg` would keep its state given `device_free` bytes of free device memory: pure arithmetic, no
 * allocation and no device needed (tgb200_create uses it with cudaMemGetInfo).  device_bytes bounds what tgb200_create
 * allocates on the device (the operands, rows [0, R) of the state and the ring, each allocation rounded up to 2 MiB);
 * reserve_bytes is what the handle keeps free for what it allocates later (validation scratch, the CSR graphs, the
 * history, get_mapping's and the projection's blocks, the legacy draw's scratch, CUDA's loading of the kernels).
 * TGB200_STATE_AUTO picks the largest R with device_bytes + reserve_bytes <= device_free, R = N when every row fits;
 * TGB200_STATE_BLOCK_ROWS and TGB200_STATE_RESIDENT_ROWS override the block rows and R as they do in tgb200_create.
 * TGB200_STATE_DEVICE plans R = N, TGB200_STATE_HOST R = 0.  fp32 with host or auto state: TGB200_ERR_UNSUPPORTED. */
typedef struct tgb200_state_plan {
  int32_t resident_rows;   /* R: rows [0, R) of M, m / mb and v on the device */
  int32_t block_rows;      /* rows per ring slot (0: no ring) */
  int64_t device_bytes;    /* device memory tgb200_create allocates */
  int64_t reserve_bytes;   /* device memory left free for later allocations */
  int64_t host_bytes;      /* pinned host memory for rows [R, N) */
} tgb200_state_plan;
TGB200_API int tgb200_plan_state(const tgb200_config* cfg, uint64_t device_free, tgb200_state_plan* out);

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

/* State of numpy's legacy generator, as np.random.get_state() returns it:
 * ('MT19937', key[624], pos, has_gauss, cached_gaussian). */
typedef struct tgb200_mt_state {
  uint32_t key[624];
  int32_t pos;          /* 0 .. 624 */
  int32_t has_gauss;    /* 0 or 1 */
  double gauss;
} tgb200_mt_state;

/* The reference's initial draw on the device, bit for bit: M = float32(np.random.normal(0, 1, (n_rows, n_voxels))) after
 * np.random.seed (:147-157), from the generator state `start`.  The handle receives rows [first_row, first_row + n_cells)
 * of a draw that begins `skip` normals into the stream (MapperConstrained discards a first draw of N x V: skip = N V,
 * :472-493); pad columns are zero.  `end_out` (may be NULL) receives the generator state after `end_normal` normals of the
 * stream, as numpy leaves it after the host draw (end_normal >= skip + (first_row + n_cells) n_voxels).  The few values
 * whose float32 rounding could depend on the last bit of log are recomputed on the host with libm's log, as numpy does;
 * *n_fixed_out (may be NULL) is their number.  Resets the Adam state like tgb200_set_mapping.  Synchronous. */
TGB200_API int tgb200_init_mapping_legacy(tgb200_mapper* h, const tgb200_mt_state* start, int64_t skip, int64_t first_row,
                                          int64_t end_normal, tgb200_mt_state* end_out, int64_t* n_fixed_out, void* stream);
/* Host only, no device: the state after n_words more 32-bit words (numpy's state after random_raw(n_words)); has_gauss and
 * gauss are copied.  tgb200_mt19937_jump_pow2 jumps by 2^log2_words words, log2_words <= 128. */
TGB200_API int tgb200_mt19937_jump(const tgb200_mt_state* in, uint64_t n_words, tgb200_mt_state* out);
TGB200_API int tgb200_mt19937_jump_pow2(const tgb200_mt_state* in, uint32_t log2_words, tgb200_mt_state* out);

/* A fresh optimizer on the current mapping: what every Mapper.train call does when it builds torch.optim.Adam([M])
 * anew (:373, :607) -- zero moments, bias correction restarts at t = 1.  M, F, the history and its length are kept. */
TGB200_API int tgb200_reset_adam(tgb200_mapper* h, void* stream);

/* Restrict the loss to a subset of the n_genes training columns (the reference builds the Mapper on S[:, train_genes],
 * mapping_utils.py:246-275, once per cross-validation fold, utils.py:580-600).  `active`: n_genes bytes (0/1), host;
 * NULL = all genes (the default; an all-ones mask is the same).  The handle then computes what a handle created on
 * S[:, active], G[:, active] computes from the same mapping: every cosine term (gene-voxel, voxel-gene, neighbourhood,
 * Getis-Ord), its history columns and tgb200_validation_terms run over the active genes, and dL/dY is exactly 0 on the
 * other gene columns.  Density, entropy, L1/L2, cell-type islands and the filter are unaffected.  The mapping, the
 * filter, the Adam state and the history are kept.  A sharded handle needs the same mask on every rank.
 * TGB200_ERR_INVALID when no gene is active or a byte is not 0/1; TGB200_ERR_STATE between step_begin and step_end. */
TGB200_API int tgb200_set_loss_genes(tgb200_mapper* h, const uint8_t* active, void* stream);

/* Mapper.train(val_each=every) (:398-403) without leaving the device: while `every` > 0, tgb200_run and step_begin /
 * step_end validate epoch e -- counted from this call, from 0 -- when e % every == 0, and write _val_loss_fn's four values
 * (:311-356: on the training matrices, over the genes of the loss mask) into history columns TGB200_HIST_VAL_* of that
 * epoch's row.  Values are those of tgb200_validation_terms after the epoch's update, bit for bit.  fp32 / bf16x3: the next
 * iteration of the same tgb200_run call computes the validation from its own forward (identical: same row pass, same
 * contraction); the last iteration of a call and constrained mode run tgb200_validation_terms' forward.  bf16 mode: that
 * exact row pass and forward once per validated epoch, which the next iteration then starts from, as after
 * tgb200_validation_terms.  No allocation and no host sync in the loop.
 * A sharded handle (n_cells_global != n_cells) validates the global mapping when it has a communicator (tgb200_comm_init_rank
 * / tgb200_set_comm): the four values are _val_loss_fn's over all n_cells_global cells, bit-identical on every rank.  The
 * forward that serves a validation inside tgb200_run carries sum_i h_i in exchange tail slot [5]; the separate forward
 * sums [Y_ext | tail] over the ranks with one more all-reduce on the handle's communicator, in the exchange buffer.
 * every = 0 (the default) turns validation off.  TGB200_ERR_STATE between step_begin and step_end; every > 0 on a sharded
 * handle without a communicator, or on a sharded constrained handle, is TGB200_ERR_UNSUPPORTED.  Allocates the
 * validation's scratch (about 8 (Ke + V) bytes, more when lambda_g2 == 0) on first use; queues no work on `stream`. */
TGB200_API int tgb200_set_validation(tgb200_mapper* h, int32_t every, void* stream);

/* Constrained mode: initial filter logits F0 (n_cells, host or device; the reference draws them at :490).
 * Resets the filter's Adam state. */
TGB200_API int tgb200_set_filter(tgb200_mapper* h, const float* F0, void* stream);
/* Filter logits F and/or sigmoid(F) (n_cells each, host or device; NULL to skip).  Replaces :638. */
TGB200_API int tgb200_get_filter(tgb200_mapper* h, float* F_out, float* f_out, void* stream);

/* ---- the hot loop ------------------------------------------------------------------ */

/* Mapper.train's loop body x n_steps (:382-396): loss, backward, Adam, and the validation of the epochs
 * tgb200_set_validation selects (:398-403).  No host syncs; per-epoch scalars go to a device-side history buffer. */
TGB200_API int tgb200_run(tgb200_mapper* h, int32_t n_steps, float learning_rate, void* stream);

/* Cell-sharded operation (one handle per rank): step_begin computes this rank's partial
 * sums; the caller all-reduces (sum) the exchange buffer across ranks (NCCL); step_end
 * finishes the iteration.  tgb200_run == step_begin + step_end when not sharded, and step_begin + NCCL all-reduce +
 * step_end on a sharded handle that has a communicator (below).
 * A handle is sharded when n_cells_global != n_cells, in plain and in constrained mode alike (a sharded constrained handle
 * needs target_count > 0).  The exchange buffer holds n_voxels x Ke floats of Y_ext = P^T S_ext over this rank's cells
 * (gene columns, two density columns, cell-type columns; Ke = n_genes + 2 + n_types rounded up to 64), then an 8-float
 * tail of row sums: [0] the per-row entropy terms (when lambda_r != 0), [1] sum |M| and [2] sum M^2 (the L1 / L2 terms),
 * [3] sum f and [4] sum (f - f^2) (constrained mode), [5] sum_i h_i on an iteration whose forward serves a pending
 * validation (tgb200_set_validation) and zero otherwise, [6..7] zero.  On a sharded handle an iteration that serves no
 * validation writes every slot no row term needs as zero, also right after a validated one.  In constrained mode the operand is f o S_ext
 * (f = sigmoid(F) of this rank's cells), so the density columns already hold the f-weighted column sums, and after the sum
 * [3] / [4] are the filter's global count and regulariser; every scalar of the filter update (lambda_d sum d / sum f,
 * sign(sum f - target_count)) is derived from the summed buffer, so each rank updates its own F entries with global
 * coefficients.  A constrained handle runs each iteration on one stream, so the filter update of iteration t is ordered
 * before the filter refresh (sigmoid(F), f o S_ext) and the exchange of iteration t + 1, in tgb200_run as in a
 * caller-driven loop. */
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
 *                           detach or destroy the handle before destroying that communicator.  Detaching while a sharded
 *                           handle validates (tgb200_set_validation(every > 0)) is TGB200_ERR_STATE
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
/* _val_loss_fn (:311-356) of the current mapping: out[4] = expression_sim, gv_sim, sp_sparsity_weighted_gv_sim, entropy
 * (HOST).  One forward on the device and one 16-byte copy, the forward and kernels tgb200_set_validation runs in the loop
 * (so the values are those bit for bit); allocates the same scratch on first use.  Synchronous on `stream`.
 * On a sharded handle with a communicator this is a collective: every rank calls it, the forward's [Y_ext | tail] is
 * summed over the ranks on the handle's communicator, and every rank gets the same four values of the global mapping.
 * TGB200_ERR_STATE between step_begin and step_end; TGB200_ERR_UNSUPPORTED on a sharded handle without a communicator
 * and on a sharded constrained handle. */
TGB200_API int tgb200_validation_terms(tgb200_mapper* h, float* out4_host, void* stream);
/* project_genes' GEMM (tangram/utils.py:368): out (n_voxels x n_cols, host or device) = softmax(M)^T X, X (n_cells x
 * n_cols) row-major f32, host or device.  tgb200_project_map's blocks and arithmetic, with each block's mapping rows
 * written as bf16 planes by the row pass (no copy of the mapping): the result equals tgb200_project_map on the
 * tgb200_get_mapping of the same M, bit for bit, in every precision.  Writes the row statistics as tgb200_get_mapping does;
 * training continues unperturbed.  Device memory: out plus two blocks of staging (see tgb200_project_map).  Synchronous. */
TGB200_API int tgb200_project(tgb200_mapper* h, const float* X, int64_t n_cols, float* out, void* stream);

/* Run-to-run agreement of R equally shaped arrays (the hyper-parameter tuner's metrics,
 * tangram/mapping_parameter_tuning.py:42-82), in one streaming pass that reads every element once and allocates
 * O(rows) scratch.  `arrays`: a HOST array of R DEVICE pointers (all on `device`), each rows x cols row-major f32 with
 * leading dimension ld; 1 <= R <= 8.
 *   pearson_out            R(R-1)/2 doubles (host or device; NULL to skip): np.corrcoef of the flattened arrays at
 *                          np.tril_indices(R, -1), i.e. pearson_corr (:42-53); sums in fp64, reduced in a fixed order
 *   vote_entropy_out       rows floats (host or device; NULL to skip): per row, the entropy of the R runs' argmax votes
 *                          over log(cols), vote_entropy (:55-69).  The argmax is np.argmax's: first column on ties, a
 *                          NaN counting as the maximum (the first NaN wins), column 0 for a row that is -inf throughout
 *   consensus_entropy_out  rows floats (host or device; NULL to skip): per row, the entropy of p / sum(p) with
 *                          p = mean over runs, over log(cols), consensus_entropy (:71-82); NaN where p holds a NaN or
 *                          an infinity, or sums to 0
 *   With cols == 1 both entropies are NaN on every row, as the reference's division by log(1) = 0 gives.
 * Fails with TGB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  Bit-reproducible on a given device.
 * Synchronous on `stream`. */
TGB200_API int tgb200_agreement(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                double* pearson_out, float* vote_entropy_out, float* consensus_entropy_out,
                                int32_t device, void* stream);

/* tgb200_agreement's Pearson pass split around sums over row shards, for a mapping cube whose rows are spread over
 * several devices or processes (the sharded tuner trial).  Each shard passes its own rows as tgb200_agreement takes
 * them (same `arrays`, R, rows, cols, ld and checks); the caller sums the outputs over the shards (an all-reduce), which
 * these entry points never do themselves.  In order:
 *   tgb200_agreement_sample    sample_out (R + 1 doubles, host or device): the sums of the shard's shift sample of each
 *                              array (min(rows cols, 4096) elements spread evenly over its rows), then the sample size.
 *                              Summed over the shards, shift[r] = sum[r] / size is the same on every shard and near the
 *                              global mean, so that the one-pass cross products keep the accuracy of a centred sum.
 *   tgb200_agreement_partials  `shift` (R doubles, host or device): that shared shift.  sums_out (R + R(R+1)/2
 *                              doubles, host or device): sum dx_r, then sum dx_r dx_s for r <= s (row-major upper
 *                              triangle), dx_r = x_r - shift[r], over the shard's elements in fp64, its per-block partials
 *                              added in block order.  vote_entropy_out / consensus_entropy_out (rows floats, host or
 *                              device; NULL to skip): the shard's rows of tgb200_agreement's per-row entropies, bit for bit.
 *   tgb200_agreement_pearson   sums (R + R(R+1)/2 doubles, host or device): the partials summed over the shards;
 *                              rows_global x cols: the element count of one whole array.  pearson_out (R(R-1)/2 doubles,
 *                              host or device): np.corrcoef at np.tril_indices(R, -1); nothing is written for R = 1.
 * One shard holding every row gives tgb200_agreement's Pearson bits.  Scratch is O(R^2 grid + rows) as there; nothing of
 * size rows x cols.  TGB200_ERR_INVALID for a null argument, R outside 1..8 or a bad shape; TGB200_ERR_NO_DEVICE without
 * an sm_90 device.  Synchronous on `stream`. */
TGB200_API int tgb200_agreement_sample(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                       double* sample_out, int32_t device, void* stream);
TGB200_API int tgb200_agreement_partials(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                         const double* shift, double* sums_out, float* vote_entropy_out,
                                         float* consensus_entropy_out, int32_t device, void* stream);
TGB200_API int tgb200_agreement_pearson(const double* sums, int32_t R, int64_t rows_global, int64_t cols,
                                        double* pearson_out, int32_t device, void* stream);

/* Annotation transfer from cells onto space (tangram/utils.py:126-153 project_cell_annotations, 205-285
 * count_cell_annotations, 820-842 cell_type_mapping), in one streaming pass over a DEVICE mapping `map` (rows x cols
 * row-major f32, leading dimension ld >= cols, on `device`).  `labels_host`: a HOST array of `rows` int32 labels in
 * [-1, n_labels); a row labelled -1 adds to no sum and gets no argmax.
 *   sums_out    n_labels x cols doubles (host or device; NULL to skip): sums_out[t, j] = sum of map[i, j] over the rows
 *               labelled t, in fp64 (the reference's int64 one-hot GEMM runs in float64); 0 for a label without rows
 *   argmax_out  rows int32 (host or device; NULL to skip): per labelled row the first column holding its maximum, a NaN
 *               counting as the maximum (np.argmax); -1 for unlabelled rows
 * No atomics, partials reduced in a fixed order: bit-reproducible.  Scratch is about 8 (rows / 128 + n_labels) cols bytes
 * for the sums and 8 rows ceil(cols / 1024) bytes for the argmax.  Fails with TGB200_ERR_INVALID (and a message in
 * tgb200_last_error) for a label outside [-1, n_labels) or ld < cols, and with TGB200_ERR_NO_DEVICE without an sm_90
 * device (no CPU fallback).  Synchronous on `stream`. */
TGB200_API int tgb200_annotate(const float* map, int64_t rows, int64_t cols, int64_t ld,
                               const int32_t* labels_host, int32_t n_labels,
                               double* sums_out, int32_t* argmax_out, int32_t device, void* stream);

/* project_genes' GEMM from any mapping (tangram/utils.py:366-368: `adata_map.X.T @ adata_sc.X` on the host, after densifying
 * a sparse adata_sc.X), with no handle: out[j, k] = sum_i map[i, j] X[i, k].
 *   map      rows x cols probabilities, row-major f32, leading dimension ld >= cols (host or device)
 *   X        dense rows x n_genes, row-major f32, leading dimension x_ld >= n_genes (host or device), or NULL for CSR:
 *   indptr   rows + 1 int64 offsets from 0 to nnz, non-decreasing (host or device)
 *   indices  nnz int32 columns in [0, n_genes), strictly increasing within a row (host or device)
 *   data     nnz f32 values (host or device)
 *   out      cols x n_genes f32 (host or device)
 *   block_rows  cells staged per block, a multiple of 2048; 0 = about an eighth of the cells, less if free memory needs it
 * Three bf16 planes per operand, six partial products on the tensor cores; accumulation chains of 512 cells, added in cell
 * order in fp32 (round-to-nearest); no atomics.  The result does not depend on how the data is staged: dense or CSR X,
 * host or device pointers and any block size give identical bits.
 * Cell blocks of the mapping and X are double-buffered (the copies of block b + 1 run on a second stream while block b
 * contracts); device memory is out plus two blocks of staging, whatever `rows` is.  A CSR block is turned into the bf16
 * planes directly, one warp per row.  TGB200_ERR_INVALID for bad shapes, a malformed indptr, a column index outside
 * [0, n_genes) or out of order (such entries are skipped, never written), or when free device memory cannot hold out and
 * one block of 2048 cells (the message gives the sizes); TGB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).
 * Synchronous on `stream`. */
TGB200_API int tgb200_project_map(const float* map, int64_t rows, int64_t cols, int64_t ld, const float* X, int64_t x_ld,
                                  const int64_t* indptr, const int32_t* indices, const float* data, int64_t nnz,
                                  int64_t n_genes, float* out, int64_t block_rows, int32_t device, void* stream);

/* Per-label column statistics of an expression matrix (scanpy's rank_genes_groups basic stats), one pass.
 *   X        dense rows x n_genes, row-major f32, leading dimension x_ld >= n_genes (host or device), or NULL for CSR:
 *   indptr / indices / data / nnz   canonical CSR as tgb200_project_map takes it (host or device)
 *   labels_host  rows int32 in [-1, n_labels) (HOST); -1 rows add to nothing
 *   sum_out, sumsq_out   n_labels x n_genes doubles (host or device): sum of x and of (double)x*(double)x
 *   nnz_out              n_labels x n_genes int64 (host or device; NULL to skip): entries with x != 0 (NaN counts)
 *   block_rows           cells staged per block, a multiple of 2048; 0 = sized from free device memory
 * Order of additions, for label t and gene k: the rows of each aligned range [2048c, 2048c + 2048) labelled t are summed
 * in fp64 in row order from 0.0 (one chain per range), and the chains are added in order of c from 0.0.  Absent CSR
 * entries and explicit zeros add +0.0, so dense and CSR input of the same matrix, host and device pointers, any block_rows
 * and re-runs give identical bits; no atomics.  Dense X in this device's memory is read in place; host X (dense or CSR)
 * and CSR from anywhere are staged in double-buffered cell blocks.  Device memory: the outputs, two blocks of staging and
 * the partials of one block's (range, label) runs (20 n_genes bytes each), independent of `rows`.
 * TGB200_ERR_INVALID for a bad shape, a malformed indptr, a column outside [0, n_genes) or out of order within its row, a
 * label outside [-1, n_labels), block_rows not a multiple of 2048, or when free device memory cannot hold one block (the
 * message gives the sizes); TGB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  Synchronous on `stream`. */
TGB200_API int tgb200_group_stats(const float* X, int64_t x_ld, const int64_t* indptr, const int32_t* indices,
                                  const float* data, int64_t nnz, int64_t rows, int64_t n_genes,
                                  const int32_t* labels_host, int32_t n_labels, double* sum_out, double* sumsq_out,
                                  int64_t* nnz_out, int64_t block_rows, int32_t device, void* stream);

/* tgb200_group_stats of y = expm1(scale * (double)x) instead of x (scanpy's highly_variable_genes, flavor="seurat":
 * the statistics of the un-logged expression; scale = ln(base) for log1p data with uns["log1p"]["base"], else 1).
 *   sum_out, sumsq_out   the fp64 sum of y and of y * y (y * y added with one fused multiply-add, whatever -fmad says)
 *   nnz_out              entries with x != 0, of the untransformed x (NaN counts), as tgb200_group_stats
 * y is computed in fp64 for every element, absent CSR entries included (expm1(+-0) = +-0 adds nothing), with the same
 * order of additions, staging, memory and checks as tgb200_group_stats: dense and CSR, host and device pointers, any
 * block_rows and re-runs give identical bits.  fp64 expm1 stays finite where scanpy's float32 expm1 overflows (x above
 * about 88.7).  TGB200_ERR_INVALID also for a scale that is not finite. */
TGB200_API int tgb200_group_stats_expm1(const float* X, int64_t x_ld, const int64_t* indptr, const int32_t* indices,
                                        const float* data, int64_t nnz, int64_t rows, int64_t n_genes,
                                        const int32_t* labels_host, int32_t n_labels, double* sum_out, double* sumsq_out,
                                        int64_t* nnz_out, int64_t block_rows, int32_t device, void* stream,
                                        double scale);

/* Spatial neighbour graph (squidpy's gr.spatial_neighbors), exact, in fp64, over a uniform cell grid on the device.
 *   coords   n x dim fp64, row-major, dim 2 or 3, finite (host or device); n fits int32
 * d(i, j) = sqrt((dx*dx + dy*dy) + dz*dz) with dx = x_j - x_i, each operation rounded on its own (no FMA): bit-identical
 * to numpy's np.sqrt(((C[j] - C[i]) ** 2).sum()).  A point is excluded from its own row by index only, so coincident
 * points are neighbours at distance 0.  Both calls are synchronous on `stream`; TGB200_ERR_INVALID for bad arguments, a
 * coordinate that is not finite, or data that cannot fit in free device memory (the message gives the sizes);
 * TGB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).
 *
 * tgb200_spatial_knn: the k nearest j != i of every point, ranked by (d, j) (ties go to the smaller index), 1 <= k <= 64
 * and k < n.  indices_out / dist_out: n x k int32 / fp64 (host or device); row i lists its k neighbours in increasing
 * column order, so it is row i of a canonical CSR with indptr = k * arange(n + 1).
 *
 * tgb200_spatial_radius: every j != i with d <= radius (finite, >= 0).  indptr_out: n + 1 int64 (host or device), always
 * written.  When 0 < indptr_out[n] <= capacity, indices_out / dist_out (int32 / fp64, host or device) receive the rows,
 * each in search order (not sorted); otherwise they are untouched.  So a caller passes capacity 0 to learn the size and
 * calls again with buffers of indptr_out[n]; both calls give the same indptr. */
TGB200_API int tgb200_spatial_knn(const double* coords, int64_t n, int32_t dim, int32_t k, int32_t* indices_out,
                                  double* dist_out, int32_t device, void* stream);
TGB200_API int tgb200_spatial_radius(const double* coords, int64_t n, int32_t dim, double radius, int64_t* indptr_out,
                                     int32_t* indices_out, double* dist_out, int64_t capacity, int32_t device,
                                     void* stream);

/* Checkpoint / resume (the reference stubs this: `raise NotImplemented`, :151-153).
 * Any pointer may be NULL to skip it.  M, m, v: n_cells x n_voxels f32, host or device. */
TGB200_API int tgb200_get_state(tgb200_mapper* h, float* M, float* m, float* v, int64_t* step, void* stream);
TGB200_API int tgb200_set_state(tgb200_mapper* h, const float* M, const float* m, const float* v, int64_t step, void* stream);

/* ---- introspection ----------------------------------------------------------------- */

/* Rows [0, *out) of M, m / mb and v are in device memory, the rest in pinned host memory (n_cells: device state). */
TGB200_API int tgb200_resident_rows(tgb200_mapper* h, int32_t* out);
/* Kernels launched by this handle since creation (for bench.py's gpu_launches). */
TGB200_API int tgb200_kernel_launches(tgb200_mapper* h, int64_t* n);
/* Runs ONE full iteration with CUDA events around each kernel on `stream`;
 * fills names[i] (static strings) / ms[i] for up to `cap` kernels, *n = count. */
TGB200_API int tgb200_profile_step(tgb200_mapper* h, float learning_rate, void* stream,
                                   const char** names, float* ms, int32_t cap, int32_t* n);
/* Algorithmic bytes and flops of one iteration for this handle's shape (DESIGN.md). */
TGB200_API int tgb200_algorithmic_cost(tgb200_mapper* h, double* hbm_bytes, double* flops);

/* Diagnostics: copy an internal device buffer to HOST memory after a step.  name: "Y" (V x Ke),
 * "dY" (V x Ke), "rdot" (n_cells), "Sx" (n_cells x Ke), "shape" (Ke, ld, fwd_splits, r_parts,
 * cell chunks of the bf16 pipeline),
 * "M", "m", "v" (n_cells x ld, the Adam state, pad columns included), "stats" (n_cells x 4: RowStat mx, inv_z,
 * log_z, h); fp32 mode: "Pf" (n_cells x ld, P of the last row pass); bf16x3 mode: "Pb" (n_cells x ld, the three
 * P planes summed), "dpf" (n_cells x ld, the backward's fp32 dP); bf16 mode only: "Pb" (n_cells x ld, the resident
 * unnormalised P the next backward consumes), "dq" (n_cells x ld, the backward's centred dP), "rcenter" (n_cells, the
 * centre dq is stored relative to), "rowc" (n_cells x 4: lse, r', h, 0 of the last update), "zsum", "inv_zt", "lseA"
 * (the offset Pb was written with: after step_end, the exact log-sum-exp of the rows before that update), "lseT" (after
 * step_begin, the exact log-sum-exp of the current rows; after step_end, free), and "pxsum", "l1sum", "l2sum" (n_cells,
 * the update's row sums, when the entropy or L1/L2 terms are on); bf16 buffers (the first moment included) widened to float.
 * "legacy_init": the last tgb200_init_mapping_legacy's ms of jump, count + scan, emit and fix-up (CUDA events), ms of host
 * polynomial work, draw blocks, values recomputed on the host, values that recomputation changed.
 * out_host may be NULL to query the size (*n). */
TGB200_API int tgb200_debug_buffer(tgb200_mapper* h, const char* name, float* out_host, int64_t cap, int64_t* n);

/* Diagnostics: enable != 0 starts recording a CUDA event after every launch on the stream it went to; enable == 0 stops
 * and returns, per launch, its name, stream and completion time in ms relative to the first one -- the only way to see
 * the bf16 chunk pipeline without a tracer.  Streams 1-3 exist only on a bf16 handle with several cell chunks:
 *   0  the caller's stream (every launch of any other handle, and of tgb200_profile_step)
 *   1  the handle's contraction stream: forward, loss stage, backward contractions
 *   2  its update stream: row-dot finalize and the streaming Adam kernel
 *   3  the stream on which tgb200_run issues the next iteration's forward chunks during the backward */
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
