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
  int32_t struct_size;     /* = sizeof(tgb200_config); ABI guard                              */
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
 * epoch's row.  Values are those of tgb200_validation_terms after the epoch's update: bit for bit, except the sparsity-weighted
 * score, which is summed from the per-gene cosines in fp32 (tgb200_validation_terms recovers them from the loss
 * coefficients on the host).  fp32 / bf16x3: the next iteration of the same tgb200_run call computes the validation from its
 * own forward (identical: same row pass, same contraction); the last iteration of a call and constrained mode run one
 * separate forward.  bf16 mode: one exact row pass and forward per validated epoch, which -- as after
 * tgb200_validation_terms -- the next iteration then starts from.  No allocation and no host sync in the loop.
 * every = 0 (the default) turns validation off.  TGB200_ERR_STATE between step_begin and step_end; every > 0 on a sharded
 * handle is TGB200_ERR_UNSUPPORTED.  Allocates the validation's scratch (about 8 (Ke + V) bytes, more when lambda_g2 == 0) on first use;
 * queues no work on `stream`. */
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
 * [3] sum f and [4] sum (f - f^2) (constrained mode), [5..7] zero.  In constrained mode the operand is f o S_ext
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
/* _val_loss_fn (:311-356) of the current mapping: out[4] = expression_sim, gv_sim, sp_sparsity_weighted_gv_sim, entropy
 * (HOST).  Synchronous, with scratch allocated per call; tgb200_set_validation computes the same inside the loop. */
TGB200_API int tgb200_validation_terms(tgb200_mapper* h, float* out4_host, void* stream);
/* project_genes' GEMM (tangram/utils.py:368): out (n_voxels x n_cols) = softmax(M)^T X,
 * X (n_cells x n_cols) row-major f32, host or device; fp32 accumulate. */
TGB200_API int tgb200_project(tgb200_mapper* h, const float* X, int64_t n_cols, float* out, void* stream);

/* Run-to-run agreement of R equally shaped arrays (the hyper-parameter tuner's metrics,
 * tangram/mapping_parameter_tuning.py:42-82), in one streaming pass that reads every element once and allocates
 * O(rows) scratch.  `arrays`: a HOST array of R DEVICE pointers (all on `device`), each rows x cols row-major f32 with
 * leading dimension ld; 1 <= R <= 8.
 *   pearson_out            R(R-1)/2 doubles (host or device; NULL to skip): np.corrcoef of the flattened arrays at
 *                          np.tril_indices(R, -1), i.e. pearson_corr (:42-53); sums in fp64, reduced in a fixed order
 *   vote_entropy_out       rows floats (host or device; NULL to skip): per row, the entropy of the R runs' argmax votes
 *                          (first column on ties) over log(cols), vote_entropy (:55-69)
 *   consensus_entropy_out  rows floats (host or device; NULL to skip): per row, the entropy of p / sum(p) with
 *                          p = mean over runs, over log(cols), consensus_entropy (:71-82)
 * Fails with TGB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).  Bit-reproducible on a given device.
 * Synchronous on `stream`. */
TGB200_API int tgb200_agreement(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                double* pearson_out, float* vote_entropy_out, float* consensus_entropy_out,
                                int32_t device, void* stream);

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
 * Arithmetic as tgb200_project: three bf16 planes per operand, six partial products on the tensor cores; accumulation
 * chains of 512 cells (tgb200_project: at most 2048), added in cell order in fp32 (round-to-nearest); no atomics.  The result does not depend on how
 * the data is staged: dense or CSR X, host or device pointers and any block size give identical bits.
 * Cell blocks of the mapping and X are double-buffered (the copies of block b + 1 run on a second stream while block b
 * contracts); device memory is out plus two blocks of staging, whatever `rows` is.  A CSR block is turned into the bf16
 * planes directly, one warp per row.  TGB200_ERR_INVALID for bad shapes, a malformed indptr, a column index outside
 * [0, n_genes) or out of order (such entries are skipped, never written), or when free device memory cannot hold out and
 * one block of 2048 cells (the message gives the sizes); TGB200_ERR_NO_DEVICE without an sm_90 device (no CPU fallback).
 * Synchronous on `stream`. */
TGB200_API int tgb200_project_map(const float* map, int64_t rows, int64_t cols, int64_t ld, const float* X, int64_t x_ld,
                                  const int64_t* indptr, const int32_t* indices, const float* data, int64_t nnz,
                                  int64_t n_genes, float* out, int64_t block_rows, int32_t device, void* stream);

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
