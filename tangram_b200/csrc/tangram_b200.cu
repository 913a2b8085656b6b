// C-ABI of the native map_cells_to_space hot path (see include/tangram_b200.h).
// Host orchestration only; every kernel is hand-written for sm_90a (H100) in the .cuh files.
#include "../../include/tangram_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "common.cuh"
#include "kernels_elem.cuh"
#include "gemm_simt.cuh"
#include "gemm_tc.cuh"
#include "adam_rows.cuh"
#include "legacy_rng.cuh"
#include "agreement.cuh"
#include "annotate.cuh"
#include "project.cuh"
#include "group_stats.cuh"
#include "neighbors.cuh"
#include "mt19937_jump.h"
#include "nccl_dl.h"

using namespace tgb;

// ---------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
static int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
#define CK(call)                                                                              \
  do {                                                                                        \
    cudaError_t e__ = (call);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return fail(TGB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), \
                  __FILE__, __LINE__);                                                        \
  } while (0)
#define CKS(expr)                 \
  do {                            \
    int s__ = (expr);             \
    if (s__ != TGB200_OK) return s__; \
  } while (0)

// `host`: mapped pinned host memory (TGB200_STATE_HOST) that kernels address directly; otherwise device memory
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  bool host = false;
  int alloc(size_t count, bool zero = true) {
    release();
    if (count == 0) return TGB200_OK;
    if (host) {
      cudaError_t e = cudaHostAlloc(&p, count * sizeof(T), cudaHostAllocMapped);
      if (e != cudaSuccess) { p = nullptr; return fail(TGB200_ERR_CUDA, "cudaHostAlloc(%zu B): %s", count * sizeof(T), cudaGetErrorString(e)); }
      n = count;                    // zeroed by the handle on the device side (zero_state), not here
      return TGB200_OK;
    }
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e != cudaSuccess) { p = nullptr; return fail(TGB200_ERR_CUDA, "cudaMalloc(%zu B): %s", count * sizeof(T), cudaGetErrorString(e)); }
    n = count;
    if (zero) {
      e = cudaMemset(p, 0, count * sizeof(T));
      if (e != cudaSuccess) return fail(TGB200_ERR_CUDA, "cudaMemset: %s", cudaGetErrorString(e));
    }
    return TGB200_OK;
  }
  void release() { if (p) { if (host) cudaFreeHost(p); else cudaFree(p); } p = nullptr; n = 0; }
  ~DevBuf() { release(); }
};

struct CsrDev {
  DevBuf<int> indptr, indices;
  DevBuf<float> vals;
  bool set = false;
  Csr view() const { return Csr{indptr.p, indices.p, vals.p}; }
};

// what the bf16-mode operand Pb holds
enum class PState {
  stale,                        // nothing valid: the next forward runs the row pass
  fresh,                        // normalised P from the row pass
  updated,                      // exp(Mnew - lse) from the streaming update; k_row_norm normalises it
};

// one launch while recording is on (tgb200_profile_step / tgb200_debug_timeline): stream 1 hi, 2 lo, 3 sf of a handle
// with streams, 0 any other (the caller's)
struct LaunchRecord {
  const char* name;
  int stream;
  cudaEvent_t ev;
};

struct tgb200_mapper {
  tgb200_config cfg;
  int N, V, K, T, Ke, ld;       // ld: leading dim of N x V arrays (elements)
  int ct_off;
  bool bf16;                    // throughput mode: bf16 operands
  bool x3;                      // parity mode on tensor cores: three bf16 planes per operand, six partial products
  bool tcm;                     // either tensor-core mode
  // state
  DevBuf<float> M, m, v;        // N x ld
  int64_t step = 0;
  // operands
  DevBuf<float> Pf;             // N x ld  (fp32 mode)
  DevBuf<__nv_bfloat16> Pb;     // N x ld  (bf16 mode)
  DevBuf<float> Sx;             // N x Ke  S_ext = [S | density cols | ct_encode | 0]
  DevBuf<__nv_bfloat16> Sxb;
  DevBuf<float> G;              // V x Ke
  DevBuf<float> d, dsrc;
  DevBuf<RowStat> stats;
  DevBuf<float> rowaux, rdot, rpart;
  DevBuf<float4> rowc;          // (lse, r, h, 0) per row for the tensor-core backward epilogue
  // tensor-core path: row normalisation carried across iterations (see k_row_norm)
  DevBuf<__nv_bfloat16> Sxs;    // N x Ke  bf16(S_ext / zt): forward B operand
  DevBuf<float> lse0, lse1, inv_zt;
  DevBuf<float> zsum, pxsum, l1sum, l2sum;   // per row, left by the streaming update (AdamRowsArgs); px / l1 / l2 only when used
  float* lseA = nullptr;        // offset the current Pb was produced with
  float* lseT = nullptr;        // exact log-sum-exp of the current rows
  // constrained mode (MapperConstrained): filter logits, their Adam state, f = sigmoid(F), S_f = f o S_ext
  bool constrained = false, have_filter = false;
  DevBuf<float> Fl, mF, vF, fsig, Sf, fscal;
  PState p_state = PState::stale;
  int r_parts = 0;
  // forward / loss
  int fwd_splits = 1;
  DevBuf<float> Ypart;          // splits x V x Ke (only when splits > 1)
  DevBuf<float> Y;              // V x Ke + kTail (exchange buffer)
  DevBuf<float> dY;             // V x Ke (fp32 mode)
  DevBuf<__nv_bfloat16> dYb;    // the tensor-core modes' dY: one bf16 plane, or three in bf16x3 mode
  DevBuf<float> ngc, ngr, WG, nwg, AG, nag, sgnG, Z, Zg, H;
  DevBuf<float> colpart, colpart_nb, colpart_go, rowpart, ctpart;
  DevBuf<float> coefA, coefB, coefAn, coefBn, coefAg, coefBg, coefAr, coefBr, densg;
  CsrDev W, WT, F, FT, A, AT;
  int nchunk = 0, ncolchunk = 0, nredchunk = 0, n_ct_blocks = 0, loss_rows = 16;
  DevBuf<float> colfin;         // finalised per-gene sums: [3 | 2 | 2][Ke]
  // training-gene mask of the loss (tgb200_set_loss_genes): gene_act[k] in {0, 1} (Ke floats) when `masked`; n_active of
  // the K genes are in the loss
  bool masked = false;
  int n_active = 0;
  DevBuf<float> gene_act;
  DevBuf<float> gw;             // Ke: sparsity weight of each gene in the loss (k_gene_weights), for the validation
  // per-epoch validation in the loop (tgb200_set_validation): epoch e (counted from that call) is validated when
  // e % val_every == 0, into history columns 12-15 of its row
  int val_every = 0;
  int64_t val_epoch = 0;
  int64_t val_row = -1;         // fp32 / bf16x3: the row whose validation this iteration's forward computes (see loss_stage)
  // sharded: a validation wrote the exchange tail (sum h in [0] and [5]); the next iteration rewrites it even when no row
  // term needs it, so that an exchange that carries no validation sums zeros there
  bool tail_stale = false;
  DevBuf<float> val_coef, val_rowpart, val_hist;   // what the validation's k_loss_scalars writes beside its four values
  // history
  DevBuf<float> hist;
  int64_t hist_len = 0, hist_cap = 0;
  // flags
  bool have_expr = false, have_density = false, have_ct = false, have_mapping = false;
  bool in_step = false;
  int64_t launches = 0;
  // last tgb200_init_mapping_legacy: ms of jump, count + scan, emit, fix-up (device, CUDA events), host polynomials,
  // then draw blocks, values recomputed on the host, values the recomputation changed
  float legacy_stats[8] = {0};
  TcContext tc;                 // driver entry points etc. for the wgmma path
  TcPlan plan_fwd, plan_dp;     // tensor maps of the two contractions, encoded once (the buffers never move)
  // backward of the bf16 mode: store-only contraction -> bf16 dq = dP - centre in HBM -> streaming Adam kernel;
  // two contractions per iteration instead of three (no separate row-dot GEMM)
  DevBuf<__nv_bfloat16> dq;     // N x ld
  DevBuf<__nv_bfloat16> mb;     // N x ld: Adam's first moment in bf16 (bf16 mode only; `m` is then not allocated).  It is an
                                // exponential average with a 10-iteration memory: bf16 rounding noise does not accumulate, and
                                // next to bf16 operands it is invisible in every parity metric (DESIGN.md); v stays fp32.
  DevBuf<float> rcenter;        // per row: last iteration's row-dot, the centre dq is stored relative to
  // the same staging for the parity mode (bf16x3): dP in fp32, exact streaming update (no chunk pipeline)
  DevBuf<float> dpf;            // N x ld
  // Pipelining of the bf16 backward over cell chunks (rows [chunk_row[c], chunk_row[c+1]), multiples of 256; {0, N} with
  // one chunk):
  //   hi (high-priority stream): forward(c) ... loss ... backward contraction(c)        -- tensor-core bound
  //   lo (low-priority stream):  row-dot finalize(c), streaming Adam(c)                 -- HBM bound
  // Adam(c) runs under the contraction of chunk c+1 and, across the iteration boundary, under the next forward's
  // chunks; forward(c) of the next iteration waits only for Adam(c).  Which stream a launch goes to is the Lanes of its
  // API call (below).
  bool pipelined = false;       // several chunks: the handle has the streams hi, lo and sf
  // SMs a pipelined contraction leaves free when an update chunk runs beside it (G(c) for c >= 1 beside A(c-1), the
  // prefetched F'(c) beside A(c+1)): without them the contraction's grid holds every SM and the update waits for it to
  // drain.  DESIGN 6b, "Running the update beside the contractions", measures the share.
  int update_sms = 0;
  // host state (TGB200_STATE_HOST, TGB200_STATE_AUTO): rows [0, R) of M, m / mb and v stay in the device buffers above,
  // rows [R, N) are in pinned host memory (Mh, mh / mbh, vh; R = 0 with host state), and a ring of two device slots of
  // `ring_rows` rows each through which every per-iteration pass streams the host rows (staged_rows): copy-in of block
  // b+1 on `cin` and copy-out of block b-1 on `cout` run on the copy engines under block b's kernel
  bool host_state = false;      // R < N
  int R = 0;
  int ring_rows = 0;
  DevBuf<float> Mh, mh, vh;
  DevBuf<__nv_bfloat16> mbh;
  DevBuf<float> rM[2], rm[2], rv[2];
  DevBuf<__nv_bfloat16> rmb[2];
  cudaStream_t cin = nullptr, cout = nullptr;
  cudaEvent_t ev_in[2] = {}, ev_comp[2] = {}, ev_free[2] = {}, ev_start = nullptr, ev_last = nullptr;
  bool ring_used = false;       // ev_last was recorded by an earlier staged pass
  int nchunks = 1, chunk_row[9] = {0};
  cudaStream_t hi = nullptr, lo = nullptr, sf = nullptr;     // sf: the NEXT iteration's forward chunks (see backward_bf16)
  cudaEvent_t ev_fork = nullptr, ev_join_hi = nullptr, ev_join_lo = nullptr, ev_join_sf = nullptr, ev_loss = nullptr;
  cudaEvent_t ev_g[8] = {}, ev_a[8] = {}, ev_f[8] = {};
  bool a_valid = false;         // ev_a[] were recorded by an earlier two-stream update and guard the rows of the next forward
  bool fwd_ahead = false;       // the previous backward issued this iteration's forward chunks on sf: the forward only waits
  // diagnostics: an event after every launch while recording is on
  bool recording = false;
  std::vector<LaunchRecord> records;
  void drop_records(size_t from) {
    for (size_t i = from; i < records.size(); ++i) cudaEventDestroy(records[i].ev);
    records.resize(from);
  }
  // cell-sharded operation: NCCL communicator of the ranks that share the voxels (tgb200_comm_init_rank / tgb200_set_comm)
  void* comm = nullptr;
  bool comm_owned = false;
  int comm_rank = 0, comm_world = 1;
  bool y_nccl = false;          // the exchange buffer lives in ncclMemAlloc memory registered with `comm`
  void* y_reg = nullptr;
  void release_exchange_registration() {
    if (!y_nccl) return;
    char e[64];
    if (NcclApi* a = nccl_api(e, sizeof(e))) {
      if (y_reg && comm) a->CommDeregister(comm, y_reg);
      a->MemFree(Y.p);
    }
    Y.p = nullptr; Y.n = 0; y_nccl = false; y_reg = nullptr;
  }
  ~tgb200_mapper() {
    release_exchange_registration();
    if (comm && comm_owned) { char e[64]; if (NcclApi* a = nccl_api(e, sizeof(e))) a->CommDestroy(comm); }
    if (hi) cudaStreamDestroy(hi);
    if (lo) cudaStreamDestroy(lo);
    if (sf) cudaStreamDestroy(sf);
    if (cin) cudaStreamDestroy(cin);
    if (cout) cudaStreamDestroy(cout);
    for (cudaEvent_t e : {ev_in[0], ev_in[1], ev_comp[0], ev_comp[1], ev_free[0], ev_free[1], ev_start, ev_last})
      if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : {ev_fork, ev_join_hi, ev_join_lo, ev_join_sf, ev_loss}) if (e) cudaEventDestroy(e);
    for (int i = 0; i < 8; ++i)
      for (cudaEvent_t e : {ev_g[i], ev_a[i], ev_f[i]}) if (e) cudaEventDestroy(e);
    drop_records(0);
  }
};

static void mark(tgb200_mapper* h, cudaStream_t s, const char* name) {
  h->launches++;
  if (!h->recording) return;
  cudaEvent_t e;
  cudaEventCreate(&e);
  cudaEventRecord(e, s);
  // without streams, hi == lo == sf == nullptr: the legacy default stream, which a caller may pass
  h->records.push_back({name, !h->pipelined ? 0 : s == h->hi ? 1 : s == h->lo ? 2 : s == h->sf ? 3 : 0, e});
}
#define LAUNCH_CHECK(name)                                                                  \
  do {                                                                                      \
    cudaError_t e__ = cudaGetLastError();                                                   \
    if (e__ != cudaSuccess) return fail(TGB200_ERR_CUDA, "launch %s: %s", name, cudaGetErrorString(e__)); \
    mark(h, s, name);                                                                       \
  } while (0)

// the fp32 S_ext every contraction consumes: f o S_ext in constrained mode, S_ext otherwise
static float* s_act(tgb200_mapper* h) { return h->constrained ? h->Sf.p : h->Sx.p; }

static bool needs_rowaux(const tgb200_config& c) { return c.lambda_l1 != 0.f || c.lambda_l2 != 0.f; }
static bool needs_rowscalars(const tgb200_config& c) {
  return c.lambda_r != 0.f || c.lambda_l1 != 0.f || c.lambda_l2 != 0.f;
}

// ---------------------------------------------------------------------------------------
extern "C" int tgb200_host_pin(void* buf, int64_t bytes, int32_t threads, int32_t device) {
  if (!buf || bytes <= 0) return fail(TGB200_ERR_INVALID, "bad argument");
  CK(cudaSetDevice(device));                      // usually a fresh host thread: bind it to the handle's device
  // first touch with several threads (a fresh 4 GB numpy buffer is a million page faults), then page-lock
  const size_t page = 4096, n = (size_t)bytes;
  const int nt = threads < 1 ? 1 : (threads > 32 ? 32 : threads);
  volatile unsigned char* b = static_cast<volatile unsigned char*>(buf);
  auto touch = [=](size_t lo, size_t hi) { for (size_t o = lo; o < hi; o += page) b[o] = 0; };
  std::vector<std::thread> pool;
  const size_t per = ((n + nt - 1) / nt + page - 1) / page * page;
  for (int t = 1; t < nt; ++t) {
    const size_t lo = (size_t)t * per, hi = lo + per < n ? lo + per : n;
    if (lo < n) pool.emplace_back(touch, lo, hi);
  }
  touch(0, per < n ? per : n);
  for (auto& th : pool) th.join();
  b[n - 1] = 0;
  CK(cudaHostRegister(buf, n, cudaHostRegisterDefault));
  return TGB200_OK;
}
extern "C" int tgb200_host_unpin(void* buf) {
  if (!buf) return fail(TGB200_ERR_INVALID, "null argument");
  CK(cudaHostUnregister(buf));
  return TGB200_OK;
}
extern "C" const char* tgb200_last_error(void) { return g_err; }
extern "C" const char* tgb200_version(void) { return "tangram_b200 0.3.0 (sm_90a)"; }

static int setup_host_state(tgb200_mapper* h, int block_rows);
static const char* state_memory_name(int32_t sm) { return sm == TGB200_STATE_HOST ? "host" : "auto"; }

// ---- state placement (tgb200_plan_state) ----------------------------------------------
// what cudaMalloc takes for one allocation at most: 2 MiB pages (small allocations share them)
static int64_t alloc_bytes(int64_t b) { return b <= 0 ? 0 : round_up(b, (int64_t)2 << 20); }
constexpr int kMaxSms = 132;                 // the most SMs an sm_90 part has: the forward's split count is largest there

// The device memory tgb200_create allocates besides M, m / mb, v and the ring: its buffers in the order it allocates
// them, each rounded up as alloc_bytes does.  Keep in step with tgb200_create (test_state_auto_gpu checks the bound).
static int64_t operand_bytes(const tgb200_config& c) {
  const int64_t N = c.n_cells, V = c.n_voxels, K = c.n_genes, T = c.n_types;
  const int64_t Ke = round_up(K + 2 + T, 64), ld = round_up(V, 64), nv = N * ld, nk = N * Ke, vk = V * Ke;
  const bool bf16 = c.precision == TGB200_PREC_BF16, x3 = c.precision == TGB200_PREC_BF16X3, tcm = bf16 || x3;
  int64_t b = 0;
  auto A = [&](int64_t bytes) { b += alloc_bytes(bytes); };
  if (x3) A(4 * nv);                                           // dpf
  if (bf16) {
    A(2 * nk); for (int i = 0; i < 4; ++i) A(4 * N);          // Sxs, lse0, lse1, inv_zt, zsum
    if (c.lambda_r != 0.f) A(4 * N);
    if (c.lambda_l1 != 0.f || c.lambda_l2 != 0.f) { A(4 * N); A(4 * N); }
    A(16 * N); A(2 * nv); A(2 * nk); A(2 * vk); A(2 * nv); A(4 * N);   // rowc, Pb, Sxb, dYb, dq, rcenter
  } else if (x3) {
    A(6 * nv); A(6 * nk); A(6 * vk);
  } else {
    A(4 * nv);
  }
  A(4 * nk); A(4 * vk); A(4 * V); A(4 * N); A((int64_t)sizeof(RowStat) * N); A(8 * N); A(4 * N);
  int nc = 1;
  if (bf16 && !c.constrained) {
    nc = N >= 32768 ? 4 : (N >= 8192 ? 2 : 1);
    while (nc > 1 && N / nc < 1024) --nc;
  }
  int splits = 1;
  if (nc == 1 && tcm) {
    splits = tc_forward_splits(kMaxSms, (int)N, (int)V, (int)Ke);
    if (x3) splits = std::max(splits, tc_splits_for_chain(N, 2048));
  } else if (!tcm) {
    splits = std::clamp((int)ceil_div(2 * kMaxSms, ceil_div(V, 128) * ceil_div(Ke, 128)), 1, (int)ceil_div(N, 512));
  }
  if (splits > 1) A(4 * splits * vk);
  A(4 * (vk + kTail));
  if (!tcm) A(4 * vk);
  if (c.constrained) { for (int i = 0; i < 4; ++i) A(4 * N); A(4 * nk); A(16); }
  const int64_t r_parts = tcm ? tc_dp_row_parts((int)V) : ceil_div(Ke, SG_BN);
  A(4 * r_parts * N);
  A(4 * Ke); A(4 * V);
  int64_t loss_rows = 16;
  while (ceil_div(V, loss_rows) > 512 && loss_rows < kLossRowsMax) loss_rows += 16;
  const int64_t nchunk = ceil_div(V, loss_rows), ncolchunk = ceil_div(Ke, kLossCols);
  A(4 * 7 * Ke); A(4 * nchunk * 3 * Ke); A(4 * Ke); A(4 * Ke); A(4 * Ke); A(4 * V);
  if (c.lambda_g2 != 0.f) { A(4 * ncolchunk * V * 2); A(4 * V); A(4 * V); }
  if (c.lambda_neighborhood_g1 > 0.f) { A(4 * vk); A(4 * Ke); A(4 * vk); A(4 * nchunk * 2 * Ke); A(4 * Ke); A(4 * Ke); }
  if (c.lambda_getis_ord > 0.f) {
    A(4 * vk); A(4 * Ke); A(4 * Ke); A(4 * vk); A(4 * nchunk * 2 * Ke); A(4 * Ke); A(4 * Ke);
  }
  if (c.lambda_ct_islands > 0.f) { A(4 * V * T); A(4 * ceil_div(V * T, 256)); }
  return b;
}

// What the handle allocates after tgb200_create and a row split must leave free.  1 GiB holds CUDA's loading of this
// library's kernels with their local memory, the legacy draw's scratch (tens of MiB at 160k x 24k), the CSR graphs of
// the spatial terms (12 B per edge), the history (64 B per epoch), tgb200_get_state's one-row scratch and a projection's
// smallest block; the projection sizes its blocks to the memory then free, and its output (n_voxels x genes floats) is the
// caller's choice.  Added to it: the validation's scratch and set_comm's copy of the exchange buffer, which scale with the
// shape.
static int64_t reserve_bytes(const tgb200_config& c) {
  const int64_t V = c.n_voxels, Ke = round_up((int64_t)c.n_genes + 2 + c.n_types, 64);
  return ((int64_t)1 << 30) + alloc_bytes(4 * (2 * Ke + 2 * V)) + alloc_bytes(4 * TGB200_HIST_COLS) +
         alloc_bytes(4 * ceil_div(Ke, kLossCols) * V * 2) + alloc_bytes(4 * (V * Ke + kTail));
}

// bytes of one row of M, m / mb and v
static int64_t state_row_bytes(const tgb200_config& c) {
  return round_up(c.n_voxels, 64) * (c.precision == TGB200_PREC_BF16 ? 4 + 2 + 4 : 4 + 4 + 4);
}

// device bytes of rows [0, R) of the state and of a ring of two slots of `rb` rows (three allocations each)
static int64_t state_device_bytes(const tgb200_config& c, int64_t R, int64_t rb) {
  const int64_t ld = round_up(c.n_voxels, 64), mb = c.precision == TGB200_PREC_BF16 ? 2 : 4;
  return 2 * alloc_bytes(4 * R * ld) + alloc_bytes(mb * R * ld) + 2 * (2 * alloc_bytes(4 * rb * ld) + alloc_bytes(mb * rb * ld));
}

static int64_t env_rows(const char* name) {
  const char* e = getenv(name);
  return e && *e ? atoll(e) : -1;
}

extern "C" int tgb200_plan_state(const tgb200_config* cfg, uint64_t device_free, tgb200_state_plan* out) {
  if (!cfg || !out) return fail(TGB200_ERR_INVALID, "null argument");
  const tgb200_config& c = *cfg;
  if (c.n_cells <= 0 || c.n_voxels <= 0 || c.n_genes <= 0 || c.n_types < 0)
    return fail(TGB200_ERR_INVALID, "bad shape cells=%d voxels=%d genes=%d types=%d", c.n_cells, c.n_voxels, c.n_genes, c.n_types);
  if (c.precision != TGB200_PREC_FP32 && c.precision != TGB200_PREC_BF16 && c.precision != TGB200_PREC_BF16X3)
    return fail(TGB200_ERR_INVALID, "unknown precision %d", c.precision);
  if (c.state_memory < TGB200_STATE_DEVICE || c.state_memory > TGB200_STATE_AUTO)
    return fail(TGB200_ERR_INVALID, "unknown state_memory %d", c.state_memory);
  if (c.state_memory != TGB200_STATE_DEVICE && c.precision == TGB200_PREC_FP32)
    return fail(TGB200_ERR_UNSUPPORTED, "state_memory = %s needs precision bf16 or bf16x3: fp32 fuses Adam into its FFMA contraction",
                state_memory_name(c.state_memory));
  const int64_t N = c.n_cells, sr = state_row_bytes(c), ops = operand_bytes(c), res = reserve_bytes(c);
  const int64_t free_b = (int64_t)std::min<uint64_t>(device_free, (uint64_t)INT64_MAX);
  // rows per ring slot: both slots take at most an eighth of what the operands leave free and 128 MiB in all -- a block
  // of 64 MiB is copied at link speed
  int64_t rb0 = env_rows("TGB200_STATE_BLOCK_ROWS");
  if (rb0 < 0) rb0 = std::min<int64_t>(std::max<int64_t>(free_b - ops, 0) / 8, (int64_t)128 << 20) / (2 * sr);
  rb0 = std::clamp<int64_t>(rb0, 1, N);
  int64_t R = N, rb = 0;
  if (c.state_memory == TGB200_STATE_HOST) {
    R = 0; rb = rb0;
  } else if (c.state_memory == TGB200_STATE_AUTO) {
    const int64_t forced = env_rows("TGB200_STATE_RESIDENT_ROWS");
    if (forced >= 0) {
      R = std::min<int64_t>(forced, N);
      rb = R < N ? std::min<int64_t>(rb0, N - R) : 0;
    } else if (ops + state_device_bytes(c, N, 0) + res > free_b) {
      // R + 2 rb rows of state fit in what the operands, the reserve and the allocations' rounding leave; the slots
      // shrink when fewer than 2 rb0 rows fit, and R + rb <= N holds because fewer than N rows fit
      const int64_t k = std::max<int64_t>(free_b - ops - res - 9 * alloc_bytes(1), 0) / sr;
      rb = std::clamp<int64_t>(std::min<int64_t>(rb0, k / 2), 1, N);
      R = std::max<int64_t>(k - 2 * rb, 0);
    }
  }
  out->resident_rows = (int32_t)R;
  out->block_rows = (int32_t)rb;
  out->device_bytes = ops + state_device_bytes(c, R, rb);
  out->reserve_bytes = res;
  out->host_bytes = (N - R) * sr;
  return TGB200_OK;
}

extern "C" int tgb200_resident_rows(tgb200_mapper* h, int32_t* out) {
  if (!h || !out) return fail(TGB200_ERR_INVALID, "null argument");
  *out = h->R;
  return TGB200_OK;
}

extern "C" int tgb200_create(const tgb200_config* cfg, tgb200_mapper** out) {
  if (!cfg || !out) return fail(TGB200_ERR_INVALID, "null argument");
  *out = nullptr;
  // a caller written before `state_memory` existed passes the struct without it: its state stays on the device
  const size_t size_v1 = offsetof(tgb200_config, state_memory);
  if (cfg->struct_size != (int32_t)sizeof(tgb200_config) && cfg->struct_size != (int32_t)size_v1)
    return fail(TGB200_ERR_INVALID, "tgb200_config.struct_size=%d, expected %zu", cfg->struct_size, sizeof(tgb200_config));
  tgb200_config full{};
  memcpy(&full, cfg, (size_t)cfg->struct_size);
  full.struct_size = (int32_t)sizeof(tgb200_config);
  cfg = &full;
  if (cfg->n_cells <= 0 || cfg->n_voxels <= 0 || cfg->n_genes <= 0 || cfg->n_types < 0)
    return fail(TGB200_ERR_INVALID, "bad shape cells=%d voxels=%d genes=%d types=%d", cfg->n_cells, cfg->n_voxels, cfg->n_genes, cfg->n_types);
  if (cfg->lambda_g1 == 0.f) return fail(TGB200_ERR_INVALID, "lambda_g1 cannot be 0.");  // mapping_utils.py:206-207
  if (cfg->precision != TGB200_PREC_FP32 && cfg->precision != TGB200_PREC_BF16 && cfg->precision != TGB200_PREC_BF16X3)
    return fail(TGB200_ERR_INVALID, "unknown precision %d", cfg->precision);
  if (cfg->density_mode < 0 || cfg->density_mode > 2) return fail(TGB200_ERR_INVALID, "unknown density_mode %d", cfg->density_mode);
  if (cfg->lambda_ct_islands > 0.f && cfg->n_types <= 0) return fail(TGB200_ERR_INVALID, "lambda_ct_islands > 0 needs n_types > 0");
  // a shard holds a block of the n_cells_global cells: fewer would count the handle as sharded and scale the density wrong
  if (cfg->n_cells_global > 0 && cfg->n_cells_global < cfg->n_cells)
    return fail(TGB200_ERR_INVALID, "n_cells_global=%lld < n_cells=%d", (long long)cfg->n_cells_global, cfg->n_cells);
  if (cfg->constrained) {
    if (cfg->density_mode == TGB200_DENSITY_SOURCE) return fail(TGB200_ERR_INVALID, "constrained mode has no d_source (mapping_optimizer.py:417-432)");
    if (cfg->lambda_neighborhood_g1 > 0.f || cfg->lambda_ct_islands > 0.f || cfg->lambda_getis_ord > 0.f || cfg->lambda_l1 != 0.f || cfg->lambda_l2 != 0.f)
      return fail(TGB200_ERR_INVALID, "constrained mode has no spatial / L1 / L2 terms (mapping_optimizer.py:417-432)");
    if (cfg->n_cells_global > 0 && cfg->n_cells_global != cfg->n_cells && cfg->target_count <= 0.f) return fail(TGB200_ERR_INVALID, "target_count must be given");
  }
  if (cfg->state_memory < TGB200_STATE_DEVICE || cfg->state_memory > TGB200_STATE_AUTO)
    return fail(TGB200_ERR_INVALID, "unknown state_memory %d", cfg->state_memory);
  if (cfg->state_memory != TGB200_STATE_DEVICE && cfg->precision == TGB200_PREC_FP32)
    return fail(TGB200_ERR_UNSUPPORTED, "state_memory = %s needs precision bf16 or bf16x3: fp32 fuses Adam into its FFMA contraction",
                state_memory_name(cfg->state_memory));
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(TGB200_ERR_NO_DEVICE, "no CUDA device visible: tangram_b200 has no CPU fallback");
  }
  if (cfg->device < 0 || cfg->device >= ndev) return fail(TGB200_ERR_INVALID, "device %d out of range (%d devices)", cfg->device, ndev);
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(TGB200_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", cfg->device, prop.major, prop.minor);
  CK(cudaSetDevice(cfg->device));
  // the row split of TGB200_STATE_AUTO, planned on the memory free before anything of this handle is allocated
  tgb200_state_plan plan{};
  if (cfg->state_memory == TGB200_STATE_AUTO) {
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    CKS(tgb200_plan_state(cfg, free_b, &plan));
  }

  tgb200_mapper* h = new tgb200_mapper();
  h->cfg = *cfg;
  if (h->cfg.n_cells_global <= 0) h->cfg.n_cells_global = cfg->n_cells;
  if (h->cfg.adam_beta1 == 0.f) h->cfg.adam_beta1 = 0.9f;
  if (h->cfg.adam_beta2 == 0.f) h->cfg.adam_beta2 = 0.999f;
  if (h->cfg.adam_eps == 0.f) h->cfg.adam_eps = 1e-8f;
  h->N = cfg->n_cells; h->V = cfg->n_voxels; h->K = cfg->n_genes; h->T = cfg->n_types;
  h->n_active = h->K;
  h->constrained = cfg->constrained != 0;
  h->bf16 = cfg->precision == TGB200_PREC_BF16;
  h->x3 = cfg->precision == TGB200_PREC_BF16X3;
  h->tcm = h->bf16 || h->x3;
  h->ct_off = h->K + 2;
  h->Ke = (int)round_up(h->K + 2 + h->T, 64);
  h->ld = (int)round_up(h->V, 64);
  const size_t nv = (size_t)h->N * h->ld, vk = (size_t)h->V * h->Ke;
  int st = TGB200_OK;
  auto A = [&](int s) { if (st == TGB200_OK) st = s; };
  h->R = cfg->state_memory == TGB200_STATE_HOST ? 0 : cfg->state_memory == TGB200_STATE_AUTO ? plan.resident_rows : h->N;
  h->host_state = h->R < h->N;
  h->Mh.host = h->mh.host = h->mbh.host = h->vh.host = true;
  const size_t nr = (size_t)h->R * h->ld, nh = nv - nr;
  if (h->x3) A(h->dpf.alloc(nv, false));
  A(h->M.alloc(nr)); A(h->v.alloc(nr));
  if (h->bf16) A(h->mb.alloc(nr)); else A(h->m.alloc(nr));
  A(h->Mh.alloc(nh)); A(h->vh.alloc(nh));
  if (h->bf16) A(h->mbh.alloc(nh)); else A(h->mh.alloc(nh));
  if (h->bf16) {
    A(h->Sxs.alloc((size_t)h->N * h->Ke)); A(h->lse0.alloc(h->N)); A(h->lse1.alloc(h->N)); A(h->inv_zt.alloc(h->N));
    A(h->zsum.alloc(h->N));
    if (cfg->lambda_r != 0.f) A(h->pxsum.alloc(h->N));
    if (cfg->lambda_l1 != 0.f || cfg->lambda_l2 != 0.f) { A(h->l1sum.alloc(h->N)); A(h->l2sum.alloc(h->N)); }
    h->lseA = h->lse0.p; h->lseT = h->lse1.p;
    A(h->rowc.alloc(h->N)); A(h->Pb.alloc(nv)); A(h->Sxb.alloc((size_t)h->N * h->Ke)); A(h->dYb.alloc(vk));
    A(h->dq.alloc(nv, false)); A(h->rcenter.alloc(h->N));
  } else if (h->x3) {
    A(h->Pb.alloc(3 * nv)); A(h->Sxb.alloc((size_t)3 * h->N * h->Ke)); A(h->dYb.alloc(3 * vk));
  } else {
    A(h->Pf.alloc(nv));
  }
  A(h->Sx.alloc((size_t)h->N * h->Ke));
  A(h->G.alloc(vk));
  A(h->d.alloc(h->V)); A(h->dsrc.alloc(h->N));
  A(h->stats.alloc(h->N)); A(h->rowaux.alloc((size_t)2 * h->N)); A(h->rdot.alloc(h->N));
  int nc = 1;
  if (h->bf16) {
    // cell chunks of the pipelined backward: 4 from 32k cells up, 2 from 8k (a rank of an 8-way sharded 100k-cell run):
    // each chunk still fills the GPU several times over
    nc = h->N >= 32768 ? 4 : (h->N >= 8192 ? 2 : 1);
    if (const char* e = getenv("TGB200_CHUNKS")) nc = atoi(e);
    if (nc < 1) nc = 1;
    if (nc > 8) nc = 8;
    // The filter update couples all rows of an iteration.  So a constrained handle has one chunk and no streams, and
    // its next k_filter_prepare follows the filter update on the same stream without waiting for an event.
    if (h->constrained) nc = 1;
    while (nc > 1 && h->N / nc < 1024) --nc;
  }
  h->nchunks = nc;
  for (int c = 0; c <= nc; ++c) h->chunk_row[c] = c == nc ? h->N : (int)round_up((int64_t)c * h->N / nc, 256);
  if (h->nchunks > 1) {                      // one chunk: nothing to overlap, everything stays on the caller's stream
    int lo_p = 0, hi_p = 0;
    cudaDeviceGetStreamPriorityRange(&lo_p, &hi_p);
    // priorities: backward contractions (they feed the streaming update) > next forward's chunks > the update itself
    const int mid_p = hi_p < lo_p ? hi_p + 1 : lo_p;
    bool ok = cudaStreamCreateWithPriority(&h->hi, cudaStreamNonBlocking, hi_p) == cudaSuccess &&
              cudaStreamCreateWithPriority(&h->sf, cudaStreamNonBlocking, mid_p) == cudaSuccess &&
              cudaStreamCreateWithPriority(&h->lo, cudaStreamNonBlocking, lo_p) == cudaSuccess;
    cudaEvent_t* evs[5] = {&h->ev_fork, &h->ev_join_hi, &h->ev_join_lo, &h->ev_join_sf, &h->ev_loss};
    for (auto e : evs) ok = ok && cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
    for (int c = 0; c < 8; ++c)
      ok = ok && cudaEventCreateWithFlags(&h->ev_g[c], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&h->ev_a[c], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&h->ev_f[c], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) A(fail(TGB200_ERR_CUDA, "stream / event creation failed: %s", cudaGetErrorString(cudaGetLastError())));
    h->pipelined = ok;
    h->update_sms = 16;
    if (const char* e = getenv("TGB200_UPDATE_SMS")) h->update_sms = std::max(0, atoi(e));
  }
  // forward split over cells (deterministic partial planes)
  h->tc.num_sms = prop.multiProcessorCount;
  if (h->nchunks > 1) {
    h->fwd_splits = 1;                       // the cell chunks of the pipelined forward accumulate straight into Y_ext
  } else if (h->tcm) {
    h->fwd_splits = tc_forward_splits(h->tc.num_sms, h->N, h->V, h->Ke);
    if (h->x3) h->fwd_splits = std::max(h->fwd_splits, tc_splits_for_chain(h->N, 2048));
  } else {                                   // the SIMT grid covers the SMs twice
    const int tiles = (int)(ceil_div(h->V, 128) * ceil_div(h->Ke, 128));
    h->fwd_splits = std::clamp((int)ceil_div(2 * h->tc.num_sms, tiles), 1, (int)ceil_div(h->N, 512));
  }
  if (h->fwd_splits > 1) A(h->Ypart.alloc((size_t)h->fwd_splits * vk));
  A(h->Y.alloc(vk + kTail));
  if (!h->tcm) A(h->dY.alloc(vk));
  if (h->constrained) {
    A(h->Fl.alloc(h->N)); A(h->mF.alloc(h->N)); A(h->vF.alloc(h->N)); A(h->fsig.alloc(h->N));
    A(h->Sf.alloc((size_t)h->N * h->Ke)); A(h->fscal.alloc(4));
  }
  h->r_parts = h->tcm ? tc_dp_row_parts(h->V) : (int)ceil_div(h->Ke, SG_BN);                   // TcEpiDpStore: one partial per voxel tile
  A(h->rpart.alloc((size_t)h->r_parts * h->N));
  A(h->ngc.alloc(h->Ke)); A(h->ngr.alloc(h->V));
  // voxel rows per CTA of the loss reductions: enough CTAs for small V, bounded partial arrays for large V
  h->loss_rows = 16;
  while (ceil_div(h->V, h->loss_rows) > 512 && h->loss_rows < kLossRowsMax) h->loss_rows += 16;
  h->nchunk = (int)ceil_div(h->V, h->loss_rows);
  A(h->colfin.alloc((size_t)7 * h->Ke));
  h->ncolchunk = (int)ceil_div(h->Ke, kLossCols);
  h->nredchunk = (int)ceil_div(h->Ke, kLossColsBlk);
  A(h->colpart.alloc((size_t)h->nchunk * 3 * h->Ke));
  A(h->coefA.alloc(h->Ke)); A(h->coefB.alloc(h->Ke));
  A(h->gw.alloc(h->Ke));
  A(h->densg.alloc(h->V));
  if (cfg->lambda_g2 != 0.f) { A(h->rowpart.alloc((size_t)h->ncolchunk * h->V * 2)); A(h->coefAr.alloc(h->V)); A(h->coefBr.alloc(h->V)); }
  if (cfg->lambda_neighborhood_g1 > 0.f) {
    A(h->WG.alloc(vk)); A(h->nwg.alloc(h->Ke)); A(h->Z.alloc(vk)); A(h->colpart_nb.alloc((size_t)h->nchunk * 2 * h->Ke));
    A(h->coefAn.alloc(h->Ke)); A(h->coefBn.alloc(h->Ke));
  }
  if (cfg->lambda_getis_ord > 0.f) {
    A(h->AG.alloc(vk)); A(h->nag.alloc(h->Ke)); A(h->sgnG.alloc(h->Ke)); A(h->Zg.alloc(vk));
    A(h->colpart_go.alloc((size_t)h->nchunk * 2 * h->Ke)); A(h->coefAg.alloc(h->Ke)); A(h->coefBg.alloc(h->Ke));
  }
  if (cfg->lambda_ct_islands > 0.f) {
    h->n_ct_blocks = (int)ceil_div((int64_t)h->V * h->T, 256);
    A(h->H.alloc((size_t)h->V * h->T)); A(h->ctpart.alloc(h->n_ct_blocks));
  }
  if (st == TGB200_OK && h->tcm) st = tc_init(h->tc, g_err, sizeof(g_err));
  if (st == TGB200_OK && h->host_state) st = setup_host_state(h, plan.block_rows);
  if (st != TGB200_OK) { delete h; return st; }
  CK(cudaDeviceSynchronize());
  *out = h;
  return TGB200_OK;
}

extern "C" int tgb200_destroy(tgb200_mapper* h) {
  if (!h) return TGB200_OK;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  delete h;
  return TGB200_OK;
}

// copy a dense host-or-device row-major matrix into a padded device matrix at a column offset
static int upload_padded(tgb200_mapper* h, const float* src, int rows, int cols, float* dst, int ld, int col_off,
                         cudaStream_t s) {
  DevBuf<float> tmp;
  CKS(tmp.alloc((size_t)rows * cols, false));
  CK(cudaMemcpyAsync(tmp.p, src, (size_t)rows * cols * sizeof(float), cudaMemcpyDefault, s));
  const long long n = (long long)rows * cols;
  k_pack_rows<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(tmp.p, rows, cols, dst, ld, col_off);
  LAUNCH_CHECK("pack_rows");
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

static int refresh_bf16_operands(tgb200_mapper* h, cudaStream_t s) {
  if (!h->tcm) return TGB200_OK;
  const long long n = (long long)h->N * h->Ke;
  if (h->x3) {
    k_split3<<<(unsigned)ceil_div(n / 4, 256), 256, 0, s>>>(s_act(h), Split3{h->Sxb.p, (size_t)n}, n / 4);
    LAUNCH_CHECK("split3");
    return TGB200_OK;
  }
  k_f32_to_bf16<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(s_act(h), h->Sxb.p, n);
  LAUNCH_CHECK("f32_to_bf16");
  return TGB200_OK;
}

static int fill_density_cols(tgb200_mapper* h, cudaStream_t s) {
  const float* w = (h->cfg.density_mode == TGB200_DENSITY_SOURCE) ? h->dsrc.p : nullptr;
  k_fill_density_cols<<<(unsigned)ceil_div(h->N, 256), 256, 0, s>>>(h->Sx.p, h->N, h->Ke, h->K, w, h->bf16 ? 1 : 0);
  LAUNCH_CHECK("fill_density_cols");
  return refresh_bf16_operands(h, s);
}

static int gene_weights(tgb200_mapper* h, cudaStream_t s) {
  k_gene_weights<<<(unsigned)ceil_div(h->Ke, 128), 128, 0, s>>>(h->V, h->K, h->Ke, h->G.p, h->masked ? h->gene_act.p : nullptr, h->gw.p);
  LAUNCH_CHECK("gene_weights");
  return TGB200_OK;
}

static int precompute_graph_constants(tgb200_mapper* h, cudaStream_t s) {
  if (!h->have_expr) return TGB200_OK;
  dim3 grid(h->V, (unsigned)ceil_div(h->Ke, 128));      // voxels on x: gridDim.y is limited to 65535
  if (h->cfg.lambda_neighborhood_g1 > 0.f && h->W.set) {
    k_spmm<<<grid, 128, 0, s>>>(h->V, h->K, h->Ke, h->W.view(), h->G.p, h->WG.p);
    LAUNCH_CHECK("spmm");
    k_col_norms<<<(unsigned)ceil_div(h->K, 128), 128, 0, s>>>(h->V, h->K, h->Ke, h->WG.p, h->nwg.p, nullptr);
    LAUNCH_CHECK("col_norms");
  }
  if (h->cfg.lambda_getis_ord > 0.f && h->A.set) {
    k_spmm<<<grid, 128, 0, s>>>(h->V, h->K, h->Ke, h->A.view(), h->G.p, h->AG.p);
    LAUNCH_CHECK("spmm");
    k_col_norms<<<(unsigned)ceil_div(h->K, 128), 128, 0, s>>>(h->V, h->K, h->Ke, h->AG.p, h->nag.p, nullptr);
    LAUNCH_CHECK("col_norms");
    k_col_norms<<<(unsigned)ceil_div(h->K, 128), 128, 0, s>>>(h->V, h->K, h->Ke, h->G.p, h->ngc.p, h->sgnG.p);
    LAUNCH_CHECK("col_norms");
  }
  return TGB200_OK;
}

extern "C" int tgb200_set_expression(tgb200_mapper* h, const float* S, const float* G, void* stream) {
  if (!h || !S || !G) return fail(TGB200_ERR_INVALID, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemsetAsync(h->Sx.p, 0, h->Sx.n * sizeof(float), s));
  CK(cudaMemsetAsync(h->G.p, 0, h->G.n * sizeof(float), s));
  CKS(upload_padded(h, S, h->N, h->K, h->Sx.p, h->Ke, 0, s));
  CKS(upload_padded(h, G, h->V, h->K, h->G.p, h->Ke, 0, s));
  k_col_norms<<<(unsigned)ceil_div(h->K, 128), 128, 0, s>>>(h->V, h->K, h->Ke, h->G.p, h->ngc.p, nullptr);
  LAUNCH_CHECK("col_norms");
  k_row_norms<<<(unsigned)ceil_div(h->V, 8), 256, 0, s>>>(h->V, h->K, h->Ke, h->G.p, h->masked ? h->gene_act.p : nullptr, h->ngr.p);
  LAUNCH_CHECK("row_norms");
  CKS(gene_weights(h, s));
  h->have_expr = true;
  h->have_ct = false;
  CKS(fill_density_cols(h, s));
  CKS(precompute_graph_constants(h, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_set_density(tgb200_mapper* h, const float* d, const float* d_source, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  if (h->cfg.density_mode != TGB200_DENSITY_NONE && !d) return fail(TGB200_ERR_INVALID, "density_mode != NONE needs d");
  if (h->cfg.density_mode == TGB200_DENSITY_SOURCE && !d_source) return fail(TGB200_ERR_INVALID, "DENSITY_SOURCE needs d_source");
  if (d) CK(cudaMemcpyAsync(h->d.p, d, h->V * sizeof(float), cudaMemcpyDefault, s));
  if (d_source) CK(cudaMemcpyAsync(h->dsrc.p, d_source, h->N * sizeof(float), cudaMemcpyDefault, s));
  h->have_density = true;
  if (h->have_expr) CKS(fill_density_cols(h, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_set_ct_encode(tgb200_mapper* h, const float* E, void* stream) {
  if (!h || !E) return fail(TGB200_ERR_INVALID, "null argument");
  if (h->T <= 0) return fail(TGB200_ERR_INVALID, "handle was created with n_types == 0");
  if (!h->have_expr) return fail(TGB200_ERR_STATE, "call tgb200_set_expression first");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(upload_padded(h, E, h->N, h->T, h->Sx.p, h->Ke, h->ct_off, s));
  CKS(refresh_bf16_operands(h, s));
  h->have_ct = true;
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

static int upload_csr(CsrDev& dst, int V, const int32_t* indptr, const int32_t* indices, const float* vals, int64_t nnz) {
  CKS(dst.indptr.alloc(V + 1, false));
  CKS(dst.indices.alloc(nnz > 0 ? nnz : 1, false));
  CKS(dst.vals.alloc(nnz > 0 ? nnz : 1, false));
  CK(cudaMemcpy(dst.indptr.p, indptr, (V + 1) * sizeof(int), cudaMemcpyHostToDevice));
  if (nnz > 0) {
    CK(cudaMemcpy(dst.indices.p, indices, nnz * sizeof(int), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dst.vals.p, vals, nnz * sizeof(float), cudaMemcpyHostToDevice));
  }
  dst.set = true;
  return TGB200_OK;
}

extern "C" int tgb200_set_graph(tgb200_mapper* h, int which, const int32_t* indptr, const int32_t* indices,
                                const float* values, int64_t nnz, void* stream) {
  if (!h || !indptr || (nnz > 0 && (!indices || !values))) return fail(TGB200_ERR_INVALID, "null argument");
  if (which < 0 || which > 2) return fail(TGB200_ERR_INVALID, "unknown graph id %d", which);
  const int V = h->V;
  if (indptr[0] != 0 || indptr[V] != nnz) return fail(TGB200_ERR_INVALID, "CSR indptr does not match nnz=%lld", (long long)nnz);
  // non-decreasing from 0 to nnz: every row range lies in [0, nnz), so the transpose below counts each entry once
  for (int j = 0; j < V; ++j)
    if (indptr[j + 1] < indptr[j]) return fail(TGB200_ERR_INVALID, "CSR indptr decreases at row %d (%d -> %d)", j, indptr[j], indptr[j + 1]);
  for (int64_t e = 0; e < nnz; ++e)
    if (indices[e] < 0 || indices[e] >= V) return fail(TGB200_ERR_INVALID, "CSR column index %d out of range", indices[e]);
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  // transpose on the host (counting sort): backward needs Op^T
  std::vector<int> tptr(V + 1, 0), tidx(nnz);
  std::vector<float> tval(nnz);
  for (int64_t e = 0; e < nnz; ++e) tptr[indices[e] + 1]++;
  for (int j = 0; j < V; ++j) tptr[j + 1] += tptr[j];
  {
    std::vector<int> cur(tptr.begin(), tptr.end() - 1);
    for (int j = 0; j < V; ++j)
      for (int e = indptr[j]; e < indptr[j + 1]; ++e) {
        const int q = cur[indices[e]]++;
        tidx[q] = j; tval[q] = values[e];
      }
  }
  CsrDev* fw = which == 0 ? &h->W : which == 1 ? &h->F : &h->A;
  CsrDev* bw = which == 0 ? &h->WT : which == 1 ? &h->FT : &h->AT;
  CKS(upload_csr(*fw, V, indptr, indices, values, nnz));
  CKS(upload_csr(*bw, V, tptr.data(), tidx.data(), tval.data(), nnz));
  CKS(precompute_graph_constants(h, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// cudaMemsetAsync(0) of M, m / mb or v: its device rows `d` and its host rows `hp`, into which a kernel writes the zeros
// (rows of ld elements: 16-byte multiples)
template <typename T>
static int zero_state(tgb200_mapper* h, DevBuf<T>& d, DevBuf<T>& hp, cudaStream_t s) {
  if (d.n) CK(cudaMemsetAsync(d.p, 0, d.n * sizeof(T), s));
  if (!hp.n) return TGB200_OK;
  const long long n16 = (long long)(hp.n * sizeof(T) / 16);
  k_zero16<<<(unsigned)std::min<long long>(ceil_div(n16, 256), 2048), 256, 0, s>>>(reinterpret_cast<uint4*>(hp.p), n16);
  LAUNCH_CHECK("zero16");
  return TGB200_OK;
}

// row r of M, m / mb or v: rows [0, R) in the device buffer `d`, rows [R, N) in the host buffer `hp`
template <typename T>
static T* state_row(const tgb200_mapper* h, const DevBuf<T>& d, const DevBuf<T>& hp, int64_t r) {
  return r < h->R ? d.p + r * h->ld : hp.p + (r - h->R) * h->ld;
}

// f(r0, r1) for each non-empty part of the state: rows [0, R) on the device, rows [R, N) in host memory
template <typename F>
static int state_parts(const tgb200_mapper* h, F f) {
  if (h->R > 0) CKS(f(0, h->R));
  if (h->R < h->N) CKS(f(h->R, h->N));
  return TGB200_OK;
}

// Host rows: zero them once (as the device rows' cudaMalloc'd buffers are), then the ring.  `block_rows` (auto state:
// the plan's) sets the rows per slot; 0 (host state) sizes the two slots from the memory the handle left free: at most an
// eighth of it and 128 MiB in all -- a block of 64 MiB is copied at link speed, and the device keeps room for the
// projection's and validation's scratch.  TGB200_STATE_BLOCK_ROWS sets the rows per block.
static int setup_host_state(tgb200_mapper* h, int block_rows) {
  DevBuf<float> none;
  DevBuf<__nv_bfloat16> none_b;
  CKS(zero_state(h, none, h->Mh, nullptr));
  if (h->bf16) CKS(zero_state(h, none_b, h->mbh, nullptr)); else CKS(zero_state(h, none, h->mh, nullptr));
  CKS(zero_state(h, none, h->vh, nullptr));
  const size_t row_bytes = (size_t)h->ld * (h->bf16 ? 4 + 2 + 4 : 4 + 4 + 4);
  int64_t rows = block_rows;
  if (rows <= 0) {
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const size_t budget = std::min<size_t>(free_b / 8, (size_t)128 << 20);
    rows = (int64_t)(budget / (2 * row_bytes));
    if (const char* e = getenv("TGB200_STATE_BLOCK_ROWS")) rows = atoll(e);
  }
  h->ring_rows = (int)std::clamp<int64_t>(rows, 1, h->N - h->R);
  const size_t n = (size_t)h->ring_rows * h->ld;
  for (int k = 0; k < 2; ++k) {
    CKS(h->rM[k].alloc(n, false)); CKS(h->rv[k].alloc(n, false));
    if (h->bf16) CKS(h->rmb[k].alloc(n, false)); else CKS(h->rm[k].alloc(n, false));
  }
  CK(cudaStreamCreateWithFlags(&h->cin, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&h->cout, cudaStreamNonBlocking));
  for (cudaEvent_t* e : {&h->ev_in[0], &h->ev_in[1], &h->ev_comp[0], &h->ev_comp[1], &h->ev_free[0], &h->ev_free[1],
                         &h->ev_start, &h->ev_last})
    CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  return TGB200_OK;
}

// a row-shifted base: row i of the block that starts at row b0 is at base + i * ld for i in [b0, b0 + ring_rows), so
// the kernels index the slot (or the host part of the state) with the mapping's own row numbers and run exactly their
// resident arithmetic
template <typename T>
static T* shifted(T* slot, int b0, int ld) {
  return reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(slot) - (uintptr_t)b0 * ld * sizeof(T));
}

struct StagedPtrs { float* M; float* m; __nv_bfloat16* mb; float* v; };

// Rows [r0, r1) of the state, each launch on `s`: `launch(b0, b1, ptrs)` with bases that row i of [b0, b1) is addressed
// from by the mapping's row number.  Rows below R are launched on the device buffers.  Rows from R on go through the ring
// in blocks of ring_rows: the copy-in of block b+1 (stream cin) and the copy-out of block b-1 (stream cout, `write`
// passes only: M, m / mb, v) overlap block b's kernel.  The resident rows are launched in as many pieces as there are
// staged blocks, plus one, one piece before each block's kernel and one after the last: the copy engines then work under
// the resident kernels as well, and the pass approaches the larger of the compute of all its rows and the transfer of its
// staged rows.  A pass with staged rows starts after the work queued on `s` and after the previous staged pass (whatever
// stream ran it) has finished with the slots and written the host copy back; `s` continues after the last copy-out.
template <typename F>
static int staged_rows(tgb200_mapper* h, cudaStream_t s, int r0, int r1, bool write, F launch) {
  const StagedPtrs dev{h->M.p, h->m.p, h->mb.p, h->v.p};
  const int rm = std::min(r1, h->R), s0 = std::max(r0, h->R);     // resident rows [r0, rm), staged rows [s0, r1)
  if (s0 >= r1) return r0 < r1 ? launch(r0, r1, dev) : TGB200_OK;
  const int ld = h->ld, n_res = std::max(rm - r0, 0), n_blocks = (int)ceil_div(r1 - s0, h->ring_rows);
  auto resident_piece = [&](int p) -> int {        // piece p of n_blocks + 1
    const int a = r0 + (int)((int64_t)n_res * p / (n_blocks + 1)), b = r0 + (int)((int64_t)n_res * (p + 1) / (n_blocks + 1));
    return a < b ? launch(a, b, dev) : TGB200_OK;
  };
  CK(cudaEventRecord(h->ev_start, s));
  CK(cudaStreamWaitEvent(h->cin, h->ev_start, 0));
  if (h->ring_used) CK(cudaStreamWaitEvent(h->cin, h->ev_last, 0));
  int k = 0;
  for (int b0 = s0; b0 < r1; b0 += h->ring_rows, ++k) {
    const int b1 = std::min(r1, b0 + h->ring_rows), sl = k & 1;
    const size_t off = (size_t)(b0 - h->R) * ld, n = (size_t)(b1 - b0) * ld;
    if (k >= 2) CK(cudaStreamWaitEvent(h->cin, h->ev_free[sl], 0));       // block k - 2 is done with this slot
    CK(cudaMemcpyAsync(h->rM[sl].p, h->Mh.p + off, n * sizeof(float), cudaMemcpyHostToDevice, h->cin));
    if (write) {
      if (h->bf16) CK(cudaMemcpyAsync(h->rmb[sl].p, h->mbh.p + off, n * sizeof(__nv_bfloat16), cudaMemcpyHostToDevice, h->cin));
      else CK(cudaMemcpyAsync(h->rm[sl].p, h->mh.p + off, n * sizeof(float), cudaMemcpyHostToDevice, h->cin));
      CK(cudaMemcpyAsync(h->rv[sl].p, h->vh.p + off, n * sizeof(float), cudaMemcpyHostToDevice, h->cin));
    }
    CK(cudaEventRecord(h->ev_in[sl], h->cin));
    CKS(resident_piece(k));
    CK(cudaStreamWaitEvent(s, h->ev_in[sl], 0));
    CKS(launch(b0, b1, StagedPtrs{shifted(h->rM[sl].p, b0, ld), h->rm[sl].p ? shifted(h->rm[sl].p, b0, ld) : nullptr,
                                  h->rmb[sl].p ? shifted(h->rmb[sl].p, b0, ld) : nullptr, shifted(h->rv[sl].p, b0, ld)}));
    CK(cudaEventRecord(h->ev_comp[sl], s));
    if (write) {
      CK(cudaStreamWaitEvent(h->cout, h->ev_comp[sl], 0));
      CK(cudaMemcpyAsync(h->Mh.p + off, h->rM[sl].p, n * sizeof(float), cudaMemcpyDeviceToHost, h->cout));
      if (h->bf16) CK(cudaMemcpyAsync(h->mbh.p + off, h->rmb[sl].p, n * sizeof(__nv_bfloat16), cudaMemcpyDeviceToHost, h->cout));
      else CK(cudaMemcpyAsync(h->mh.p + off, h->rm[sl].p, n * sizeof(float), cudaMemcpyDeviceToHost, h->cout));
      CK(cudaMemcpyAsync(h->vh.p + off, h->rv[sl].p, n * sizeof(float), cudaMemcpyDeviceToHost, h->cout));
      CK(cudaEventRecord(h->ev_free[sl], h->cout));
    } else {
      CK(cudaEventRecord(h->ev_free[sl], s));
    }
  }
  CKS(resident_piece(n_blocks));
  // everything of this pass: the last kernel on s and, for a write pass, the copy-outs (cout is in order)
  if (write) CK(cudaEventRecord(h->ev_last, h->cout));
  else CK(cudaEventRecord(h->ev_last, s));
  CK(cudaStreamWaitEvent(s, h->ev_last, 0));
  h->ring_used = true;
  return TGB200_OK;
}

static int zero_moments(tgb200_mapper* h, cudaStream_t s) {
  if (h->bf16) CKS(zero_state(h, h->mb, h->mbh, s));
  else CKS(zero_state(h, h->m, h->mh, s));
  CKS(zero_state(h, h->v, h->vh, s));
  return TGB200_OK;
}

static int reset_optimizer(tgb200_mapper* h, cudaStream_t s) {
  CKS(zero_moments(h, s));
  if (h->bf16) CK(cudaMemsetAsync(h->rcenter.p, 0, h->rcenter.n * sizeof(float), s));
  h->step = 0;
  h->hist_len = 0;
  h->in_step = false;
  h->p_state = PState::stale;
  h->fwd_ahead = false;
  return TGB200_OK;
}

// torch.optim.Adam([M], lr) is rebuilt by every Mapper.train call (mapping_optimizer.py:373, :607): fresh moments,
// bias correction restarts at t = 1.  M (and F), the history and the resident P are kept.
extern "C" int tgb200_reset_adam(tgb200_mapper* h, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (h->in_step) return fail(TGB200_ERR_STATE, "reset_adam inside a step");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(zero_moments(h, s));
  if (h->constrained) {
    CK(cudaMemsetAsync(h->mF.p, 0, h->mF.n * sizeof(float), s));
    CK(cudaMemsetAsync(h->vF.p, 0, h->vF.n * sizeof(float), s));
  }
  h->step = 0;
  return TGB200_OK;
}

// The loss over a subset of the training genes (one cross-validation fold): the handle then computes what a handle created
// on S[:, active], G[:, active] computes.  The per-voxel norms of G (lambda_g2) follow the mask; M, F, the Adam state and
// the history are kept.  An all-ones mask is no mask.
extern "C" int tgb200_set_loss_genes(tgb200_mapper* h, const uint8_t* active, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (h->in_step) return fail(TGB200_ERR_STATE, "set_loss_genes inside a step");
  int n = h->K;
  std::vector<float> flags;
  if (active) {
    flags.assign(h->Ke, 0.f);
    n = 0;
    for (int k = 0; k < h->K; ++k) {
      if (active[k] > 1) return fail(TGB200_ERR_INVALID, "active[%d] = %d, expected 0 or 1", k, (int)active[k]);
      flags[k] = (float)active[k];
      n += active[k];
    }
    if (n == 0) return fail(TGB200_ERR_INVALID, "no gene is active");
  }
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  h->masked = n < h->K;
  h->n_active = n;
  if (h->masked) {
    if (!h->gene_act.p) CKS(h->gene_act.alloc(h->Ke, false));
    CK(cudaMemcpyAsync(h->gene_act.p, flags.data(), sizeof(float) * h->Ke, cudaMemcpyHostToDevice, s));
  }
  if (h->have_expr) {
    k_row_norms<<<(unsigned)ceil_div(h->V, 8), 256, 0, s>>>(h->V, h->K, h->Ke, h->G.p, h->masked ? h->gene_act.p : nullptr, h->ngr.p);
    LAUNCH_CHECK("row_norms");
    CKS(gene_weights(h, s));
  }
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// The scratch of the validation's loss scalars (val_loss_params), allocated on first use and kept: never in the loop.
static int alloc_validation(tgb200_mapper* h) {
  if (!h->val_coef.p) CKS(h->val_coef.alloc(2 * (size_t)h->Ke + 2 * (size_t)h->V));
  if (!h->val_hist.p) CKS(h->val_hist.alloc(TGB200_HIST_COLS));
  if (!h->rowpart.p && !h->val_rowpart.p) CKS(h->val_rowpart.alloc((size_t)h->ncolchunk * h->V * 2));
  return TGB200_OK;
}

// A sharded handle validates only with a communicator of its own to sum the validation forward's [Y_ext | tail] on (a
// caller-driven exchange has no slot for a second all-reduce), and only in plain mode.
static int check_validation_supported(const tgb200_mapper* h) {
  if (h->cfg.n_cells_global == h->N) return TGB200_OK;
  if (h->constrained) return fail(TGB200_ERR_UNSUPPORTED, "validation on a sharded constrained handle");
  if (!h->comm) return fail(TGB200_ERR_UNSUPPORTED, "validation on a sharded handle without a communicator");
  return TGB200_OK;
}

// Per-epoch validation inside tgb200_run / step_end (Mapper.train(val_each=), mapping_optimizer.py:398-403).
extern "C" int tgb200_set_validation(tgb200_mapper* h, int32_t every, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (every < 0) return fail(TGB200_ERR_INVALID, "every = %d < 0", every);
  if (h->in_step) return fail(TGB200_ERR_STATE, "set_validation inside a step");
  if (every > 0) CKS(check_validation_supported(h));
  CK(cudaSetDevice(h->cfg.device));
  if (every > 0) CKS(alloc_validation(h));
  (void)stream;                                      // nothing is queued: the switch takes effect at the next step
  h->val_every = every;
  h->val_epoch = 0;
  h->val_row = -1;
  return TGB200_OK;
}

extern "C" int tgb200_set_mapping(tgb200_mapper* h, const float* M0, void* stream) {
  if (!h || !M0) return fail(TGB200_ERR_INVALID, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(zero_state(h, h->M, h->Mh, s));
  CKS(state_parts(h, [&](int r0, int r1) -> int {
    CK(cudaMemcpy2DAsync(state_row(h, h->M, h->Mh, r0), (size_t)h->ld * sizeof(float), M0 + (size_t)r0 * h->V,
                         (size_t)h->V * sizeof(float), (size_t)h->V * sizeof(float), r1 - r0, cudaMemcpyDefault, s));
    return TGB200_OK;
  }));
  CKS(reset_optimizer(h, s));
  h->have_mapping = true;
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_set_filter(tgb200_mapper* h, const float* F0, void* stream) {
  if (!h || !F0) return fail(TGB200_ERR_INVALID, "null argument");
  if (!h->constrained) return fail(TGB200_ERR_INVALID, "handle was not created in constrained mode");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpyAsync(h->Fl.p, F0, h->N * sizeof(float), cudaMemcpyDefault, s));
  CK(cudaMemsetAsync(h->mF.p, 0, h->N * sizeof(float), s));
  CK(cudaMemsetAsync(h->vF.p, 0, h->N * sizeof(float), s));
  h->have_filter = true;
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_get_filter(tgb200_mapper* h, float* F_out, float* f_out, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (!h->constrained || !h->have_filter) return fail(TGB200_ERR_STATE, "no filter on this handle");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  if (F_out) CK(cudaMemcpyAsync(F_out, h->Fl.p, h->N * sizeof(float), cudaMemcpyDefault, s));
  if (f_out) {
    k_sigmoid<<<(unsigned)ceil_div(h->N, 256), 256, 0, s>>>(h->Fl.p, h->N, h->fsig.p);     // :638
    LAUNCH_CHECK("sigmoid");
    CK(cudaMemcpyAsync(f_out, h->fsig.p, h->N * sizeof(float), cudaMemcpyDefault, s));
  }
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_init_mapping_normal(tgb200_mapper* h, uint64_t seed, void* stream) {
  return tgb200_init_mapping_normal_rows(h, seed, 0, stream);
}

extern "C" int tgb200_init_mapping_normal_rows(tgb200_mapper* h, uint64_t seed, int64_t first_row, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (first_row < 0) return fail(TGB200_ERR_INVALID, "first_row < 0");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(state_parts(h, [&](int r0, int r1) -> int {      // the device rows and the host rows: the same draw per global row
    const long long nq = (long long)(r1 - r0) * (h->ld / 4);
    k_init_normal<<<(unsigned)ceil_div(nq, 256), 256, 0, s>>>(state_row(h, h->M, h->Mh, r0), r1 - r0, h->V, h->ld, seed,
                                                                 (long long)first_row + r0);
    LAUNCH_CHECK("init_normal");
    return TGB200_OK;
  }));
  CKS(reset_optimizer(h, s));
  h->have_mapping = true;
  return TGB200_OK;
}

// ---------------------------------------------------------------------------------------
// numpy's legacy normal stream on the device (legacy_rng.cuh; skip-ahead in mt19937_jump.h)

static bool valid_mt_state(const tgb200_mt_state* st) {
  return st->pos >= 0 && st->pos <= mtj::kN && (st->has_gauss == 0 || st->has_gauss == 1);
}

static int check_jump_args(const tgb200_mt_state* in, const tgb200_mt_state* out) {
  if (!in || !out) return fail(TGB200_ERR_INVALID, "null argument");
  if (!valid_mt_state(in)) return fail(TGB200_ERR_INVALID, "bad generator state (pos %d, has_gauss %d)", in->pos, in->has_gauss);
  if (!mtj::field().ok()) return fail(TGB200_ERR_STATE, "MT19937 characteristic polynomial not found");
  return TGB200_OK;
}

extern "C" int tgb200_mt19937_jump(const tgb200_mt_state* in, uint64_t n_words, tgb200_mt_state* out) {
  CKS(check_jump_args(in, out));
  tgb200_mt_state r = *in;
  if (n_words) mtj::jump(in->key, in->pos, (unsigned __int128)n_words - 1, r.key, &r.pos);
  *out = r;
  return TGB200_OK;
}

extern "C" int tgb200_mt19937_jump_pow2(const tgb200_mt_state* in, uint32_t log2_words, tgb200_mt_state* out) {
  if (log2_words > 128) return fail(TGB200_ERR_INVALID, "log2_words > 128");
  CKS(check_jump_args(in, out));
  const unsigned __int128 n_minus_1 = log2_words == 128 ? ~(unsigned __int128)0 : ((unsigned __int128)1 << log2_words) - 1;
  tgb200_mt_state r = *in;
  mtj::jump(in->key, in->pos, n_minus_1, r.key, &r.pos);
  *out = r;
  return TGB200_OK;
}

// numpy's legacy_gauss on the four words of one accepted attempt, with libm's log and sqrt: the value numpy computes in
// this process.  comp 0 is f x2 (returned first), 1 is f x1 (cached).  The squares go through volatile temporaries so
// that no compiler contracts x1 x1 + x2 x2 into an FMA; every other product is exact or cannot be contracted.
static double polar_value_host(const uint32_t w[4], int comp) {
  const double d1 = ((w[0] >> 5) * 67108864.0 + (w[1] >> 6)) / 9007199254740992.0;
  const double d2 = ((w[2] >> 5) * 67108864.0 + (w[3] >> 6)) / 9007199254740992.0;
  const double x1 = 2.0 * d1 - 1.0, x2 = 2.0 * d2 - 1.0;
  volatile double s1 = x1 * x1, s2 = x2 * x2;
  const double r2 = s1 + s2;
  const double f = std::sqrt(-2.0 * std::log(r2) / r2);
  return f * (comp ? x1 : x2);
}

// Jump polynomials of the device draw, computed once per process and kept: [0] x^(L - 624), [1 + j] x^(2^j L) for the
// draw-block length L.  *ms: host time spent here (phi included when this call found it).
static int legacy_polys(int levels, std::vector<uint64_t>& flat, double* ms) {
  static std::mutex mu;
  static std::vector<std::vector<uint64_t>> polys;
  std::lock_guard<std::mutex> lock(mu);
  const auto t0 = std::chrono::steady_clock::now();
  const mtj::Field& F = mtj::field();
  if (!F.ok()) return fail(TGB200_ERR_STATE, "MT19937 characteristic polynomial not found");
  if (polys.empty()) {
    polys.push_back(F.x_pow(lrng::kWordsPerCta - lrng::kN));
    polys.push_back(F.x_pow(lrng::kWordsPerCta));
  }
  while ((int)polys.size() < 1 + levels) {
    std::vector<uint64_t> p = polys.back();
    F.square(p);
    polys.push_back(std::move(p));
  }
  flat.clear();
  for (int i = 0; i < 1 + levels; ++i) flat.insert(flat.end(), polys[i].begin(), polys[i].end());
  *ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return TGB200_OK;
}

struct EventSet {
  cudaEvent_t e[5] = {};
  ~EventSet() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
  float ms(int a, int b) const { float t = 0.f; cudaEventElapsedTime(&t, e[a], e[b]); return t; }
};

extern "C" int tgb200_init_mapping_legacy(tgb200_mapper* h, const tgb200_mt_state* start, int64_t skip, int64_t first_row,
                                          int64_t end_normal, tgb200_mt_state* end_out, int64_t* n_fixed_out, void* stream) {
  using namespace lrng;
  if (!h || !start) return fail(TGB200_ERR_INVALID, "null argument");
  if (!valid_mt_state(start))
    return fail(TGB200_ERR_INVALID, "bad generator state (pos %d, has_gauss %d)", start->pos, start->has_gauss);
  if (skip < 0 || first_row < 0) return fail(TGB200_ERR_INVALID, "skip and first_row must be >= 0");
  const int64_t V = h->V, N = h->N;
  const int64_t t_lo = skip + first_row * V, t_hi = t_lo + N * V;       // stream normals that land in this handle
  if (end_normal < t_hi) return fail(TGB200_ERR_INVALID, "end_normal < skip + (first_row + n_cells) * n_voxels");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  const int hg = start->has_gauss;
  const int64_t a_end = end_normal > hg ? (end_normal - hg + 1) / 2 - 1 : -1;   // last accepted attempt consumed
  const int64_t a_lo = t_lo > hg ? (t_lo - hg) / 2 : 0;                        // first one this handle needs
  float* stats = h->legacy_stats;
  std::fill(stats, stats + 8, 0.f);
  EventSet ev;
  for (cudaEvent_t& e : ev.e) CK(cudaEventCreate(&e));
  CKS(zero_state(h, h->M, h->Mh, s));
  EndRecord end_h{-1, {0, 0, 0, 0}};
  int64_t n_fixed = 0, n_changed = 0;
  std::vector<float> patch_vals;
  if (a_end >= 0) {
    CK(cudaFuncSetAttribute(k_mt_jump, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kJumpSmem));   // per device
    // draw blocks: the expected attempts (a_end + 1) / (pi / 4) plus 10 standard deviations; doubled if ever short
    const double pa = 0.78539816339744831, na = (double)(a_end + 1);
    int64_t nb = (int64_t)((na / pa + 10.0 * std::sqrt(na * (1.0 - pa)) / pa) / kAttemptsPerCta) + 2;
    DevBuf<uint32_t> key0, starts;
    DevBuf<uint64_t> polys;
    DevBuf<long long> counts, offs;
    CKS(key0.alloc(kN, false));
    CK(cudaMemcpy(key0.p, start->key, kN * sizeof(uint32_t), cudaMemcpyHostToDevice));
    std::vector<long long> offs_h;
    std::vector<uint64_t> flat;
    DrawParams p{};
    p.key0 = key0.p;
    p.pos0 = start->pos;
    p.t_lo = t_lo;
    p.t_hi = t_hi;
    p.has_gauss = hg;
    p.V = h->V;
    p.ld = h->ld;
    p.M = h->M.p;
    p.Mh = h->Mh.p;
    p.split = (long long)h->R * h->ld;
    p.a_end = a_end;
    for (;;) {
      if (nb > (1LL << 30)) return fail(TGB200_ERR_INVALID, "draw of %lld normals is too large", (long long)end_normal);
      int levels = 0;
      while ((1LL << levels) + 1 < nb) ++levels;
      double host_ms = 0.0;
      CKS(legacy_polys(levels, flat, &host_ms));
      stats[4] += (float)host_ms;
      CKS(polys.alloc(flat.size(), false));
      CK(cudaMemcpy(polys.p, flat.data(), flat.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
      CKS(starts.alloc((size_t)nb * kN, false));
      CKS(counts.alloc(nb, false));
      CKS(offs.alloc(nb + 1, false));
      CK(cudaEventRecord(ev.e[0], s));
      // level -1: start 1 = the window 624 words before MT block B + kBlocksPerCta; level j: starts
      // [1 + 2^j, 1 + 2^(j+1)) = starts [1, 1 + 2^j) jumped by 2^j draw blocks
      if (nb > 1) {
        CK(cudaMemcpyAsync(starts.p, key0.p, kN * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
        k_mt_jump<<<1, kN, kJumpSmem, s>>>(starts.p, starts.p + kN, polys.p);
        LAUNCH_CHECK("mt_jump");
        for (int j = 0; j < levels; ++j) {
          const int64_t stride = 1LL << j, cnt = std::min<int64_t>(stride, nb - 1 - stride);
          k_mt_jump<<<(unsigned)cnt, kN, kJumpSmem, s>>>(starts.p + kN, starts.p + (1 + stride) * kN,
                                                          polys.p + (size_t)(1 + j) * kPolyWords);
          LAUNCH_CHECK("mt_jump");
        }
      }
      CK(cudaEventRecord(ev.e[1], s));
      p.starts = starts.p;
      p.counts = counts.p;
      p.offs = offs.p;
      k_legacy_pass<false><<<(unsigned)nb, kN, 0, s>>>(p);
      LAUNCH_CHECK("legacy_count");
      k_scan_counts<<<1, 1024, 0, s>>>(counts.p, (int)nb, offs.p);
      LAUNCH_CHECK("legacy_scan");
      CK(cudaEventRecord(ev.e[2], s));
      offs_h.resize(nb + 1);
      CK(cudaMemcpyAsync(offs_h.data(), offs.p, (nb + 1) * sizeof(long long), cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      if (offs_h[nb] > a_end) break;
      nb *= 2;
    }
    stats[5] = (float)nb;
    // draw blocks [b_lo, b_hi] hold accepted attempts a_lo .. a_end
    const int64_t b_lo = std::upper_bound(offs_h.begin(), offs_h.end(), (long long)a_lo) - offs_h.begin() - 1;
    const int64_t b_hi = std::upper_bound(offs_h.begin(), offs_h.end(), (long long)a_end) - offs_h.begin() - 1;
    const int flag_cap = (int)std::min<int64_t>(4096 + ((N * V) >> 16), 1 << 24);
    DevBuf<Flagged> flags;
    DevBuf<int> n_flags;
    DevBuf<EndRecord> end_d;
    CKS(flags.alloc(flag_cap, false));
    CKS(n_flags.alloc(1, true));
    CKS(end_d.alloc(1, true));
    p.b_first = (int)b_lo;
    p.end = end_d.p;
    p.flags = flags.p;
    p.n_flags = n_flags.p;
    p.flag_cap = flag_cap;
    k_legacy_pass<true><<<(unsigned)(b_hi - b_lo + 1), kN, 0, s>>>(p);
    LAUNCH_CHECK("legacy_emit");
    CK(cudaEventRecord(ev.e[3], s));
    int nf = 0;
    CK(cudaMemcpyAsync(&nf, n_flags.p, sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(&end_h, end_d.p, sizeof(EndRecord), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (nf > flag_cap) return fail(TGB200_ERR_STATE, "%d values near a float32 rounding midpoint (room for %d)", nf, flag_cap);
    if (end_h.attempt < 0) return fail(TGB200_ERR_STATE, "legacy draw: the last attempt was not found");
    // host fix-up: libm's log for every value whose float32 rounding could depend on the last bit of log
    std::vector<Flagged> fl(nf);
    std::vector<float> dev_vals(nf);
    if (nf) CK(cudaMemcpy(fl.data(), flags.p, nf * sizeof(Flagged), cudaMemcpyDeviceToHost));
    auto elem = [&](long long idx) { return state_row(h, h->M, h->Mh, idx / h->ld) + idx % h->ld; };
    for (int i = 0; i < nf; ++i) CK(cudaMemcpyAsync(&dev_vals[i], elem(fl[i].idx), sizeof(float), cudaMemcpyDefault, s));
    CK(cudaStreamSynchronize(s));
    patch_vals.resize(nf);
    for (int i = 0; i < nf; ++i) {
      patch_vals[i] = (float)polar_value_host(fl[i].w, fl[i].comp);
      if (std::memcmp(&patch_vals[i], &dev_vals[i], sizeof(float)) != 0) {
        CK(cudaMemcpyAsync(elem(fl[i].idx), &patch_vals[i], sizeof(float), cudaMemcpyDefault, s));
        ++n_changed;
      }
    }
    n_fixed = nf;
  }
  float cached = (float)start->gauss;
  if (hg && t_lo == 0) CK(cudaMemcpyAsync(state_row(h, h->M, h->Mh, 0), &cached, sizeof(float), cudaMemcpyDefault, s));   // normal 0
  if (a_end >= 0) CK(cudaEventRecord(ev.e[4], s));
  CKS(reset_optimizer(h, s));
  h->have_mapping = true;
  CK(cudaStreamSynchronize(s));
  if (a_end >= 0) {
    stats[0] = ev.ms(0, 1);
    stats[1] = ev.ms(1, 2);
    stats[2] = ev.ms(2, 3);
    stats[3] = ev.ms(3, 4);
  }
  stats[6] = (float)n_fixed;
  stats[7] = (float)n_changed;
  if (end_out) {
    tgb200_mt_state e = *start;
    e.has_gauss = 0;
    e.gauss = 0.0;
    if (a_end >= 0) {                          // 4 (attempt + 1) words consumed; an odd count leaves f x1 cached
      mtj::jump(start->key, start->pos, (unsigned __int128)(4 * end_h.attempt + 3), e.key, &e.pos);
      if ((end_normal - hg) & 1) {
        e.has_gauss = 1;
        e.gauss = polar_value_host(end_h.w, 1);
      }
    }
    *end_out = e;
  }
  if (n_fixed_out) *n_fixed_out = n_fixed;
  return TGB200_OK;
}

// ---------------------------------------------------------------------------------------
// rows [row0, row0 + nrows) of M -> P (row 0 of `P` is row `row0` of the mapping when P is a scratch block)
template <typename PT>
static int launch_softmax_rows(tgb200_mapper* h, cudaStream_t s, PT* P, int want_entropy, float* rowaux,
                               Split3 split = Split3{nullptr, 0}, int row0 = 0, int nrows = -1) {
  const int nvec = h->ld / 4;
  if (nrows < 0) nrows = h->N - row0;
  // rows [b0, b1): one launch over the resident M, or one per ring block of host state (`o` rows into P / rowaux / split)
  auto rows = [&](int b0, int b1, const StagedPtrs& sp) -> int {
    const int nr = b1 - b0;
    const size_t o = (size_t)(b0 - row0);
    const float* Mp = sp.M + (size_t)b0 * h->ld;
    RowStat* st = h->stats.p + b0;
    PT* Po = P ? P + o * h->ld : nullptr;
    float* ra = rowaux ? rowaux + 2 * o : nullptr;
    Split3 sp3 = split;
    if (sp3.base) sp3.base += o * h->ld;
    // One CTA per row, the row cached in registers between the max / exp-sum / emit passes.  Wide rows use more threads
    // with fewer float4 slots each: registers/thread stay <= 40..64, so 48-64 warps stay resident per SM (256 x 12 slots
    // held 24, and the row pass was latency-bound at 0.46 of the HBM peak).  Rows wider than 6144 float4 re-read M.
#define SMX(T, ITEMS, MINB)                                                                         \
  k_softmax_rows<PT, T, ITEMS, MINB><<<nr, T, 0, s>>>(Mp, h->ld, h->V, Po, h->ld, st, ra, want_entropy, sp3)
    if (nvec <= 256 * 1) SMX(256, 1, 1);
    else if (nvec <= 256 * 2) SMX(256, 2, 1);
    else if (nvec <= 256 * 4) SMX(256, 4, 1);
    else if (nvec <= 512 * 3) SMX(512, 3, 3);
    else if (nvec <= 512 * 4) SMX(512, 4, 3);
    else if (nvec <= 512 * 5) SMX(512, 5, 3);
    else if (nvec <= 1024 * 3) SMX(1024, 3, 2);
    else if (nvec <= 1024 * 4) SMX(1024, 4, 1);
    else if (nvec <= 1024 * 6) SMX(1024, 6, 1);
    else SMX(1024, 0, 1);
#undef SMX
    LAUNCH_CHECK("softmax_rows");
    return TGB200_OK;
  };
  return staged_rows(h, s, row0, row0 + nrows, false, rows);
}

static LossParams make_loss_params(tgb200_mapper* h) {
  LossParams p;
  memset(&p, 0, sizeof(p));
  const tgb200_config& c = h->cfg;
  p.V = h->V; p.K = h->K; p.Ke = h->Ke; p.T = h->T; p.ct_off = h->ct_off; p.density_mode = c.density_mode;
  p.act = h->masked ? h->gene_act.p : nullptr; p.Kact = h->n_active;
  p.n_cells_global = c.n_cells_global;
  p.lam_g1 = c.lambda_g1; p.lam_d = c.lambda_d; p.lam_g2 = c.lambda_g2; p.lam_r = c.lambda_r;
  p.lam_l1 = c.lambda_l1; p.lam_l2 = c.lambda_l2; p.lam_nb = c.lambda_neighborhood_g1;
  p.lam_ct = c.lambda_ct_islands; p.lam_go = c.lambda_getis_ord;
  p.G = h->G.p; p.d = h->d.p; p.Y = h->Y.p; p.ngc = h->ngc.p; p.ngr = h->ngr.p;
  p.W = h->W.view(); p.WT = h->WT.view(); p.F = h->F.view(); p.FT = h->FT.view(); p.A = h->A.view(); p.AT = h->AT.view();
  p.WG = h->WG.p; p.nwg = h->nwg.p; p.AG = h->AG.p; p.nag = h->nag.p; p.sgnG = h->sgnG.p;
  p.Z = h->Z.p; p.Zg = h->Zg.p; p.H = h->H.p;
  p.colpart = h->colpart.p; p.colpart_nb = h->colpart_nb.p; p.colpart_go = h->colpart_go.p;
  p.rowpart = h->rowpart.p; p.ctpart = h->ctpart.p; p.n_ct_blocks = h->n_ct_blocks;
  p.coefA = h->coefA.p; p.coefB = h->coefB.p; p.coefAn = h->coefAn.p; p.coefBn = h->coefBn.p;
  p.coefAg = h->coefAg.p; p.coefBg = h->coefBg.p; p.coefAr = h->coefAr.p; p.coefBr = h->coefBr.p;
  p.densg = h->densg.p;
  p.constrained = h->constrained ? 1 : 0;
  p.lam_c = c.lambda_count; p.lam_f = c.lambda_f_reg; p.target_count = c.target_count; p.fscal = h->fscal.p;
  return p;
}

static int check_ready(tgb200_mapper* h) {
  const tgb200_config& c = h->cfg;
  if (!h->have_expr) return fail(TGB200_ERR_STATE, "tgb200_set_expression has not been called");
  if (!h->have_mapping) return fail(TGB200_ERR_STATE, "no mapping: call tgb200_set_mapping or tgb200_init_mapping_normal");
  if (c.density_mode != TGB200_DENSITY_NONE && !h->have_density) return fail(TGB200_ERR_STATE, "density term enabled but tgb200_set_density not called");
  if (c.lambda_ct_islands > 0.f && (!h->have_ct || !h->F.set)) return fail(TGB200_ERR_STATE, "lambda_ct_islands > 0 needs ct_encode and the neighborhood_filter graph");
  if (c.lambda_neighborhood_g1 > 0.f && !h->W.set) return fail(TGB200_ERR_STATE, "lambda_neighborhood_g1 > 0 needs the voxel_weights graph");
  if (c.lambda_getis_ord > 0.f && !h->A.set) return fail(TGB200_ERR_STATE, "lambda_getis_ord > 0 needs the spatial_weights graph");
  if (h->constrained && !h->have_filter) return fail(TGB200_ERR_STATE, "constrained mode: call tgb200_set_filter first");
  return TGB200_OK;
}

// The streams of one API call, chosen once at its start.  On a handle with streams the caller's stream forks into `work`
// (hi: forward, loss, backward contractions), which feeds `update` (lo: row-dot finalize, streaming Adam) and `ahead`
// (sf: the next iteration's forward chunks) through per-chunk events, and all three join the caller's stream at the end.
// Otherwise, and in tgb200_profile_step, every lane is the caller's stream.
struct Lanes { cudaStream_t caller, work, update, ahead; };
static Lanes lanes_of(const tgb200_mapper* h, cudaStream_t s) {
  return h->pipelined ? Lanes{s, h->hi, h->lo, h->sf} : Lanes{s, s, s, s};
}
static int fork_streams(tgb200_mapper* h, const Lanes& L) {
  if (L.work == L.caller) return TGB200_OK;
  CK(cudaEventRecord(h->ev_fork, L.caller));
  CK(cudaStreamWaitEvent(L.work, h->ev_fork, 0));
  return TGB200_OK;
}
static int join_streams(tgb200_mapper* h, const Lanes& L) {
  if (L.work == L.caller) return TGB200_OK;
  CK(cudaEventRecord(h->ev_join_hi, L.work));
  CK(cudaStreamWaitEvent(L.caller, h->ev_join_hi, 0));
  CK(cudaEventRecord(h->ev_join_lo, L.update));
  CK(cudaStreamWaitEvent(L.caller, h->ev_join_lo, 0));
  CK(cudaEventRecord(h->ev_join_sf, L.ahead));
  CK(cudaStreamWaitEvent(L.caller, h->ev_join_sf, 0));
  return TGB200_OK;
}

// the tensor maps of the forward contraction, encoded on first use (the buffers never move)
static int forward_plan(tgb200_mapper* h) {
  if (h->plan_fwd.ready) return TGB200_OK;
  const __nv_bfloat16* sB = h->bf16 ? h->Sxs.p : h->Sxb.p;
  return tc_forward_plan(h->tc, h->plan_fwd, h->Pb.p, (size_t)h->N * h->ld, sB, (size_t)h->N * h->Ke, h->x3 ? 3 : 1, h->N, h->V,
                         h->Ke, h->ld, g_err, sizeof(g_err));
}

// bf16 mode, cells of chunk c: exact row statistics from the sums the update left (k_row_norm), the scaled forward operand,
// and -- when the forward is chunked -- this chunk's contribution to Y_ext.  `lseA` / `lseT` as they are for THAT forward.
// `keep_sms`: SMs the contraction leaves to an update chunk running beside it (tc_launch).
static int forward_chunk(tgb200_mapper* h, cudaStream_t s, int c, int fresh, const float* lseA, float* lseT, int keep_sms) {
  float* rowaux = needs_rowaux(h->cfg) ? h->rowaux.p : nullptr;
  CKS(forward_plan(h));
  const int r0 = h->chunk_row[c], r1 = h->chunk_row[c + 1];
  // rows of this chunk: the streaming Adam kernel of the previous iteration must have written their P and row sums (on
  // the caller's stream, after the join of the call that ran it, the wait is already satisfied)
  if (h->a_valid) CK(cudaStreamWaitEvent(s, h->ev_a[c], 0));
  k_row_norm<<<(unsigned)ceil_div(r1 - r0, 256), 256, 0, s>>>(fresh, h->zsum.p, h->pxsum.p, h->l1sum.p, h->l2sum.p,
                                                             lseA, lseT, h->inv_zt.p, h->stats.p, rowaux, r0, r1);
  LAUNCH_CHECK("row_norm");
  const long long nq = (long long)(r1 - r0) * (h->Ke / 4);
  k_scale_rows_bf16<<<(unsigned)ceil_div(nq, 256), 256, 0, s>>>(s_act(h), h->inv_zt.p, r0, r1, h->Ke, h->Sxs.p);
  LAUNCH_CHECK("scale_rows");
  if (h->nchunks > 1) {
    // chunk 0 overwrites the exchange buffer, the others add to it (same stream, fixed order): no partial planes to sum
    CKS(tc_forward_launch_rows(h->tc, h->plan_fwd, 1, h->Y.p, c > 0 ? 1 : 0, r0, r1, h->V, h->Ke, keep_sms, s, g_err, sizeof(g_err)));
    mark(h, s, "tc_gemm_fwd");
  }
  return TGB200_OK;
}

// forward: P, row statistics, Y_ext partial sums over this handle's cells
static int forward_pass(tgb200_mapper* h, cudaStream_t s, int want_entropy) {
  float* rowaux = needs_rowaux(h->cfg) ? h->rowaux.p : nullptr;
  if (h->bf16) {
    // The row pass runs only when P is not already resident (first iteration / after a state load):
    // in steady state the previous backward epilogue has written P and its row sums.
    if (h->p_state == PState::stale) {
      CKS(launch_softmax_rows<__nv_bfloat16>(h, s, h->Pb.p, 1, rowaux));
      h->p_state = PState::fresh;
    }
    if (h->fwd_ahead) {           // issued by the previous iteration's backward (forward_chunk under the streaming Adam kernel)
      h->fwd_ahead = false;
      for (int c = 0; c < h->nchunks; ++c) CK(cudaStreamWaitEvent(s, h->ev_f[c], 0));
    } else {
      for (int c = 0; c < h->nchunks; ++c) CKS(forward_chunk(h, s, c, h->p_state == PState::fresh ? 1 : 0, h->lseA, h->lseT, 0));
    }
    if (h->nchunks > 1) return TGB200_OK;
  } else if (h->x3) {
    // parity mode on tensor cores: exact row pass every iteration, P written as three bf16 planes
    CKS(launch_softmax_rows<float>(h, s, (float*)nullptr, want_entropy, rowaux, Split3{h->Pb.p, (size_t)h->N * h->ld}));
  } else {
    CKS(launch_softmax_rows<float>(h, s, h->Pf.p, want_entropy, rowaux));
  }
  const size_t vk = (size_t)h->V * h->Ke;
  float* out = h->fwd_splits > 1 ? h->Ypart.p : h->Y.p;
  if (h->tcm) {
    CKS(forward_plan(h));
    CKS(tc_forward_launch(h->tc, h->plan_fwd, h->x3 ? 6 : 1, out, h->N, h->V, h->Ke, h->fwd_splits, s, g_err, sizeof(g_err)));
    mark(h, s, "tc_gemm_fwd");
  } else {
    GemmArgs g;
    g.A = h->Pf.p; g.lda = h->ld; g.B = s_act(h); g.ldb = h->Ke;
    g.M = h->V; g.N = h->Ke; g.K = h->N;
    g.k_per_split = (int)round_up(ceil_div(h->N, h->fwd_splits), 16);
    EpiStorePartial epi{out, h->Ke, vk};
    dim3 grid((unsigned)ceil_div(h->Ke, SG_BN), (unsigned)ceil_div(h->V, SG_BM), h->fwd_splits);
    k_gemm_simt<false, false, EpiStorePartial><<<grid, SG_THREADS, 0, s>>>(g, epi);
    LAUNCH_CHECK("simt_gemm_fwd");
  }
  return TGB200_OK;
}

// sharded: the exchange buffer must hold this rank's complete partial sum of Y_ext, not the forward's partial planes
static int sum_forward_planes(tgb200_mapper* h, cudaStream_t s) {
  if (h->cfg.n_cells_global == h->N || h->fwd_splits <= 1) return TGB200_OK;
  const size_t vk = (size_t)h->V * h->Ke;
  k_sum_planes<<<(unsigned)ceil_div(vk, 256), 256, 0, s>>>(h->Ypart.p, h->fwd_splits, vk, h->Y.p);
  LAUNCH_CHECK("sum_planes");
  return TGB200_OK;
}

// first half of an iteration, up to the exchange buffer: the forward and the row-scalar partials
static int iteration_begin(tgb200_mapper* h, const Lanes& L) {
  cudaStream_t s = L.work;
  if (h->constrained) {
    // f = sigmoid(F), S_f = f o S_ext (:507, :519) and the operand copies the contractions read
    const long long nq = (long long)h->N * (h->Ke / 4);
    k_filter_prepare<<<(unsigned)ceil_div(nq, 256), 256, 0, s>>>(h->Fl.p, h->Sx.p, h->N, h->Ke, h->fsig.p, h->Sf.p);
    LAUNCH_CHECK("filter_prepare");
    CKS(refresh_bf16_operands(h, s));
  }
  // a pending validation (fp32 / bf16x3) needs the row entropies of this forward; P is the same bits either way
  const bool val = h->val_row >= 0;
  CKS(forward_pass(h, s, h->cfg.lambda_r != 0.f || val ? 1 : 0));
  const size_t vk = (size_t)h->V * h->Ke;
  const bool sharded = h->cfg.n_cells_global != h->N;
  const bool rows = needs_rowscalars(h->cfg) || h->constrained || val;
  if (rows || h->tail_stale) {
    // sharded: the pending validation's sum of entropies rides in tail[5], so that it is summed over ranks with Y_ext.
    // Without row data (only a stale tail to clear) every slot is written 0.
    k_row_scalar_reduce<<<1, 1024, 0, s>>>(rows ? h->stats.p : nullptr, needs_rowaux(h->cfg) ? h->rowaux.p : nullptr,
                                           h->constrained ? h->fsig.p : nullptr, h->N, val && sharded ? 1 : 0, h->Y.p + vk);
    LAUNCH_CHECK("row_scalar_reduce");
  }
  h->tail_stale = val && sharded;
  return sum_forward_planes(h, s);
}

extern "C" int tgb200_exchange_buffer(tgb200_mapper* h, float** device_ptr, int64_t* n_floats) {
  if (!h || !device_ptr || !n_floats) return fail(TGB200_ERR_INVALID, "null argument");
  *device_ptr = h->Y.p;
  *n_floats = (int64_t)h->V * h->Ke + kTail;
  return TGB200_OK;
}

static int ensure_history(tgb200_mapper* h, int64_t need, cudaStream_t s) {
  if (need <= h->hist_cap) return TGB200_OK;
  int64_t cap = h->hist_cap ? h->hist_cap : 1024;
  while (cap < need) cap *= 2;
  DevBuf<float> nb;
  CKS(nb.alloc((size_t)cap * TGB200_HIST_COLS));
  if (h->hist_len > 0) {
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(nb.p, h->hist.p, (size_t)h->hist_len * TGB200_HIST_COLS * sizeof(float), cudaMemcpyDeviceToDevice));
  }
  h->hist.release();
  h->hist.p = nb.p; h->hist.n = nb.n; nb.p = nullptr; nb.n = 0;
  h->hist_cap = cap;
  return TGB200_OK;
}

// Y_ext (first summed over the forward's partial planes when `from_partials`) -> finalised per-gene sums in colfin;
// p.colpart then points at them for k_loss_scalars
static int reduce_columns(tgb200_mapper* h, cudaStream_t s, LossParams& p, bool from_partials, int with_g2) {
  const bool planes = from_partials && h->fwd_splits > 1;
  dim3 vgrid(h->nredchunk, h->nchunk);          // four columns per thread
  auto reduce = p.act ? k_loss_reduce<true> : k_loss_reduce<false>;
  reduce<<<vgrid, kLossCols, 0, s>>>(p, planes ? h->Ypart.p : h->Y.p, planes ? h->fwd_splits : 1, with_g2, h->loss_rows);
  LAUNCH_CHECK("loss_reduce");
  k_col_finalize<<<dim3((unsigned)ceil_div(h->Ke, 128), 3), 128, 0, s>>>(h->colpart.p, h->nchunk, 3, h->Ke, h->colfin.p);
  LAUNCH_CHECK("col_finalize");
  p.colpart = h->colfin.p;
  return TGB200_OK;
}

// per-voxel partials of the row cosine: the training's own when lambda_g2 != 0, the validation's otherwise
static float* any_rowpart(tgb200_mapper* h) { return h->rowpart.p ? h->rowpart.p : h->val_rowpart.p; }

// _val_loss_fn's parameters (:311-356): gene-voxel and voxel-gene cosines with weight 1,
// no other term; the four values go to `out` (device), everything else k_loss_scalars writes goes to the validation's own
// scratch, so the training's coefficients, dY and filter scalars are left alone
static LossParams val_loss_params(tgb200_mapper* h, float* out) {
  LossParams p = make_loss_params(h);
  p.rowpart = any_rowpart(h);
  p.coefA = h->val_coef.p; p.coefB = h->val_coef.p + h->Ke;
  p.coefAr = h->val_coef.p + 2 * (size_t)h->Ke; p.coefBr = p.coefAr + h->V;
  p.lam_g2 = 1.f; p.lam_g1 = 1.f; p.lam_nb = 0.f; p.lam_go = 0.f; p.lam_ct = 0.f; p.density_mode = 0;
  p.constrained = 0;
  p.gw = h->gw.p; p.val_out = out;
  p.val_log_v = logf((float)h->V); p.val_n = (float)h->cfg.n_cells_global;
  // sharded: sum h travels in its own tail slot ([0] stays the lambda_r term of the exchange); unsharded: [0], as it was
  p.val_ent = h->cfg.n_cells_global != h->N ? kTailValEntropy : 0;
  return p;
}

static float* val_out_of(tgb200_mapper* h, int64_t row) {
  return h->hist.p + (size_t)row * TGB200_HIST_COLS + TGB200_HIST_VAL_TOTAL;
}

// everything on V x Ke: reductions, scalars + history row, dY_ext.  With a validation pending (h->val_row, fp32 / bf16x3),
// this iteration's forward is the validation's forward: the same row pass (entropies requested) and the same contraction
// of the same mapping, so the validation only adds the row statistics and one k_loss_scalars.
static int loss_stage(tgb200_mapper* h, cudaStream_t s, float* hist_row, bool reduce_partials_first) {
  LossParams p = make_loss_params(h);
  const tgb200_config& c = h->cfg;
  const bool val = h->val_row >= 0;
  if (h->val_every > 0) p.hist_fill = NAN;
  if (val) p.rowpart = any_rowpart(h);
  dim3 rgrid(h->ncolchunk, h->nchunk);          // spatial kernels: one column per thread
  CKS(reduce_columns(h, s, p, reduce_partials_first, c.lambda_g2 != 0.f || val ? 1 : 0));
  const dim3 fgrid2((unsigned)ceil_div(h->Ke, 128), 2);
  if (c.lambda_neighborhood_g1 > 0.f) {
    k_spatial_colstats<<<rgrid, kLossCols, 0, s>>>(h->V, h->K, h->Ke, h->W.view(), h->Y.p, h->WG.p, h->Z.p, h->colpart_nb.p, h->loss_rows);
    LAUNCH_CHECK("spatial_colstats");
    k_col_finalize<<<fgrid2, 128, 0, s>>>(h->colpart_nb.p, h->nchunk, 2, h->Ke, h->colfin.p + (size_t)3 * h->Ke);
    LAUNCH_CHECK("col_finalize");
    p.colpart_nb = h->colfin.p + (size_t)3 * h->Ke;
  }
  if (c.lambda_getis_ord > 0.f) {
    k_spatial_colstats<<<rgrid, kLossCols, 0, s>>>(h->V, h->K, h->Ke, h->A.view(), h->Y.p, h->AG.p, h->Zg.p, h->colpart_go.p, h->loss_rows);
    LAUNCH_CHECK("spatial_colstats");
    k_col_finalize<<<fgrid2, 128, 0, s>>>(h->colpart_go.p, h->nchunk, 2, h->Ke, h->colfin.p + (size_t)5 * h->Ke);
    LAUNCH_CHECK("col_finalize");
    p.colpart_go = h->colfin.p + (size_t)5 * h->Ke;
  }
  if (c.lambda_ct_islands > 0.f) {
    k_ct_islands<<<h->n_ct_blocks, 256, 0, s>>>(p);
    LAUNCH_CHECK("ct_islands");
  }
  k_loss_scalars<false><<<1, 1024, 0, s>>>(p, 1, h->nredchunk, hist_row);
  LAUNCH_CHECK("loss_scalars");
  if (val) {
    LossParams pv = val_loss_params(h, val_out_of(h, h->val_row));
    pv.colpart = p.colpart;                             // the column sums reduce_columns finalised
    k_loss_scalars<true><<<1, 1024, 0, s>>>(pv, 1, h->nredchunk, h->val_hist.p);
    LAUNCH_CHECK("loss_scalars");
    h->val_row = -1;
  }
  dim3 dgrid(h->V, h->nredchunk);                       // voxels on x: gridDim.y is limited to 65535
  // fp32 dY_ext in fp32 mode (dY is not allocated otherwise), its bf16 copy or three bf16 planes on tensor cores
  k_dy_assemble<<<dgrid, kLossCols, 0, s>>>(p, h->dY.p, h->bf16 ? h->dYb.p : nullptr,
                                            h->x3 ? Split3{h->dYb.p, (size_t)h->V * h->Ke} : Split3{nullptr, 0});
  LAUNCH_CHECK("dy_assemble");
  return TGB200_OK;
}

// The double a caller wrote when it passed `f` through a float field: the shortest decimal that rounds to `f`
// (0.999f -> 0.999, not 0.99900001287...).  torch computes Adam's scalars from the Python doubles.
static double as_written(float f) {
  char buf[32];
  for (int digits = 1; digits <= 9; ++digits) {
    snprintf(buf, sizeof(buf), "%.*g", digits, (double)f);
    if (strtof(buf, nullptr) == f) return strtod(buf, nullptr);
  }
  return (double)f;
}

static AdamScalars adam_scalars(const tgb200_config& c, int64_t t, float lr) {
  // torch/optim/adam.py (_single_tensor_adam, non-capturable): python-double scalar math, each scalar cast to fp32 by the
  // kernel that takes it
  const double b1 = as_written(c.adam_beta1), b2 = as_written(c.adam_beta2);
  const double bc1 = 1.0 - std::pow(b1, (double)t), bc2 = 1.0 - std::pow(b2, (double)t);
  AdamScalars a;
  a.beta1 = c.adam_beta1; a.beta2 = c.adam_beta2;
  a.one_minus_beta1 = (float)(1.0 - b1); a.one_minus_beta2 = (float)(1.0 - b2);
  a.step_size = (float)(as_written(lr) / bc1);
  a.bc2_sqrt = (float)std::pow(bc2, 0.5);                       // bias_correction2 ** 0.5
  a.inv_bc2_sqrt = (float)(1.0 / std::pow(bc2, 0.5));          // torch divides by a Python scalar as a * fp32(1 / b)
  a.eps = c.adam_eps;
  return a;
}

static int filter_update(tgb200_mapper* h, cudaStream_t s, const AdamScalars& a) {
  k_filter_update<<<(unsigned)ceil_div(h->N, 256), 256, 0, s>>>(h->N, h->rdot.p, h->fsig.p, h->fscal.p, h->cfg.lambda_count,
                                                                 h->cfg.lambda_f_reg, a, h->Fl.p, h->mF.p, h->vF.p);
  LAUNCH_CHECK("filter_update");
  return TGB200_OK;
}

// Backward of the bf16 mode: dq = bf16(S_ext dY_ext^T - centre) + row-dot partials from the store-only contraction,
// then one streaming pass does softmax-Jacobian + Adam + the next forward's P.  (mapping_optimizer.py:395-396)
// `next_forward`: the next iteration of this call starts with a plain forward, which may then be issued ahead.
static int backward_bf16(tgb200_mapper* h, const Lanes& L, const AdamScalars& a, bool next_forward) {
  if (!h->plan_dp.ready) {
    CKS(tc_dpstore_epi_plan(h->tc, h->plan_dp, h->Pb.p, h->dq.p, h->N, h->ld, g_err, sizeof(g_err)));
    CKS(tc_dpstore_plan(h->tc, h->plan_dp, h->Sxb.p, 0, h->dYb.p, 0, 1, h->N, h->V, h->Ke, g_err, sizeof(g_err)));
  }
  cudaStream_t s = L.work, su = L.update;
  const bool two_streams = su != s;
  const bool prefetch = two_streams && next_forward;
  if (prefetch) CK(cudaEventRecord(h->ev_loss, s));                   // the loss stage has consumed the partial planes of Y_ext
  for (int c = 0; c < h->nchunks; ++c) {
    const int r0 = h->chunk_row[c], r1 = h->chunk_row[c + 1];
    TcEpiDpStore epi{h->plan_dp.pt, h->plan_dp.dq, h->ld, h->rcenter.p, h->rpart.p, h->N};
    // G(c) runs beside A(c - 1); G(0) follows the loss stage, which waited for every update of the previous iteration
    CKS(tc_dpstore_launch(h->tc, h->plan_dp, 1, epi, r0, r1, h->V, h->Ke, two_streams && c > 0 ? h->update_sms : 0, s, g_err,
                          sizeof(g_err)));
    mark(h, s, "tc_gemm_bwd_dp");
    if (two_streams) {
      CK(cudaEventRecord(h->ev_g[c], s));
      CK(cudaStreamWaitEvent(su, h->ev_g[c], 0));
    }
    k_rowdot_finalize_staged<<<(unsigned)ceil_div(r1 - r0, 256), 256, 0, su>>>(h->rpart.p, h->r_parts, h->N, r0, r1, h->lseT, h->inv_zt.p,
                                                                               h->stats.p, h->rcenter.p, h->rdot.p, h->rowc.p);
    { cudaStream_t s = su; LAUNCH_CHECK("rowdot_finalize"); }
    if (h->constrained) CKS(filter_update(h, su, a));
    // host state: the ring blocks nest inside the chunk, so chunk c's update still runs under chunk c+1's contraction
    CKS(staged_rows(h, su, r0, r1, true, [&](int b0, int b1, const StagedPtrs& sp) -> int {
      AdamRowsArgs ar{sp.M, sp.mb, sp.v, h->dq.p, h->Pb.p, reinterpret_cast<const RowConst*>(h->rowc.p),
                      h->zsum.p, h->pxsum.p, h->l1sum.p, h->l2sum.p, h->ld, h->V, b0, b1,
                      h->cfg.lambda_r, h->cfg.lambda_l1, h->cfg.lambda_l2, a};
      if (adam_rows_launch(ar, su)) return fail(TGB200_ERR_CUDA, "launch adam_rows: %s", cudaGetErrorString(cudaGetLastError()));
      mark(h, su, "adam_rows");
      return TGB200_OK;
    }));
    if (two_streams) CK(cudaEventRecord(h->ev_a[c], su));
    h->a_valid = two_streams;
    // The next iteration's forward for this chunk goes to a third stream as soon as its rows are updated: the backward
    // contractions G(c+1..) run ahead on `s` (they feed the update), the update stream is never without tensor-core work
    // beside it, and nothing queues behind a kernel that still waits for the update.
    // (lseT of this iteration is the offset the new P was written with = lseA of the next; the other buffer is free.)
    if (prefetch) {
      if (c == 0) CK(cudaStreamWaitEvent(L.ahead, h->ev_loss, 0));
      // F'(c) waits for A(c) and runs beside A(c + 1); the last one has no update left beside it
      CKS(forward_chunk(h, L.ahead, c, 0, h->lseT, h->lseA, c + 1 < h->nchunks ? h->update_sms : 0));   // waits for ev_a[c]
      CK(cudaEventRecord(h->ev_f[c], L.ahead));
    }
  }
  h->fwd_ahead = prefetch;
  // Pb now holds exp(Mnew - lseT): lseT becomes the offset of the resident P
  float* t = h->lseA; h->lseA = h->lseT; h->lseT = t;
  h->p_state = PState::updated;
  return TGB200_OK;
}

// Backward of the parity mode (bf16x3): six partial products of S_ext dY_ext^T into fp32 dP + exact row-dot partials,
// then the exact streaming update.  Two contractions per iteration instead of three here too.  (mapping_optimizer.py:395-396)
static int backward_bf16x3(tgb200_mapper* h, cudaStream_t s, const AdamScalars& a) {
  const size_t nkp = (size_t)h->N * h->Ke, vkp = (size_t)h->V * h->Ke, nvp = (size_t)h->N * h->ld;
  if (!h->plan_dp.ready)
    CKS(tc_dpstore_plan(h->tc, h->plan_dp, h->Sxb.p, nkp, h->dYb.p, vkp, 3, h->N, h->V, h->Ke, g_err, sizeof(g_err)));
  TcEpiDpStoreF32 epi{h->dpf.p, h->ld, h->Pb.p, nvp, h->rpart.p, h->N};
  // all six partial products: with only the three or four largest the one-step tests leave their 1e-5 band (measured
  // 28.6 / 25.8 it/s at C3 instead of 21.2 -- not worth the parity-grade mode's point)
  CKS(tc_dpstore_launch(h->tc, h->plan_dp, 6, epi, 0, h->N, h->V, h->Ke, 0, s, g_err, sizeof(g_err)));
  mark(h, s, "tc_gemm_bwd_dp");
  k_rowdot_finalize<<<(unsigned)ceil_div(h->N, 256), 256, 0, s>>>(h->rpart.p, h->r_parts, h->N, h->rdot.p);
  LAUNCH_CHECK("rowdot_finalize");
  if (h->constrained) CKS(filter_update(h, s, a));
  return staged_rows(h, s, 0, h->N, true, [&](int b0, int b1, const StagedPtrs& sp) -> int {
    AdamRowsExactArgs ar{sp.M, sp.m, sp.v, h->dpf.p, h->stats.p, h->rdot.p, h->ld, h->V, b0, b1,
                         h->cfg.lambda_r, h->cfg.lambda_l1, h->cfg.lambda_l2, a};
    if (adam_rows_exact_launch(ar, s)) return fail(TGB200_ERR_CUDA, "launch adam_rows_exact: %s", cudaGetErrorString(cudaGetLastError()));
    mark(h, s, "adam_rows");
    return TGB200_OK;
  });
}

// Backward of the fp32 cross-check mode: FFMA contractions (row-dot GEMM, then the backward GEMM with the fused exact
// epilogue)
static int backward_fp32(tgb200_mapper* h, cudaStream_t s, const AdamScalars& a) {
  GemmArgs g;
  g.A = h->Pf.p; g.lda = h->ld; g.B = h->dY.p; g.ldb = h->Ke;
  g.M = h->N; g.N = h->Ke; g.K = h->V; g.k_per_split = (int)round_up(h->V, 16);
  EpiRowDot epi_r{s_act(h), h->Ke, h->rpart.p};
  dim3 grid_r((unsigned)ceil_div(h->Ke, SG_BN), (unsigned)ceil_div(h->N, SG_BM), 1);
  k_gemm_simt<true, false, EpiRowDot><<<grid_r, SG_THREADS, 0, s>>>(g, epi_r);
  LAUNCH_CHECK("simt_gemm_rowdot");
  k_rowdot_finalize<<<(unsigned)ceil_div(h->N, 256), 256, 0, s>>>(h->rpart.p, h->r_parts, h->N, h->rdot.p);
  LAUNCH_CHECK("rowdot_finalize");
  if (h->constrained) CKS(filter_update(h, s, a));
  g.A = s_act(h); g.lda = h->Ke; g.B = h->dY.p; g.ldb = h->Ke;
  g.M = h->N; g.N = h->V; g.K = h->Ke; g.k_per_split = h->Ke;
  EpiAdam epi{h->M.p, h->m.p, h->v.p, h->ld, h->V, h->stats.p, h->rdot.p, h->cfg.lambda_r, h->cfg.lambda_l1, h->cfg.lambda_l2, a};
  dim3 grid((unsigned)ceil_div(h->V, SG_BN), (unsigned)ceil_div(h->N, SG_BM), 1);
  k_gemm_simt<true, true, EpiAdam><<<grid, SG_THREADS, 0, s>>>(g, epi);
  LAUNCH_CHECK("simt_gemm_bwd_adam");
  return TGB200_OK;
}

// The one exchange of an iteration (SURVEY 8(e)): sum over ranks of [Y_ext partial | row-scalar partials], in place.
static int exchange_partials(tgb200_mapper* h, cudaStream_t s) {
  NcclApi* api = nccl_api(g_err, sizeof(g_err));
  if (!api) return TGB200_ERR_STATE;
  const size_t count = (size_t)h->V * h->Ke + kTail;
  const int r = api->AllReduce(h->Y.p, h->Y.p, count, kNcclFloat32, kNcclSum, h->comm, s);
  if (r != 0) return fail(TGB200_ERR_CUDA, "ncclAllReduce: %s", api->GetErrorString(r));
  return TGB200_OK;
}

// The separate validation forward (and all of tgb200_validation_terms), into out[0..3] (device), on `s`.  bf16 mode re-runs
// the exact row pass, so the per-row entropy exists whatever lambda_r is; P is then fresh and the next iteration starts
// from it.  A sharded handle sums [Y_ext | tail] over the ranks on its communicator first, in the exchange buffer itself:
// the iteration that wrote it has consumed it, and the next forward overwrites it.
static int validation_forward(tgb200_mapper* h, cudaStream_t s, float* out) {
  if (h->bf16) { h->p_state = PState::stale; h->fwd_ahead = false; }
  CKS(forward_pass(h, s, 1));
  LossParams p = val_loss_params(h, out);
  const bool sharded = h->cfg.n_cells_global != h->N;
  k_row_scalar_reduce<<<1, 1024, 0, s>>>(h->stats.p, nullptr, nullptr, h->N, sharded ? 1 : 0, h->Y.p + (size_t)h->V * h->Ke);
  LAUNCH_CHECK("row_scalar_reduce");
  h->tail_stale = sharded;
  if (sharded) {
    CKS(sum_forward_planes(h, s));
    CKS(exchange_partials(h, s));
  }
  CKS(reduce_columns(h, s, p, !sharded, 1));
  k_loss_scalars<true><<<1, 1024, 0, s>>>(p, 1, h->nredchunk, h->val_hist.p);
  LAUNCH_CHECK("loss_scalars");
  return TGB200_OK;
}

static bool val_due(const tgb200_mapper* h) { return h->val_every > 0 && h->val_epoch % h->val_every == 0; }

// second half of an iteration, from the exchange buffer: loss stage, backward and update, and the epoch's validation.
// `more`: another iteration of the same call follows.  The history must have room for one more row.
static int iteration_end(tgb200_mapper* h, const Lanes& L, float lr, bool more) {
  cudaStream_t s = L.work;
  float* hist_row = h->hist.p + (size_t)h->hist_len * TGB200_HIST_COLS;
  // sharded: the caller all-reduced Y (already the sum of every rank's partial planes)
  const bool sharded = h->cfg.n_cells_global != h->N;
  CKS(loss_stage(h, s, hist_row, !sharded));

  const AdamScalars a = adam_scalars(h->cfg, h->step + 1, lr);
  // a validated bf16 epoch runs its own row pass after the update: no next forward issued ahead of it
  if (h->bf16) CKS(backward_bf16(h, L, a, more && !val_due(h)));
  else if (h->x3) CKS(backward_bf16x3(h, s, a));
  else CKS(backward_fp32(h, s, a));
  // the validation of this epoch, on the mapping its update produced (mapping_optimizer.py:398-403)
  if (val_due(h)) {
    // fp32 / bf16x3 with an iteration to follow: the next iteration's forward serves it.  Constrained mode keeps the
    // separate forward, which still sees the filter of this epoch; the next forward sees the updated one.
    if (more && !h->bf16 && !h->constrained) {
      h->val_row = h->hist_len;
    } else {
      if (L.update != s) {                     // the row pass reads every row the update stream wrote
        CK(cudaEventRecord(h->ev_join_lo, L.update));
        CK(cudaStreamWaitEvent(s, h->ev_join_lo, 0));
      }
      CKS(validation_forward(h, s, val_out_of(h, h->hist_len)));
    }
  }
  if (h->val_every > 0) h->val_epoch++;
  h->step++;
  h->hist_len++;
  return TGB200_OK;
}

extern "C" int tgb200_step_begin(tgb200_mapper* h, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CKS(check_ready(h));
  if (h->in_step) return fail(TGB200_ERR_STATE, "step_begin called twice without step_end");
  const Lanes L = lanes_of(h, (cudaStream_t)stream);
  CKS(fork_streams(h, L));
  CKS(iteration_begin(h, L));
  CKS(join_streams(h, L));
  h->in_step = true;
  return TGB200_OK;
}

extern "C" int tgb200_step_end(tgb200_mapper* h, float lr, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  if (!h->in_step) return fail(TGB200_ERR_STATE, "step_end without step_begin");
  CKS(ensure_history(h, h->hist_len + 1, (cudaStream_t)stream));
  const Lanes L = lanes_of(h, (cudaStream_t)stream);
  CKS(fork_streams(h, L));                   // the caller may have all-reduced the exchange buffer on its stream
  CKS(iteration_end(h, L, lr, false));
  CKS(join_streams(h, L));
  h->in_step = false;
  return TGB200_OK;
}

// With a communicator in hand, move the exchange buffer into memory NCCL allocated itself and register it: the in-place
// all-reduce then runs as an in-switch (NVLS) reduction on user buffers.  Best effort: any failure keeps the plain buffer.
static void register_exchange_buffer(tgb200_mapper* h) {
  char e[128];
  NcclApi* a = nccl_api(e, sizeof(e));
  if (!a || !a->MemAlloc || !a->MemFree || !a->CommRegister || !a->CommDeregister || h->y_nccl || !h->comm) return;
  cudaSetDevice(h->cfg.device);
  cudaDeviceSynchronize();
  void* buf = nullptr;
  const size_t bytes = h->Y.n * sizeof(float);
  if (a->MemAlloc(&buf, bytes) != 0 || !buf) { (void)cudaGetLastError(); return; }
  if (cudaMemcpy(buf, h->Y.p, bytes, cudaMemcpyDeviceToDevice) != cudaSuccess) { a->MemFree(buf); (void)cudaGetLastError(); return; }
  void* reg = nullptr;
  if (a->CommRegister(h->comm, buf, bytes, &reg) != 0) { a->MemFree(buf); (void)cudaGetLastError(); return; }
  const size_t n = h->Y.n;
  h->Y.release();
  h->Y.p = static_cast<float*>(buf); h->Y.n = n;
  h->y_nccl = true; h->y_reg = reg;
}

extern "C" int tgb200_comm_unique_id(void* id_out, int64_t cap) {
  if (!id_out || cap < (int64_t)sizeof(NcclUniqueId)) return fail(TGB200_ERR_INVALID, "id buffer must hold %zu bytes", sizeof(NcclUniqueId));
  NcclApi* api = nccl_api(g_err, sizeof(g_err));
  if (!api) return TGB200_ERR_STATE;
  NcclUniqueId id;
  const int r = api->GetUniqueId(&id);
  if (r != 0) return fail(TGB200_ERR_CUDA, "ncclGetUniqueId: %s", api->GetErrorString(r));
  memcpy(id_out, &id, sizeof(id));
  return TGB200_OK;
}

// A communicator that outlives handles: created once per process and group of ranks, lent to handles with tgb200_set_comm
// (ncclCommInitRank costs a second or more at 8 ranks -- too much to pay in every Mapper constructor).
extern "C" int tgb200_comm_create(const void* unique_id, int32_t rank, int32_t world, int32_t device, void** comm_out) {
  if (!unique_id || !comm_out) return fail(TGB200_ERR_INVALID, "null argument");
  if (world < 1 || rank < 0 || rank >= world) return fail(TGB200_ERR_INVALID, "bad rank %d of %d", rank, world);
  NcclApi* api = nccl_api(g_err, sizeof(g_err));
  if (!api) return TGB200_ERR_STATE;
  CK(cudaSetDevice(device));
  NcclUniqueId id;
  memcpy(&id, unique_id, sizeof(id));
  void* comm = nullptr;
  const int r = api->CommInitRank(&comm, world, id, rank);
  if (r != 0) return fail(TGB200_ERR_CUDA, "ncclCommInitRank: %s", api->GetErrorString(r));
  *comm_out = comm;
  return TGB200_OK;
}

extern "C" int tgb200_comm_init_rank(tgb200_mapper* h, const void* unique_id, int32_t rank, int32_t world) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (h->comm) return fail(TGB200_ERR_STATE, "this handle already has a communicator");
  void* comm = nullptr;
  CKS(tgb200_comm_create(unique_id, rank, world, h->cfg.device, &comm));
  h->comm = comm; h->comm_owned = true; h->comm_rank = rank; h->comm_world = world;
  register_exchange_buffer(h);
  return TGB200_OK;
}
extern "C" int tgb200_comm_destroy(void* comm) {
  if (!comm) return TGB200_OK;
  NcclApi* api = nccl_api(g_err, sizeof(g_err));
  if (!api) return TGB200_ERR_STATE;
  const int r = api->CommDestroy(comm);
  if (r != 0) return fail(TGB200_ERR_CUDA, "ncclCommDestroy: %s", api->GetErrorString(r));
  return TGB200_OK;
}

extern "C" int tgb200_set_comm(tgb200_mapper* h, void* nccl_comm, int32_t rank, int32_t world) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (nccl_comm && (world < 1 || rank < 0 || rank >= world)) return fail(TGB200_ERR_INVALID, "bad rank %d of %d", rank, world);
  if (nccl_comm && !nccl_api(g_err, sizeof(g_err))) return TGB200_ERR_STATE;
  if (!nccl_comm && h->val_every > 0 && h->cfg.n_cells_global != h->N)
    return fail(TGB200_ERR_STATE, "set_comm(NULL) while a sharded handle validates: call tgb200_set_validation(0) first");
  if (h->y_nccl) {              // back to a plain buffer before the communicator it is registered with goes away
    DevBuf<float> plain;
    CKS(plain.alloc(h->Y.n, false));
    CK(cudaDeviceSynchronize());
    CK(cudaMemcpy(plain.p, h->Y.p, h->Y.n * sizeof(float), cudaMemcpyDeviceToDevice));
    h->release_exchange_registration();
    h->Y.p = plain.p; h->Y.n = plain.n; plain.p = nullptr; plain.n = 0;
  }
  if (h->comm && h->comm_owned) { if (NcclApi* a = nccl_api(g_err, sizeof(g_err))) a->CommDestroy(h->comm); }
  h->comm = nccl_comm; h->comm_owned = false; h->comm_rank = rank; h->comm_world = nccl_comm ? world : 1;
  register_exchange_buffer(h);
  return TGB200_OK;
}

extern "C" int tgb200_run(tgb200_mapper* h, int32_t n_steps, float lr, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (n_steps < 0) return fail(TGB200_ERR_INVALID, "n_steps < 0");
  const bool sharded = h->cfg.n_cells_global != h->N;
  if (sharded && !h->comm)
    return fail(TGB200_ERR_STATE, "cell-sharded handle without a communicator: call tgb200_comm_init_rank / tgb200_set_comm, or drive "
                                  "step_begin / all-reduce / step_end yourself");
  CK(cudaSetDevice(h->cfg.device));
  CKS(ensure_history(h, h->hist_len + n_steps, (cudaStream_t)stream));
  if (n_steps == 0) return TGB200_OK;
  CKS(check_ready(h));
  if (h->in_step) return fail(TGB200_ERR_STATE, "run inside a step");
  const Lanes L = lanes_of(h, (cudaStream_t)stream);
  CKS(fork_streams(h, L));                   // iterations chain through the handle's own streams and events
  int st = TGB200_OK;
  for (int i = 0; i < n_steps && st == TGB200_OK; ++i) {
    st = iteration_begin(h, L);
    if (st == TGB200_OK && sharded) st = exchange_partials(h, L.work);
    if (st == TGB200_OK) st = iteration_end(h, L, lr, i + 1 < n_steps);
  }
  h->val_row = -1;                           // set only when an iteration follows, unless that iteration failed
  CKS(join_streams(h, L));
  return st;
}

// ---------------------------------------------------------------------------------------
extern "C" int tgb200_history_len(tgb200_mapper* h, int64_t* n) {
  if (!h || !n) return fail(TGB200_ERR_INVALID, "null argument");
  *n = h->hist_len;
  return TGB200_OK;
}

extern "C" int tgb200_get_history(tgb200_mapper* h, int64_t first, int64_t count, float* out, void* stream) {
  if (!h || (!out && count > 0)) return fail(TGB200_ERR_INVALID, "null argument");
  if (first < 0 || count < 0 || first + count > h->hist_len) return fail(TGB200_ERR_INVALID, "history range [%lld,%lld) outside [0,%lld)", (long long)first, (long long)(first + count), (long long)h->hist_len);
  if (count == 0) return TGB200_OK;
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaMemcpyAsync(out, h->hist.p + (size_t)first * TGB200_HIST_COLS, (size_t)count * TGB200_HIST_COLS * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_get_mapping(tgb200_mapper* h, float* out, void* stream) {
  if (!h || !out) return fail(TGB200_ERR_INVALID, "null argument");
  if (!h->have_mapping) return fail(TGB200_ERR_STATE, "no mapping set");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  // softmax(M) in fp32 (:406-407), through device memory the iterations leave idle between calls -- no allocation here:
  //   fp32 mode          Pf (the forward operand itself)
  //   bf16x3 mode        the three bf16 P planes (6 B/element, rewritten by every forward pass)
  //   bf16 mode          dq (2 B/element: half of the rows at a time)
  const size_t nv = (size_t)h->N * h->ld;
  DevBuf<float> tmp;
  float* scratch = h->Pf.p;
  size_t cap_elems = nv;
  if (h->x3) { scratch = reinterpret_cast<float*>(h->Pb.p); cap_elems = 3 * nv / 2; }
  else if (h->bf16) { scratch = reinterpret_cast<float*>(h->dq.p); cap_elems = nv / 2; }
  int blk = (int)(cap_elems / (size_t)h->ld);
  if (blk > h->N) blk = h->N;
  if (blk < 1) { CKS(tmp.alloc((size_t)h->ld, false)); scratch = tmp.p; blk = 1; }     // one-row mapping in bf16 mode
  for (int r0 = 0; r0 < h->N; r0 += blk) {
    const int nr = h->N - r0 < blk ? h->N - r0 : blk;
    CKS(launch_softmax_rows<float>(h, s, scratch, 0, nullptr, Split3{nullptr, 0}, r0, nr));
    CK(cudaMemcpy2DAsync(out + (size_t)r0 * h->V, (size_t)h->V * sizeof(float), scratch, (size_t)h->ld * sizeof(float),
                         (size_t)h->V * sizeof(float), nr, cudaMemcpyDefault, s));
  }
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// fp32 staging of the bf16 first moment between the caller and `mb`: the idle dq buffer, half of the rows at a time
// (`one_row` for a one-row mapping)
static int moment_scratch(tgb200_mapper* h, DevBuf<float>& one_row, float** scratch, int* blk) {
  *scratch = reinterpret_cast<float*>(h->dq.p);
  *blk = h->N / 2;
  if (*blk < 1) { CKS(one_row.alloc((size_t)h->ld, false)); *scratch = one_row.p; *blk = 1; }
  return TGB200_OK;
}

extern "C" int tgb200_get_state(tgb200_mapper* h, float* M, float* m, float* v, int64_t* step, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  const size_t w = (size_t)h->V * sizeof(float), pitch = (size_t)h->ld * sizeof(float);
  // each part of the state (device rows, host rows) on its own
  auto get = [&](float* dst, const DevBuf<float>& d, const DevBuf<float>& hp) {
    return state_parts(h, [&](int a, int b) -> int {
      CK(cudaMemcpy2DAsync(dst + (size_t)a * h->V, w, state_row(h, d, hp, a), pitch, w, b - a, cudaMemcpyDefault, s));
      return TGB200_OK;
    });
  };
  if (M) CKS(get(M, h->M, h->Mh));
  if (m && !h->bf16) CKS(get(m, h->m, h->mh));
  if (m && h->bf16) {         // bf16 first moment -> fp32 for the caller
    float* scratch;
    int blk;
    DevBuf<float> one_row;
    CKS(moment_scratch(h, one_row, &scratch, &blk));
    CKS(state_parts(h, [&](int a, int b) -> int {
      for (int r0 = a; r0 < b; r0 += blk) {
        const int nr = b - r0 < blk ? b - r0 : blk;
        const long long n = (long long)nr * h->ld;
        k_bf16_to_f32<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(state_row(h, h->mb, h->mbh, r0), scratch, n);
        LAUNCH_CHECK("bf16_to_f32");
        CK(cudaMemcpy2DAsync(m + (size_t)r0 * h->V, w, scratch, pitch, w, nr, cudaMemcpyDefault, s));
      }
      return TGB200_OK;
    }));
  }
  if (v) CKS(get(v, h->v, h->vh));
  if (step) *step = h->step;
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_set_state(tgb200_mapper* h, const float* M, const float* m, const float* v, int64_t step, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (step < 0) return fail(TGB200_ERR_INVALID, "step < 0");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  const size_t w = (size_t)h->V * sizeof(float), pitch = (size_t)h->ld * sizeof(float);
  auto set = [&](const float* src, DevBuf<float>& d, DevBuf<float>& hp) {
    return state_parts(h, [&](int a, int b) -> int {
      CK(cudaMemcpy2DAsync(state_row(h, d, hp, a), pitch, src + (size_t)a * h->V, w, w, b - a, cudaMemcpyDefault, s));
      return TGB200_OK;
    });
  };
  if (M) {
    CKS(set(M, h->M, h->Mh)); h->have_mapping = true; h->p_state = PState::stale;
    h->fwd_ahead = false;
    if (h->bf16) CK(cudaMemsetAsync(h->rcenter.p, 0, h->rcenter.n * sizeof(float), s));
  }
  if (m && !h->bf16) CKS(set(m, h->m, h->mh));
  if (m && h->bf16) {         // fp32 from the caller -> bf16 (exact for values that came out of tgb200_get_state)
    float* scratch;
    int blk;
    DevBuf<float> one_row;
    CKS(moment_scratch(h, one_row, &scratch, &blk));
    CKS(state_parts(h, [&](int a, int b) -> int {
      for (int r0 = a; r0 < b; r0 += blk) {
        const int nr = b - r0 < blk ? b - r0 : blk;
        const long long n = (long long)nr * h->ld;
        CK(cudaMemsetAsync(scratch, 0, (size_t)n * sizeof(float), s));            // pad columns stay zero
        CK(cudaMemcpy2DAsync(scratch, pitch, m + (size_t)r0 * h->V, w, w, nr, cudaMemcpyDefault, s));
        k_f32_to_bf16<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(scratch, state_row(h, h->mb, h->mbh, r0), n);
        LAUNCH_CHECK("f32_to_bf16");
      }
      return TGB200_OK;
    }));
  }
  if (v) CKS(set(v, h->v, h->vh));
  h->step = step;
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// _val_loss_fn (:311-356) on demand: the validation forward tgb200_set_validation runs in the loop, then one 16-byte copy
extern "C" int tgb200_validation_terms(tgb200_mapper* h, float* out4, void* stream) {
  if (!h || !out4) return fail(TGB200_ERR_INVALID, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(check_ready(h));
  if (h->in_step) return fail(TGB200_ERR_STATE, "validation_terms inside a step");
  CKS(check_validation_supported(h));
  CKS(alloc_validation(h));
  DevBuf<float> d4;
  CKS(d4.alloc(4, false));
  CKS(validation_forward(h, s, d4.p));
  CK(cudaMemcpyAsync(out4, d4.p, 4 * sizeof(float), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// ---------------------------------------------------------------------------------------
extern "C" int tgb200_kernel_launches(tgb200_mapper* h, int64_t* n) {
  if (!h || !n) return fail(TGB200_ERR_INVALID, "null argument");
  *n = h->launches;
  return TGB200_OK;
}

extern "C" int tgb200_profile_step(tgb200_mapper* h, float lr, void* stream, const char** names, float* ms,
                                   int32_t cap, int32_t* n) {
  if (!h || !names || !ms || !n) return fail(TGB200_ERR_INVALID, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(check_ready(h));
  if (h->in_step) return fail(TGB200_ERR_STATE, "profile_step inside a step");
  CKS(ensure_history(h, h->hist_len + 1, s));
  cudaEvent_t e0;
  CK(cudaEventCreate(&e0));
  CK(cudaStreamSynchronize(s));
  CK(cudaEventRecord(e0, s));
  // the step's launches are appended to the records; a timeline recording in progress keeps them
  const bool timeline = h->recording;
  const size_t first = h->records.size();
  h->recording = true;
  const Lanes L{s, s, s, s};                 // one stream, one kernel at a time: clean per-kernel durations
  int st = iteration_begin(h, L);
  if (st == TGB200_OK) st = iteration_end(h, L, lr, false);
  h->recording = timeline;
  cudaStreamSynchronize(s);
  int cnt = 0;
  cudaEvent_t prev = e0;
  for (size_t i = first; i < h->records.size(); ++i) {
    float f = 0.f;
    cudaEventElapsedTime(&f, prev, h->records[i].ev);
    if (cnt < cap) { names[cnt] = h->records[i].name; ms[cnt] = f; cnt++; }
    prev = h->records[i].ev;
  }
  cudaEventDestroy(e0);
  if (!timeline) h->drop_records(first);
  *n = cnt;
  return st;
}

extern "C" int tgb200_debug_timeline(tgb200_mapper* h, int32_t enable, const char** names, int32_t* streams, float* end_ms,
                                     int32_t cap, int32_t* n) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  if (!enable) {
    int cnt = 0;
    for (const LaunchRecord& r : h->records) {
      float f = 0.f;
      cudaEventElapsedTime(&f, h->records[0].ev, r.ev);
      if (names && streams && end_ms && cnt < cap) { names[cnt] = r.name; streams[cnt] = r.stream; end_ms[cnt] = f; cnt++; }
    }
    if (n) *n = cnt;
  }
  h->drop_records(0);
  h->recording = enable != 0;
  return TGB200_OK;
}

// n elements of `planes` bf16 planes, summed from the last plane to the first in fp32 on the host
static int widen_bf16(const __nv_bfloat16* src, int64_t n, int planes, float* out) {
  std::vector<__nv_bfloat16> tmp((size_t)n * planes);
  CK(cudaMemcpy(tmp.data(), src, tmp.size() * sizeof(__nv_bfloat16), cudaMemcpyDefault));
  for (int64_t i = 0; i < n; ++i) {
    float acc = __bfloat162float(tmp[(size_t)(planes - 1) * n + i]);
    for (int pl = planes - 2; pl >= 0; --pl) acc += __bfloat162float(tmp[(size_t)pl * n + i]);
    out[i] = acc;
  }
  return TGB200_OK;
}

extern "C" int tgb200_debug_buffer(tgb200_mapper* h, const char* name, float* out_host, int64_t cap, int64_t* n) {
  if (!h || !name || !n) return fail(TGB200_ERR_INVALID, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  const std::string nm(name);
  const float* src = nullptr;
  int64_t cnt = 0;
  const int64_t vk = (int64_t)h->V * h->Ke, nv = (int64_t)h->N * h->ld;
  // bf16 buffers (`planes` bf16 planes of n elements, summed) widened to float
  auto widened = [&](const __nv_bfloat16* p, int64_t count, int planes) -> int {
    *n = count;
    if (!out_host) return TGB200_OK;
    if (cap < count) return fail(TGB200_ERR_INVALID, "buffer '%s' needs %lld floats", name, (long long)count);
    return widen_bf16(p, count, planes, out_host);
  };
  // the state: its device rows, then its host rows
  auto state = [&](const auto& d, const auto& hp) -> int {
    *n = nv;
    if (!out_host) return TGB200_OK;
    if (cap < nv) return fail(TGB200_ERR_INVALID, "buffer '%s' needs %lld floats", name, (long long)nv);
    const size_t nr = (size_t)h->R * h->ld;
    if constexpr (sizeof(*d.p) == 2) {
      if (nr) CKS(widen_bf16(d.p, (int64_t)nr, 1, out_host));
      if (hp.n) CKS(widen_bf16(hp.p, (int64_t)hp.n, 1, out_host + nr));
    } else {
      if (nr) CK(cudaMemcpy(out_host, d.p, nr * sizeof(float), cudaMemcpyDefault));
      if (hp.n) CK(cudaMemcpy(out_host + nr, hp.p, hp.n * sizeof(float), cudaMemcpyDefault));
    }
    return TGB200_OK;
  };
  if (nm == "Y") { src = h->Y.p; cnt = vk; }
  else if (nm == "M") return state(h->M, h->Mh);
  else if (nm == "v") return state(h->v, h->vh);
  else if (nm == "m") return h->bf16 ? state(h->mb, h->mbh) : state(h->m, h->mh);
  else if (nm == "Pb" && h->x3) return widened(h->Pb.p, nv, 3);
  else if (nm == "Pf" && !h->tcm) { src = h->Pf.p; cnt = nv; }
  else if (nm == "dpf" && h->x3) { src = h->dpf.p; cnt = nv; }
  else if (nm == "stats") { src = reinterpret_cast<const float*>(h->stats.p); cnt = (int64_t)h->N * 4; }
  else if (nm == "rowc" && h->bf16) { src = reinterpret_cast<const float*>(h->rowc.p); cnt = (int64_t)h->N * 4; }
  else if (nm == "zsum" && h->bf16) { src = h->zsum.p; cnt = h->N; }
  else if (nm == "inv_zt" && h->bf16) { src = h->inv_zt.p; cnt = h->N; }
  else if (nm == "lseA" && h->bf16) { src = h->lseA; cnt = h->N; }
  else if (nm == "lseT" && h->bf16) { src = h->lseT; cnt = h->N; }
  else if (nm == "pxsum" && h->pxsum.p) { src = h->pxsum.p; cnt = h->N; }
  else if (nm == "l1sum" && h->l1sum.p) { src = h->l1sum.p; cnt = h->N; }
  else if (nm == "l2sum" && h->l2sum.p) { src = h->l2sum.p; cnt = h->N; }
  else if (nm == "dY") {
    src = h->dY.p; cnt = vk;
    if (h->tcm && out_host) {     // only the bf16 copy (or its three planes) exists on the tensor-core paths
      if (cap < cnt) return fail(TGB200_ERR_INVALID, "buffer 'dY' needs %lld floats", (long long)cnt);
      CKS(widen_bf16(h->dYb.p, vk, h->x3 ? 3 : 1, out_host));
      *n = cnt;
      return TGB200_OK;
    }
  }
  else if ((nm == "dq" || nm == "Pb") && h->bf16) return widened(nm == "dq" ? h->dq.p : h->Pb.p, nv, 1);
  else if (nm == "rcenter" && h->bf16) { src = h->rcenter.p; cnt = h->N; }
  else if (nm == "rdot") { src = h->rdot.p; cnt = h->N; }
  // the loss's constant norms of G (per gene, per voxel) and of the graph products W G, (A + I) G (per gene)
  else if (nm == "ngc") { src = h->ngc.p; cnt = h->K; }
  else if (nm == "ngr") { src = h->ngr.p; cnt = h->V; }
  else if (nm == "nwg" && h->nwg.p) { src = h->nwg.p; cnt = h->K; }
  else if (nm == "nag" && h->nag.p) { src = h->nag.p; cnt = h->K; }
  else if (nm == "Sx") { src = h->Sx.p; cnt = (int64_t)h->N * h->Ke; }
  else if (nm == "tail") { src = h->Y.p + vk; cnt = kTail; }       // the row-scalar sums after Y_ext (k_row_scalar_reduce)
  else if (h->constrained && (nm == "F" || nm == "f" || nm == "mF" || nm == "vF")) {
    src = nm == "F" ? h->Fl.p : nm == "f" ? h->fsig.p : nm == "mF" ? h->mF.p : h->vF.p;
    cnt = h->N;
  }
  else if (nm == "Sf" && h->constrained) { src = h->Sf.p; cnt = (int64_t)h->N * h->Ke; }
  else if (nm == "fscal" && h->constrained) { src = h->fscal.p; cnt = 2; }
  else if (nm == "shape") {   // Ke, ld, fwd_splits, r_parts, cell chunks of the bf16 pipeline
    *n = 5;
    if (!out_host) return TGB200_OK;
    if (cap < 5) return fail(TGB200_ERR_INVALID, "cap < 5");
    out_host[0] = (float)h->Ke; out_host[1] = (float)h->ld; out_host[2] = (float)h->fwd_splits; out_host[3] = (float)h->r_parts;
    out_host[4] = (float)h->nchunks;
    return TGB200_OK;
  } else if (nm == "ring") {    // rows per staging block of host state (0: resident state)
    *n = 1;
    if (!out_host) return TGB200_OK;
    if (cap < 1) return fail(TGB200_ERR_INVALID, "cap < 1");
    out_host[0] = (float)h->ring_rows;
    return TGB200_OK;
  } else if (nm == "legacy_init") {
    *n = 8;
    if (!out_host) return TGB200_OK;
    if (cap < 8) return fail(TGB200_ERR_INVALID, "cap < 8");
    for (int i = 0; i < 8; ++i) out_host[i] = h->legacy_stats[i];
    return TGB200_OK;
  } else return fail(TGB200_ERR_INVALID, "unknown debug buffer '%s'", name);
  *n = cnt;
  if (out_host) {
    if (cap < cnt) return fail(TGB200_ERR_INVALID, "buffer '%s' needs %lld floats", name, (long long)cnt);
    CK(cudaMemcpy(out_host, src, cnt * sizeof(float), cudaMemcpyDefault));
  }
  return TGB200_OK;
}


extern "C" int tgb200_algorithmic_cost(tgb200_mapper* h, double* hbm_bytes, double* flops) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  const double N = h->N, V = h->V, K = h->K, T = h->T;
  const double sS = h->bf16 ? 2.0 : 4.0;
  // SURVEY.md 8(d): 28 N V = M read in forward (4) + M, m, v read and written (24); with the first moment kept in bf16
  // (bf16 mode) m costs 2 + 2 instead of 4 + 4 -> 24 N V ("if the moments are kept in BF16 ... state which")
  if (hbm_bytes) *hbm_bytes = (h->bf16 ? 24.0 : 28.0) * N * V + 2.0 * sS * N * K + 8.0 * V * K;
  if (flops) *flops = 4.0 * N * V * K + (h->cfg.lambda_ct_islands > 0.f ? 4.0 * N * V * T : 0.0);
  return TGB200_OK;
}

// ---------------------------------------------------------------------------------------
// Stateless entry points (no handle): the device checks they share.

// Makes `device` current if it is a visible sm_90 device; *n_sms receives its SM count.
static int use_sm90_device(int32_t device, int* n_sms) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(TGB200_ERR_NO_DEVICE, "no CUDA device visible: tangram_b200 has no CPU fallback");
  }
  if (device < 0 || device >= ndev) return fail(TGB200_ERR_INVALID, "device %d out of range (%d devices)", device, ndev);
  int major = 0, minor = 0;                      // attribute queries: cudaGetDeviceProperties costs milliseconds
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  CK(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  CK(cudaDeviceGetAttribute(n_sms, cudaDevAttrMultiProcessorCount, device));
  if (major != 9 || minor != 0)
    return fail(TGB200_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", device, major, minor);
  CK(cudaSetDevice(device));
  return TGB200_OK;
}

static int require_device_memory(const void* p, int32_t device, const char* what) {
  cudaPointerAttributes at;
  CK(cudaPointerGetAttributes(&at, p));
  if ((at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) || at.device != device)
    return fail(TGB200_ERR_INVALID, "%s is not device memory of device %d", what, device);
  return TGB200_OK;
}

// Agreement of R runs (tangram/mapping_parameter_tuning.py:42-82).
template <int R>
static void launch_agreement(const AgrArgs& a, int grid, bool rows, cudaStream_t s) {
  if (rows) k_agreement<R, true><<<grid, kAgrThreads, 0, s>>>(a);
  else k_agreement<R, false><<<grid, kAgrThreads, 0, s>>>(a);
}

static void launch_agreement(const AgrArgs& a, int R, int grid, bool rows, cudaStream_t s) {
  switch (R) {
    case 1: launch_agreement<1>(a, grid, rows, s); break;
    case 2: launch_agreement<2>(a, grid, rows, s); break;
    case 3: launch_agreement<3>(a, grid, rows, s); break;
    case 4: launch_agreement<4>(a, grid, rows, s); break;
    case 5: launch_agreement<5>(a, grid, rows, s); break;
    case 6: launch_agreement<6>(a, grid, rows, s); break;
    case 7: launch_agreement<7>(a, grid, rows, s); break;
    default: launch_agreement<8>(a, grid, rows, s); break;
  }
}

// The checks every agreement entry point makes on its arrays, in this order: R, the shape, the device, each array.
// Fills the arrays, shape and load width of *a and, if grid is given, the grid of k_agreement<R, rows>: enough blocks
// for every row, at most what fits on the device at once.
static int agreement_setup(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld, int32_t device,
                           bool per_row, AgrArgs* a, int* grid) {
  if (R < 1 || R > kAgrMaxRuns) return fail(TGB200_ERR_INVALID, "R=%d runs, supported 1..%d", R, kAgrMaxRuns);
  if (rows <= 0 || cols <= 0 || ld < cols || cols > INT32_MAX)
    return fail(TGB200_ERR_INVALID, "bad shape rows=%lld cols=%lld ld=%lld", (long long)rows, (long long)cols, (long long)ld);
  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  *a = AgrArgs{};
  a->rows = rows; a->cols = cols; a->ld = ld;
  a->vec = ld % 4 == 0;
  for (int r = 0; r < R; ++r) {
    if (!arrays[r]) return fail(TGB200_ERR_INVALID, "array %d is null", r);
    char what[32];
    snprintf(what, sizeof(what), "array %d", r);
    CKS(require_device_memory(arrays[r], device, what));
    a->x[r] = arrays[r];
    if (reinterpret_cast<uintptr_t>(arrays[r]) % 16) a->vec = 0;
  }
  if (!grid) return TGB200_OK;
  int per_sm = 0;
#define AGR_OCC(RR) \
  case RR: CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, per_row ? k_agreement<RR, true> : k_agreement<RR, false>, kAgrThreads, 0)); break;
  switch (R) { AGR_OCC(1) AGR_OCC(2) AGR_OCC(3) AGR_OCC(4) AGR_OCC(5) AGR_OCC(6) AGR_OCC(7) AGR_OCC(8) }
#undef AGR_OCC
  const int warps = kAgrThreads / kWarp;
  const int64_t need = ceil_div(rows, warps);
  *grid = (int)std::max<int64_t>(1, std::min<int64_t>(need, (int64_t)std::max(per_sm, 1) * n_sms));
  return TGB200_OK;
}

extern "C" int tgb200_agreement(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                double* pearson_out, float* vote_out, float* cons_out, int32_t device, void* stream) {
  if (!arrays) return fail(TGB200_ERR_INVALID, "null argument");
  const bool per_row = vote_out || cons_out;
  AgrArgs a;
  int grid = 0;
  CKS(agreement_setup(arrays, R, rows, cols, ld, device, per_row, &a, &grid));
  cudaStream_t s = (cudaStream_t)stream;
  const int NS = R + R * (R + 1) / 2;
  // scratch is O(R^2 grid + rows): the per-block partials, the shifts, the correlations, the per-row results
  DevBuf<double> shift, part, corr;
  DevBuf<float> vote, cons;
  CKS(shift.alloc(R, false)); CKS(part.alloc((size_t)grid * NS, false)); CKS(corr.alloc(R > 1 ? R * (R - 1) / 2 : 1, false));
  if (vote_out) CKS(vote.alloc(rows, false));
  if (cons_out) CKS(cons.alloc(rows, false));
  a.shift = shift.p; a.part = part.p; a.vote = vote.p; a.cons = cons.p;
  k_agreement_shift<<<R, kAgrThreads, 0, s>>>(a, shift.p, 0);
  CK(cudaGetLastError());
  launch_agreement(a, R, grid, per_row, s);
  CK(cudaGetLastError());
  if (R > 1) {
    k_agreement_finish<<<1, 64, 0, s>>>(part.p, grid, R, (double)rows * (double)cols, corr.p);
    CK(cudaGetLastError());
    if (pearson_out) CK(cudaMemcpyAsync(pearson_out, corr.p, sizeof(double) * R * (R - 1) / 2, cudaMemcpyDefault, s));
  }
  if (vote_out) CK(cudaMemcpyAsync(vote_out, vote.p, sizeof(float) * rows, cudaMemcpyDefault, s));
  if (cons_out) CK(cudaMemcpyAsync(cons_out, cons.p, sizeof(float) * rows, cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// tgb200_agreement in three steps around the caller's sums over row shards.
extern "C" int tgb200_agreement_sample(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                       double* sample_out, int32_t device, void* stream) {
  if (!arrays || !sample_out) return fail(TGB200_ERR_INVALID, "null argument");
  AgrArgs a;
  CKS(agreement_setup(arrays, R, rows, cols, ld, device, false, &a, nullptr));
  cudaStream_t s = (cudaStream_t)stream;
  DevBuf<double> out;
  CKS(out.alloc(R + 1, false));
  k_agreement_shift<<<R, kAgrThreads, 0, s>>>(a, out.p, 1);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(sample_out, out.p, sizeof(double) * (R + 1), cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_agreement_partials(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                         const double* shift, double* sums_out, float* vote_out, float* cons_out,
                                         int32_t device, void* stream) {
  if (!arrays || !shift || !sums_out) return fail(TGB200_ERR_INVALID, "null argument");
  const bool per_row = vote_out || cons_out;
  AgrArgs a;
  int grid = 0;
  CKS(agreement_setup(arrays, R, rows, cols, ld, device, per_row, &a, &grid));
  cudaStream_t s = (cudaStream_t)stream;
  const int NS = R + R * (R + 1) / 2;
  DevBuf<double> sh, part, tot;
  DevBuf<float> vote, cons;
  CKS(sh.alloc(R, false)); CKS(part.alloc((size_t)grid * NS, false)); CKS(tot.alloc(NS, false));
  if (vote_out) CKS(vote.alloc(rows, false));
  if (cons_out) CKS(cons.alloc(rows, false));
  CK(cudaMemcpyAsync(sh.p, shift, sizeof(double) * R, cudaMemcpyDefault, s));
  a.shift = sh.p; a.part = part.p; a.vote = vote.p; a.cons = cons.p;
  launch_agreement(a, R, grid, per_row, s);
  CK(cudaGetLastError());
  k_agreement_total<<<1, 64, 0, s>>>(part.p, grid, R, tot.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(sums_out, tot.p, sizeof(double) * NS, cudaMemcpyDefault, s));
  if (vote_out) CK(cudaMemcpyAsync(vote_out, vote.p, sizeof(float) * rows, cudaMemcpyDefault, s));
  if (cons_out) CK(cudaMemcpyAsync(cons_out, cons.p, sizeof(float) * rows, cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_agreement_pearson(const double* sums, int32_t R, int64_t rows_global, int64_t cols,
                                        double* pearson_out, int32_t device, void* stream) {
  if (!sums || !pearson_out) return fail(TGB200_ERR_INVALID, "null argument");
  if (R < 1 || R > kAgrMaxRuns) return fail(TGB200_ERR_INVALID, "R=%d runs, supported 1..%d", R, kAgrMaxRuns);
  if (rows_global <= 0 || cols <= 0)
    return fail(TGB200_ERR_INVALID, "bad shape rows=%lld cols=%lld", (long long)rows_global, (long long)cols);
  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  if (R == 1) return TGB200_OK;                        // no pair
  cudaStream_t s = (cudaStream_t)stream;
  const int NS = R + R * (R + 1) / 2, NP = R * (R - 1) / 2;
  DevBuf<double> tot, corr;
  CKS(tot.alloc(NS, false)); CKS(corr.alloc(NP, false));
  CK(cudaMemcpyAsync(tot.p, sums, sizeof(double) * NS, cudaMemcpyDefault, s));
  k_agreement_pearson<<<1, 32, 0, s>>>(tot.p, R, (double)rows_global * (double)cols, corr.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(pearson_out, corr.p, sizeof(double) * NP, cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// Label sums and row argmax of a mapping (tangram/utils.py:126-153, 205-285, 820-842).
extern "C" int tgb200_annotate(const float* map, int64_t rows, int64_t cols, int64_t ld, const int32_t* labels,
                               int32_t n_labels, double* sums_out, int32_t* argmax_out, int32_t device, void* stream) {
  if (!map || !labels) return fail(TGB200_ERR_INVALID, "null argument");
  if (rows <= 0 || cols <= 0 || ld < cols || rows > INT32_MAX || cols > INT32_MAX)
    return fail(TGB200_ERR_INVALID, "bad shape rows=%lld cols=%lld ld=%lld", (long long)rows, (long long)cols, (long long)ld);
  if (n_labels < 1) return fail(TGB200_ERR_INVALID, "n_labels=%d, must be at least 1", n_labels);
  // stable counting sort of the labelled rows by label; each label's segment cut into items of kAnnChunk rows
  std::vector<int> seg(n_labels + 1, 0);
  for (int64_t i = 0; i < rows; ++i) {
    const int32_t l = labels[i];
    if (l < -1 || l >= n_labels)
      return fail(TGB200_ERR_INVALID, "label %d of row %lld is outside [-1, %d)", l, (long long)i, n_labels);
    if (l >= 0) ++seg[l + 1];
  }
  for (int t = 0; t < n_labels; ++t) seg[t + 1] += seg[t];
  const int n_labelled = seg[n_labels];
  std::vector<int> perm(std::max(n_labelled, 1)), next(seg.begin(), seg.end() - 1);
  for (int64_t i = 0; i < rows; ++i)
    if (labels[i] >= 0) perm[next[labels[i]]++] = (int)i;
  std::vector<int> item_start, label_items(n_labels + 1);
  for (int t = 0; t < n_labels; ++t) {
    label_items[t] = (int)item_start.size();
    for (int p = seg[t]; p < seg[t + 1]; p += kAnnChunk) item_start.push_back(p);
  }
  const int n_items = (int)item_start.size();
  label_items[n_labels] = n_items;
  item_start.push_back(n_labelled);

  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  CKS(require_device_memory(map, device, "the mapping"));
  if (!sums_out && !argmax_out) return TGB200_OK;
  cudaStream_t s = (cudaStream_t)stream;
  AnnArgs a{};
  a.map = map; a.cols = cols; a.ld = ld;
  a.vec = ld % 4 == 0 && reinterpret_cast<uintptr_t>(map) % 16 == 0;
  a.n_items = n_items;
  a.n_slabs = (int)ceil_div(cols, kAnnSlab);
  // scratch: the permutation and item tables, n_items x cols fp64 partials, n_labelled x slabs argmax partials
  DevBuf<int> d_perm, d_items, d_label_items, d_argmax, amax_idx;
  DevBuf<double> part, sums;
  DevBuf<float> amax_val;
  CKS(d_perm.alloc(perm.size(), false)); CKS(d_items.alloc(item_start.size(), false));
  CK(cudaMemcpyAsync(d_perm.p, perm.data(), sizeof(int) * perm.size(), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_items.p, item_start.data(), sizeof(int) * item_start.size(), cudaMemcpyHostToDevice, s));
  a.perm = d_perm.p; a.item_start = d_items.p;
  if (sums_out) {
    CKS(d_label_items.alloc(label_items.size(), false));
    CK(cudaMemcpyAsync(d_label_items.p, label_items.data(), sizeof(int) * label_items.size(), cudaMemcpyHostToDevice, s));
    CKS(part.alloc(std::max<size_t>((size_t)n_items * cols, 1), false));
    CKS(sums.alloc((size_t)n_labels * cols, false));
    a.part = part.p;
  }
  if (argmax_out) {
    CKS(amax_val.alloc(std::max<size_t>((size_t)n_labelled * a.n_slabs, 1), false));
    CKS(amax_idx.alloc(std::max<size_t>((size_t)n_labelled * a.n_slabs, 1), false));
    CKS(d_argmax.alloc(rows, false));
    CK(cudaMemsetAsync(d_argmax.p, 0xff, sizeof(int) * rows, s));            // -1 for the unlabelled rows
    a.amax_val = amax_val.p; a.amax_idx = amax_idx.p;
  }
  if (n_items > 0) {
    const dim3 grid(a.n_slabs, std::min(n_items, 65535));
    if (sums_out && argmax_out) k_annotate<true, true><<<grid, kAnnThreads, 0, s>>>(a);
    else if (sums_out) k_annotate<true, false><<<grid, kAnnThreads, 0, s>>>(a);
    else k_annotate<false, true><<<grid, kAnnThreads, 0, s>>>(a);
    CK(cudaGetLastError());
  }
  if (sums_out) {
    const dim3 grid((unsigned)ceil_div(cols, kAnnThreads), std::min(n_labels, 65535));
    k_annotate_sums<<<grid, kAnnThreads, 0, s>>>(part.p, d_label_items.p, n_labels, cols, sums.p);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(sums_out, sums.p, sizeof(double) * n_labels * cols, cudaMemcpyDefault, s));
  }
  if (argmax_out) {
    if (n_labelled > 0) {
      const int grid = (int)std::min<int64_t>(ceil_div(n_labelled, kAnnThreads), (int64_t)8 * n_sms);
      k_annotate_argmax<<<grid, kAnnThreads, 0, s>>>(amax_val.p, amax_idx.p, d_perm.p, n_labelled, a.n_slabs, d_argmax.p);
      CK(cudaGetLastError());
    }
    CK(cudaMemcpyAsync(argmax_out, d_argmax.p, sizeof(int32_t) * rows, cudaMemcpyDefault, s));
  }
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// Projection of X through any mapping (tangram/utils.py:366-368), streamed over cell blocks.
namespace {
constexpr int64_t kProjUnit = 2048;      // blocks are multiples of 2048 cells
// cells per accumulation chain: a truncating tensor-core chain of c same-sign terms drifts by up to c / 8 u (DESIGN 2);
// 512 keeps all-positive data (probabilities times expression) well inside 3e-6 rel-Frobenius.  It divides kProjUnit,
// so the chains, and the order they are added in, do not depend on the block size.
constexpr int64_t kProjChain = 512;
constexpr int64_t kProjBlocks = 8;       // default: about this many blocks, so the copies of one hide under the others
struct CopyStream {                      // the second stream and its events, released on every return path
  cudaStream_t s = nullptr;
  cudaEvent_t start = nullptr, copied[2] = {}, freed[2] = {};
  ~CopyStream() {
    for (cudaEvent_t e : {start, copied[0], copied[1], freed[0], freed[1]}) if (e) cudaEventDestroy(e);
    if (s) cudaStreamDestroy(s);
  }
};
}  // namespace

// The projection of tgb200_project_map and tgb200_project.  The mapping rows come from `map` (fp32, row stride `ld`,
// copied on the copy stream, then k_split3) or, with a handle `h` and no `map`, from softmax(M): the row pass writes each
// block's three planes directly, and the statistics of its rows as tgb200_get_mapping does.  Both write the same planes
// for the same probabilities, so a handle's projection equals tgb200_project_map of its tgb200_get_mapping, bit for bit.
static int project_blocks(tgb200_mapper* h, const float* map, int64_t rows, int64_t cols, int64_t ld, const float* X,
                          int64_t x_ld, const int64_t* indptr, const int32_t* indices, const float* data, int64_t nnz,
                          int64_t n_genes, float* out, int64_t block_rows, int32_t device, cudaStream_t s) {
  const bool csr = X == nullptr;
  if (csr == (indptr == nullptr)) return fail(TGB200_ERR_INVALID, "give exactly one of X (dense) and indptr (CSR)");
  if (rows <= 0 || cols <= 0 || ld < cols || n_genes <= 0 || rows > INT32_MAX || cols > INT32_MAX || n_genes > INT32_MAX - 64 ||
      (!csr && x_ld < n_genes))
    return fail(TGB200_ERR_INVALID, "bad shape rows=%lld cols=%lld ld=%lld n_genes=%lld x_ld=%lld", (long long)rows,
                (long long)cols, (long long)ld, (long long)n_genes, (long long)x_ld);
  if (csr && (nnz < 0 || (nnz > 0 && (!indices || !data))))
    return fail(TGB200_ERR_INVALID, "CSR with nnz=%lld needs indices and data", (long long)nnz);
  if (block_rows < 0 || block_rows % kProjUnit)
    return fail(TGB200_ERR_INVALID, "block_rows=%lld is not a multiple of %lld", (long long)block_rows, (long long)kProjUnit);
  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  // the row pointers are read on the host: every block's entry range is then known to lie inside [0, nnz)
  std::vector<int64_t> ip;
  if (csr) {
    ip.resize(rows + 1);
    CK(cudaMemcpyAsync(ip.data(), indptr, sizeof(int64_t) * (rows + 1), cudaMemcpyDefault, s));
    CK(cudaStreamSynchronize(s));
    if (ip[0] != 0 || ip[rows] != nnz)
      return fail(TGB200_ERR_INVALID, "CSR indptr runs from %lld to %lld, expected 0 to nnz=%lld", (long long)ip[0],
                  (long long)ip[rows], (long long)nnz);
    for (int64_t r = 0; r < rows; ++r)
      if (ip[r + 1] < ip[r]) return fail(TGB200_ERR_INVALID, "CSR indptr decreases at row %lld", (long long)r);
  }
  const int64_t ldm = round_up(cols, 64), ldx = round_up(n_genes, 64), cap = round_up(rows, kProjUnit);
  auto max_nnz = [&](int64_t B) {
    int64_t m = 0;
    for (int64_t r0 = 0; csr && r0 < rows; r0 += B) m = std::max(m, ip[std::min(rows, r0 + B)] - ip[r0]);
    return m;
  };
  // out, then per block: the mapping in three bf16 planes and, from `map`, twice in fp32 (copy target, double-buffered), X in
  // three planes and, double-buffered, in fp32 (dense) or as the block's CSR entries
  auto need = [&](int64_t B) {
    double b = 4.0 * cols * ldx + (h ? 0.0 : 2 * 4.0 * B * ldm) + 6.0 * B * ldm + 6.0 * B * ldx;
    return b + (csr ? 2 * (8.0 * max_nnz(B) + 8.0 * (B + 1)) : 2 * 4.0 * B * ldx);
  };
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const double avail = (double)free_b - 256.0 * (1 << 20);    // headroom for the launches' own allocations
  int64_t B = block_rows > 0 ? std::min(block_rows, cap)
                             : std::min(cap, std::max(kProjUnit, round_up(ceil_div(rows, kProjBlocks), kProjUnit)));
  while (block_rows == 0 && B > kProjUnit && need(B) > avail) B -= kProjUnit;
  if (need(B) > avail)
    return fail(TGB200_ERR_INVALID, "projecting a %lld x %lld mapping onto %lld genes needs %.2f GiB on device %d in blocks of "
                "%lld cells (%.2f GiB of it for the result); %.2f GiB are free", (long long)rows, (long long)cols,
                (long long)n_genes, need(B) / 1073741824.0, device, (long long)B, 4.0 * cols * ldx / 1073741824.0,
                free_b / 1073741824.0);

  DevBuf<float> O, Mf[2], Xf[2], D[2];
  DevBuf<__nv_bfloat16> Mp, Xp;
  DevBuf<int64_t> P[2];
  DevBuf<int> I[2], bad;
  CKS(O.alloc((size_t)cols * ldx, false));
  CKS(Mp.alloc((size_t)3 * B * ldm, false)); CKS(Xp.alloc((size_t)3 * B * ldx, false));
  CKS(bad.alloc(1, false));
  const int64_t block_nnz = max_nnz(B);
  for (int k = 0; k < 2; ++k) {
    if (!h) CKS(Mf[k].alloc((size_t)B * ldm, false));
    if (csr) {
      CKS(P[k].alloc(B + 1, false)); CKS(I[k].alloc(std::max<int64_t>(block_nnz, 1), false));
      CKS(D[k].alloc(std::max<int64_t>(block_nnz, 1), false));
    } else {
      CKS(Xf[k].alloc((size_t)B * ldx, false));
    }
  }
  // zeroed on `stream` before cp.start is recorded, so the copy stream's first writes come after them whatever kind of
  // stream the caller passed: the flag starts at 0 and the staging's pad columns stay finite
  CK(cudaMemsetAsync(bad.p, 0, sizeof(int), s));
  for (int k = 0; k < 2; ++k) {
    if (!h) CK(cudaMemsetAsync(Mf[k].p, 0, sizeof(float) * Mf[k].n, s));
    if (!csr) CK(cudaMemsetAsync(Xf[k].p, 0, sizeof(float) * Xf[k].n, s));
  }
  TcContext tc;
  if (tc_init(tc, g_err, sizeof(g_err))) return TGB200_ERR_CUDA;
  TcPlan pl;                                                   // the planes never move within the call
  if (tc_forward_plan(tc, pl, Mp.p, (size_t)B * ldm, Xp.p, (size_t)B * ldx, 3, (int)B, (int)cols, (int)ldx, (int)ldm, g_err,
                      sizeof(g_err)))
    return TGB200_ERR_CUDA;
  CopyStream cp;
  CK(cudaStreamCreateWithFlags(&cp.s, cudaStreamNonBlocking));
  for (cudaEvent_t* e : {&cp.start, &cp.copied[0], &cp.copied[1], &cp.freed[0], &cp.freed[1]})
    CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  CK(cudaEventRecord(cp.start, s));                            // inputs written on `stream` before the call
  CK(cudaStreamWaitEvent(cp.s, cp.start, 0));

  const int64_t n_blocks = ceil_div(rows, B);
  // block b's inputs into slot b % 2 on the copy stream, once the contraction stream has consumed block b - 2 from it
  auto stage = [&](int64_t b) -> int {
    const int k = (int)(b & 1);
    const int64_t r0 = b * B, nb = std::min(B, rows - r0), nb64 = round_up(nb, 64);
    if (b >= 2) CK(cudaStreamWaitEvent(cp.s, cp.freed[k], 0));
    if (nb < nb64 && !csr)                                     // the last k-block reads up to nb64 rows: zero the tail
      CK(cudaMemsetAsync(Xf[k].p + nb * ldx, 0, sizeof(float) * (nb64 - nb) * ldx, cp.s));
    if (!h)
      CK(cudaMemcpy2DAsync(Mf[k].p, sizeof(float) * ldm, map + r0 * ld, sizeof(float) * ld, sizeof(float) * cols, nb,
                           cudaMemcpyDefault, cp.s));
    if (csr) {
      const int64_t e0 = ip[r0], ne = ip[r0 + nb] - e0;
      CK(cudaMemcpyAsync(P[k].p, ip.data() + r0, sizeof(int64_t) * (nb + 1), cudaMemcpyHostToDevice, cp.s));
      if (ne > 0) {
        CK(cudaMemcpyAsync(I[k].p, indices + e0, sizeof(int32_t) * ne, cudaMemcpyDefault, cp.s));
        CK(cudaMemcpyAsync(D[k].p, data + e0, sizeof(float) * ne, cudaMemcpyDefault, cp.s));
      }
    } else {
      CK(cudaMemcpy2DAsync(Xf[k].p, sizeof(float) * ldx, X + r0 * x_ld, sizeof(float) * x_ld, sizeof(float) * n_genes, nb,
                           cudaMemcpyDefault, cp.s));
    }
    CK(cudaEventRecord(cp.copied[k], cp.s));
    return TGB200_OK;
  };
  CKS(stage(0));
  for (int64_t b = 0; b < n_blocks; ++b) {
    const int k = (int)(b & 1);
    const int64_t r0 = b * B, nb = std::min(B, rows - r0), nb64 = round_up(nb, 64);
    CK(cudaStreamWaitEvent(s, cp.copied[k], 0));
    const Split3 mp{Mp.p, (size_t)B * ldm};
    if (h) {
      CKS(launch_softmax_rows<float>(h, s, (float*)nullptr, 0, nullptr, mp, (int)r0, (int)nb));     // ldm == h->ld
    } else {
      const long long m4 = nb * ldm / 4;
      k_split3<<<(unsigned)ceil_div(m4, 256), 256, 0, s>>>(Mf[k].p, mp, m4);
      CK(cudaGetLastError());
    }
    if (nb < nb64)                                             // the last k-block reads up to nb64 rows: zero the tail
      for (int p = 0; p < 3; ++p) CK(cudaMemsetAsync(Mp.p + ((size_t)p * B + nb) * ldm, 0, 2 * (nb64 - nb) * ldm, s));
    if (csr) {
      const CsrSplitArgs a{P[k].p, I[k].p, D[k].p, (int)nb, (int)nb64, (int)n_genes, (int)ldx, Split3{Xp.p, (size_t)B * ldx}, bad.p};
      k_csr_split3<<<(unsigned)ceil_div(nb64 * kWarp, kProjThreads), kProjThreads, 0, s>>>(a);
    } else {
      const long long x4 = nb64 * ldx / 4;
      k_split3<<<(unsigned)ceil_div(x4, 256), 256, 0, s>>>(Xf[k].p, Split3{Xp.p, (size_t)B * ldx}, x4);
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(cp.freed[k], s));
    // chains of 512 cells, added into out in cell order by the accumulating epilogue (fp32, round-to-nearest)
    for (int64_t c0 = 0; c0 < nb; c0 += kProjChain)
      CKS(tc_forward_launch_rows(tc, pl, 6, O.p, b > 0 || c0 > 0, (int)c0, (int)std::min(nb, c0 + kProjChain), (int)cols,
                                 (int)ldx, 0, s, g_err, sizeof(g_err)));
    if (b + 1 < n_blocks) CKS(stage(b + 1));                   // after block b's launches: its copies run under them
  }
  int bad_host = 0;
  CK(cudaMemcpyAsync(&bad_host, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad_host)
    return fail(TGB200_ERR_INVALID, "a CSR column index is outside [0, %lld) or not strictly increasing within its row",
                (long long)n_genes);
  CK(cudaMemcpy2DAsync(out, sizeof(float) * n_genes, O.p, sizeof(float) * ldx, sizeof(float) * n_genes, cols,
                       cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_project_map(const float* map, int64_t rows, int64_t cols, int64_t ld, const float* X, int64_t x_ld,
                                  const int64_t* indptr, const int32_t* indices, const float* data, int64_t nnz,
                                  int64_t n_genes, float* out, int64_t block_rows, int32_t device, void* stream) {
  if (!map || !out) return fail(TGB200_ERR_INVALID, "null argument");
  return project_blocks(nullptr, map, rows, cols, ld, X, x_ld, indptr, indices, data, nnz, n_genes, out, block_rows, device,
                        (cudaStream_t)stream);
}

// softmax(M)^T X (tangram/utils.py:368) from the handle's M, X dense
extern "C" int tgb200_project(tgb200_mapper* h, const float* X, int64_t n_cols, float* out, void* stream) {
  if (!h || !X || !out || n_cols <= 0) return fail(TGB200_ERR_INVALID, "bad argument");
  if (!h->have_mapping) return fail(TGB200_ERR_STATE, "no mapping set");
  return project_blocks(h, nullptr, h->N, h->V, h->ld, X, n_cols, nullptr, nullptr, nullptr, 0, n_cols, out, 0, h->cfg.device,
                        (cudaStream_t)stream);
}

// Per-label column statistics of an expression matrix (scanpy's rank_genes_groups basic statistics), streamed over cell
// blocks of whole summation ranges (see group_stats.cuh for the order of additions).
namespace {
constexpr int64_t kGsBlocks = 8;          // default: about this many blocks, so the copies of one hide under the others
constexpr int64_t kGsMaxBlock = 32 * kGsRange;   // 32 ranges x the slabs fill the device; larger blocks only add partials
}  // namespace

// The pass behind tgb200_group_stats (value = kIdentity) and tgb200_group_stats_expm1 (kExpm1, y = expm1(scale * x)).
static int group_stats_pass(GsValue value, double scale, const float* X, int64_t x_ld, const int64_t* indptr,
                            const int32_t* indices, const float* data, int64_t nnz, int64_t rows, int64_t n_genes,
                            const int32_t* labels, int32_t n_labels, double* sum_out, double* sumsq_out,
                            int64_t* nnz_out, int64_t block_rows, int32_t device, void* stream) {
  const bool csr = X == nullptr;
  if (csr == (indptr == nullptr)) return fail(TGB200_ERR_INVALID, "give exactly one of X (dense) and indptr (CSR)");
  if (!labels || !sum_out || !sumsq_out) return fail(TGB200_ERR_INVALID, "null argument");
  if (rows <= 0 || n_genes <= 0 || rows > INT32_MAX || n_genes > INT32_MAX - kGsSlab || (!csr && x_ld < n_genes))
    return fail(TGB200_ERR_INVALID, "bad shape rows=%lld n_genes=%lld x_ld=%lld", (long long)rows, (long long)n_genes,
                (long long)x_ld);
  if (n_labels < 1) return fail(TGB200_ERR_INVALID, "n_labels=%d, must be at least 1", n_labels);
  if (csr && (nnz < 0 || (nnz > 0 && (!indices || !data))))
    return fail(TGB200_ERR_INVALID, "CSR with nnz=%lld needs indices and data", (long long)nnz);
  if (block_rows < 0 || block_rows % kGsRange)
    return fail(TGB200_ERR_INVALID, "block_rows=%lld is not a multiple of %d", (long long)block_rows, kGsRange);
  // per range of kGsRange cells: its labelled rows stably sorted by label (offsets in the range), cut into runs of one label
  const int64_t n_ranges = ceil_div(rows, kGsRange);
  std::vector<int> perm_g, run_label, run_len, cnt(n_labels, 0), touched;
  std::vector<int64_t> range_perm(n_ranges + 1, 0), range_run(n_ranges + 1, 0);
  perm_g.reserve(rows);
  for (int64_t c = 0; c < n_ranges; ++c) {
    const int64_t i0 = c * kGsRange, i1 = std::min(rows, i0 + kGsRange);
    touched.clear();
    for (int64_t i = i0; i < i1; ++i) {
      const int32_t l = labels[i];
      if (l < -1 || l >= n_labels)
        return fail(TGB200_ERR_INVALID, "label %d of row %lld is outside [-1, %d)", l, (long long)i, n_labels);
      if (l >= 0 && cnt[l]++ == 0) touched.push_back(l);
    }
    std::sort(touched.begin(), touched.end());
    const size_t base = perm_g.size();
    int at = 0;
    for (int l : touched) {                      // cnt[l] becomes the start of label l's run in the range
      run_label.push_back(l);
      run_len.push_back(cnt[l]);
      const int n = cnt[l];
      cnt[l] = at;
      at += n;
    }
    perm_g.resize(base + at);
    for (int64_t i = i0; i < i1; ++i)
      if (labels[i] >= 0) perm_g[base + cnt[labels[i]]++] = (int)(i - i0);
    for (int l : touched) cnt[l] = 0;
    range_perm[c + 1] = (int64_t)perm_g.size();
    range_run[c + 1] = (int64_t)run_label.size();
  }

  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  cudaStream_t s = (cudaStream_t)stream;
  // the row pointers are read on the host: every block's entry range is then known to lie inside [0, nnz)
  std::vector<int64_t> ip;
  if (csr) {
    ip.resize(rows + 1);
    CK(cudaMemcpyAsync(ip.data(), indptr, sizeof(int64_t) * (rows + 1), cudaMemcpyDefault, s));
    CK(cudaStreamSynchronize(s));
    if (ip[0] != 0 || ip[rows] != nnz)
      return fail(TGB200_ERR_INVALID, "CSR indptr runs from %lld to %lld, expected 0 to nnz=%lld", (long long)ip[0],
                  (long long)ip[rows], (long long)nnz);
    for (int64_t r = 0; r < rows; ++r)
      if (ip[r + 1] < ip[r]) return fail(TGB200_ERR_INVALID, "CSR indptr decreases at row %lld", (long long)r);
  }
  bool in_place = false;                         // dense X in this device's memory is read where it lives
  if (!csr) {
    cudaPointerAttributes at;
    CK(cudaPointerGetAttributes(&at, X));
    in_place = (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == device;
  }
  const int64_t T = n_labels, G = n_genes, ldx = round_up(n_genes, 4), cap = round_up(rows, kGsRange);
  // the most of something over the blocks of B cells: of runs, of labelled rows, of stored entries
  auto block_max = [&](int64_t B, auto&& f) {
    int64_t m = 0;
    for (int64_t r0 = 0; r0 < rows; r0 += B) m = std::max<int64_t>(m, f(r0, std::min(rows, r0 + B)));
    return m;
  };
  auto runs_of = [&](int64_t r0, int64_t r1) { return range_run[ceil_div(r1, kGsRange)] - range_run[r0 / kGsRange]; };
  auto perm_of = [&](int64_t r0, int64_t r1) { return range_perm[ceil_div(r1, kGsRange)] - range_perm[r0 / kGsRange]; };
  auto nnz_of = [&](int64_t r0, int64_t r1) { return csr ? ip[r1] - ip[r0] : 0; };
  auto table_ints = [&](int64_t B) {
    return block_max(B, perm_of) + 2 * block_max(B, runs_of) + B / kGsRange + T + 3;
  };
  // outputs, the partials of one block's runs, and per block double-buffered: its tables and its X (dense staging or CSR)
  auto need = [&](int64_t B) {
    double b = 24.0 * T * G + 20.0 * block_max(B, runs_of) * G + 2 * 4.0 * table_ints(B);
    if (csr) b += 2 * (8.0 * block_max(B, nnz_of) + 8.0 * (B + 1));
    else if (!in_place) b += 2 * 4.0 * B * ldx;
    return b;
  };
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const double avail = (double)free_b - 256.0 * (1 << 20);    // headroom for the launches' own allocations
  int64_t B = block_rows > 0 ? std::min(block_rows, cap)
                             : std::min({cap, kGsMaxBlock, std::max<int64_t>(kGsRange, round_up(ceil_div(rows, kGsBlocks), kGsRange))});
  while (block_rows == 0 && B > kGsRange && need(B) > avail) B -= kGsRange;
  if (need(B) > avail)
    return fail(TGB200_ERR_INVALID, "group statistics of %lld cells x %lld genes over %d labels need %.2f GiB on device %d in "
                "blocks of %lld cells (%.2f GiB of it for the result); %.2f GiB are free", (long long)rows, (long long)G,
                n_labels, need(B) / 1073741824.0, device, (long long)B, 24.0 * T * G / 1073741824.0,
                free_b / 1073741824.0);

  const int64_t n_blocks = ceil_div(rows, B), max_runs = block_max(B, runs_of);
  DevBuf<double> sum, sq, psum, psq;
  DevBuf<long long> cntd;
  DevBuf<int> pcnt, tab[2], I[2], bad;
  DevBuf<int64_t> P[2];
  DevBuf<float> Xf[2], D[2];
  CKS(sum.alloc((size_t)T * G, false)); CKS(sq.alloc((size_t)T * G, false)); CKS(cntd.alloc((size_t)T * G, false));
  CKS(psum.alloc((size_t)std::max<int64_t>(max_runs, 1) * G, false));
  CKS(psq.alloc((size_t)std::max<int64_t>(max_runs, 1) * G, false));
  CKS(pcnt.alloc((size_t)std::max<int64_t>(max_runs, 1) * G, false));
  CKS(bad.alloc(1, false));
  const int64_t block_nnz = block_max(B, nnz_of);
  for (int k = 0; k < 2; ++k) {
    CKS(tab[k].alloc(table_ints(B), false));
    if (csr) {
      CKS(P[k].alloc(B + 1, false)); CKS(I[k].alloc(std::max<int64_t>(block_nnz, 1), false));
      CKS(D[k].alloc(std::max<int64_t>(block_nnz, 1), false));
    } else if (!in_place) {
      CKS(Xf[k].alloc((size_t)B * ldx, false));
    }
  }
  // zeroed on `stream` before cp.start is recorded, so they come before everything the copy stream orders after it
  CK(cudaMemsetAsync(sum.p, 0, sizeof(double) * sum.n, s));
  CK(cudaMemsetAsync(sq.p, 0, sizeof(double) * sq.n, s));
  CK(cudaMemsetAsync(cntd.p, 0, sizeof(long long) * cntd.n, s));
  CK(cudaMemsetAsync(bad.p, 0, sizeof(int), s));
  CopyStream cp;
  CK(cudaStreamCreateWithFlags(&cp.s, cudaStreamNonBlocking));
  for (cudaEvent_t* e : {&cp.start, &cp.copied[0], &cp.copied[1], &cp.freed[0], &cp.freed[1]})
    CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
  CK(cudaEventRecord(cp.start, s));                            // inputs written on `stream` before the call
  CK(cudaStreamWaitEvent(cp.s, cp.start, 0));

  // block b's tables, one int array: perm | run_start | range_runs | lab_ptr | lab_runs (kept until the call returns)
  struct Tab { std::vector<int> v; int np, nr, nrg; };
  std::vector<Tab> tabs(n_blocks);
  auto build_table = [&](int64_t b) {
    Tab& t = tabs[b];
    const int64_t c0 = b * B / kGsRange, c1 = std::min(n_ranges, c0 + B / kGsRange);
    t.nrg = (int)(c1 - c0); t.np = (int)(range_perm[c1] - range_perm[c0]); t.nr = (int)(range_run[c1] - range_run[c0]);
    t.v.assign((size_t)t.np + 2 * t.nr + t.nrg + T + 3, 0);
    int* perm = t.v.data();
    int* run_start = perm + t.np;
    int* range_runs = run_start + t.nr + 1;
    int* lab_ptr = range_runs + t.nrg + 1;
    int* lab_runs = lab_ptr + T + 1;
    for (int64_t c = c0; c < c1; ++c)
      for (int64_t p = range_perm[c]; p < range_perm[c + 1]; ++p)
        perm[p - range_perm[c0]] = perm_g[p] + (int)((c - c0) * kGsRange);
    for (int k = 0; k < t.nr; ++k) run_start[k + 1] = run_start[k] + run_len[range_run[c0] + k];
    for (int64_t c = c0; c <= c1; ++c) range_runs[c - c0] = (int)(range_run[c] - range_run[c0]);
    for (int k = 0; k < t.nr; ++k) ++lab_ptr[run_label[range_run[c0] + k] + 1];
    for (int64_t l = 0; l < T; ++l) lab_ptr[l + 1] += lab_ptr[l];
    std::vector<int> next(lab_ptr, lab_ptr + T);
    for (int k = 0; k < t.nr; ++k) lab_runs[next[run_label[range_run[c0] + k]]++] = k;      // range order within a label
  };
  // block b's tables and X into slot b % 2 on the copy stream, once the compute stream has consumed block b - 2 from it
  auto stage = [&](int64_t b) -> int {
    const int k = (int)(b & 1);
    const int64_t r0 = b * B, nb = std::min(B, rows - r0);
    build_table(b);
    if (b >= 2) CK(cudaStreamWaitEvent(cp.s, cp.freed[k], 0));
    CK(cudaMemcpyAsync(tab[k].p, tabs[b].v.data(), sizeof(int) * tabs[b].v.size(), cudaMemcpyHostToDevice, cp.s));
    if (csr) {
      const int64_t e0 = ip[r0], ne = ip[r0 + nb] - e0;
      CK(cudaMemcpyAsync(P[k].p, ip.data() + r0, sizeof(int64_t) * (nb + 1), cudaMemcpyHostToDevice, cp.s));
      if (ne > 0) {
        CK(cudaMemcpyAsync(I[k].p, indices + e0, sizeof(int32_t) * ne, cudaMemcpyDefault, cp.s));
        CK(cudaMemcpyAsync(D[k].p, data + e0, sizeof(float) * ne, cudaMemcpyDefault, cp.s));
      }
    } else if (!in_place) {
      CK(cudaMemcpy2DAsync(Xf[k].p, sizeof(float) * ldx, X + r0 * x_ld, sizeof(float) * x_ld, sizeof(float) * n_genes, nb,
                           cudaMemcpyDefault, cp.s));
    }
    CK(cudaEventRecord(cp.copied[k], cp.s));
    return TGB200_OK;
  };
  CKS(stage(0));
  const unsigned n_slabs = (unsigned)ceil_div(G, kGsSlab);
  for (int64_t b = 0; b < n_blocks; ++b) {
    const int k = (int)(b & 1);
    const int64_t r0 = b * B, nb = std::min(B, rows - r0);
    const Tab& t = tabs[b];
    CK(cudaStreamWaitEvent(s, cp.copied[k], 0));
    GsArgs a{};
    a.n_genes = G;
    a.perm = tab[k].p;
    a.run_start = a.perm + t.np;
    a.range_runs = a.run_start + t.nr + 1;
    const int* lab_ptr = a.range_runs + t.nrg + 1;
    a.psum = psum.p; a.psq = psq.p; a.pcnt = pcnt.p;
    a.scale = scale;
    if (csr) {
      a.indptr = P[k].p; a.indices = I[k].p; a.data = D[k].p;
      k_gs_csr_check<<<(unsigned)ceil_div(nb * kWarp, kGsThreads), kGsThreads, 0, s>>>(P[k].p, I[k].p, (int)nb, G, bad.p);
      CK(cudaGetLastError());
    } else {
      a.x = in_place ? X + r0 * x_ld : Xf[k].p;
      a.ld = in_place ? x_ld : ldx;
      a.vec = a.ld % 4 == 0 && reinterpret_cast<uintptr_t>(a.x) % 16 == 0;
    }
    if (t.nr > 0) {
      const dim3 grid(n_slabs, (unsigned)t.nrg);
      if (value == GsValue::kExpm1) {
        if (csr) k_group_stats<true, GsValue::kExpm1><<<grid, kGsThreads, 0, s>>>(a);
        else k_group_stats<false, GsValue::kExpm1><<<grid, kGsThreads, 0, s>>>(a);
      } else {
        if (csr) k_group_stats<true, GsValue::kIdentity><<<grid, kGsThreads, 0, s>>>(a);
        else k_group_stats<false, GsValue::kIdentity><<<grid, kGsThreads, 0, s>>>(a);
      }
      CK(cudaGetLastError());
      const dim3 fgrid((unsigned)ceil_div(G, kGsThreads), (unsigned)std::min<int64_t>(T, 65535));
      k_group_stats_fold<<<fgrid, kGsThreads, 0, s>>>(psum.p, psq.p, pcnt.p, lab_ptr, lab_ptr + T + 1, n_labels, G, sum.p,
                                                      sq.p, cntd.p);
      CK(cudaGetLastError());
    }
    CK(cudaEventRecord(cp.freed[k], s));
    if (b + 1 < n_blocks) CKS(stage(b + 1));                   // after block b's launches: its copies run under them
  }
  int bad_host = 0;
  CK(cudaMemcpyAsync(&bad_host, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad_host)
    return fail(TGB200_ERR_INVALID, "a CSR column index is outside [0, %lld) or not strictly increasing within its row",
                (long long)n_genes);
  CK(cudaMemcpyAsync(sum_out, sum.p, sizeof(double) * T * G, cudaMemcpyDefault, s));
  CK(cudaMemcpyAsync(sumsq_out, sq.p, sizeof(double) * T * G, cudaMemcpyDefault, s));
  if (nnz_out) CK(cudaMemcpyAsync(nnz_out, cntd.p, sizeof(int64_t) * T * G, cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_group_stats(const float* X, int64_t x_ld, const int64_t* indptr, const int32_t* indices,
                                  const float* data, int64_t nnz, int64_t rows, int64_t n_genes,
                                  const int32_t* labels, int32_t n_labels, double* sum_out, double* sumsq_out,
                                  int64_t* nnz_out, int64_t block_rows, int32_t device, void* stream) {
  return group_stats_pass(GsValue::kIdentity, 1.0, X, x_ld, indptr, indices, data, nnz, rows, n_genes, labels, n_labels,
                          sum_out, sumsq_out, nnz_out, block_rows, device, stream);
}

extern "C" int tgb200_group_stats_expm1(const float* X, int64_t x_ld, const int64_t* indptr, const int32_t* indices,
                                        const float* data, int64_t nnz, int64_t rows, int64_t n_genes,
                                        const int32_t* labels, int32_t n_labels, double* sum_out, double* sumsq_out,
                                        int64_t* nnz_out, int64_t block_rows, int32_t device, void* stream,
                                        double scale) {
  if (!std::isfinite(scale)) return fail(TGB200_ERR_INVALID, "scale=%g is not finite", scale);
  return group_stats_pass(GsValue::kExpm1, scale, X, x_ld, indptr, indices, data, nnz, rows, n_genes, labels, n_labels,
                          sum_out, sumsq_out, nnz_out, block_rows, device, stream);
}

#ifdef TGB_OVERLAP_PROBE
// Debug build only (tools/overlap_probe.py): can a contraction chunk and an update chunk run side by side on disjoint SMs?
// `kind` 0 is the backward contraction G over chunk 1's rows, 1 the forward contraction F' over chunk 1's rows; its grid
// is capped at `cap` clusters (0: as many as fit) on the hi stream.  The update runs over chunk 0's rows on the lo
// stream, as the product launches it (`update_ctas` 0) or as a persistent grid of `update_ctas` CTAs that each hold a
// whole SM.  `what`: 1 the contraction alone, 2 the update alone, 3 both at once.  For each of `reps` repetitions `out`
// gets three ms: start to the end of the contraction, to the end of the update, to the end of both.  The kernels read
// and write the handle's buffers as a step does; what they leave there is not a training state.
extern "C" TGB200_API int tgb200_debug_overlap_probe(tgb200_mapper* h, int32_t kind, int32_t cap, int32_t update_ctas,
                                                     int32_t what, int32_t reps, float* out) {
  if (!h || !out || reps < 1 || what < 1 || what > 3) return fail(TGB200_ERR_INVALID, "bad argument");
  if (!h->bf16 || !h->pipelined || h->host_state || !h->plan_dp.ready || !h->plan_fwd.ready)
    return fail(TGB200_ERR_STATE, "needs a resident, pipelined bf16 handle that has run an iteration");
  CK(cudaSetDevice(h->cfg.device));
  const int c0 = h->chunk_row[0], c1 = h->chunk_row[1], c2 = h->chunk_row[2];
  const AdamScalars a = adam_scalars(h->cfg, h->step > 0 ? h->step : 1, 0.1f);
  const AdamRowsArgs ar{h->M.p, h->mb.p, h->v.p, h->dq.p, h->Pb.p, reinterpret_cast<const RowConst*>(h->rowc.p),
                        h->zsum.p, h->pxsum.p, h->l1sum.p, h->l2sum.p, h->ld, h->V, c0, c1,
                        h->cfg.lambda_r, h->cfg.lambda_l1, h->cfg.lambda_l2, a};
  const bool plain = ar.lam_r == 0.f && ar.lam_l1 == 0.f && ar.lam_l2 == 0.f;
  const int keep = cap > 0 ? std::max(0, h->tc.num_sms - 2 * cap) : 0;   // every SM of an H100 holds a cluster CTA
  cudaEvent_t ev[4];
  for (auto& e : ev) CK(cudaEventCreate(&e));
  int st = TGB200_OK;
  CK(cudaDeviceSynchronize());
  for (int r = 0; r < reps && st == TGB200_OK; ++r) {
    CK(cudaEventRecord(ev[0], h->hi));
    CK(cudaStreamWaitEvent(h->lo, ev[0], 0));
    if (what & 1) {
      if (kind == 0) {
        TcEpiDpStore epi{h->plan_dp.pt, h->plan_dp.dq, h->ld, h->rcenter.p, h->rpart.p, h->N};
        st = tc_dpstore_launch(h->tc, h->plan_dp, 1, epi, c1, c2, h->V, h->Ke, keep, h->hi, g_err, sizeof(g_err));
      } else {
        st = tc_forward_launch_rows(h->tc, h->plan_fwd, 1, h->Y.p, 1, c1, c2, h->V, h->Ke, keep, h->hi, g_err, sizeof(g_err));
      }
    }
    if (what & 2) {
      if (update_ctas <= 0) {
        if (adam_rows_launch(ar, h->lo)) st = fail(TGB200_ERR_CUDA, "launch adam_rows");
      } else if (plain) {
        k_adam_rows_probe<true><<<update_ctas, 512, 0, h->lo>>>(ar);
      } else {
        k_adam_rows_probe<false><<<update_ctas, 512, 0, h->lo>>>(ar);
      }
      if (cudaGetLastError() != cudaSuccess) st = fail(TGB200_ERR_CUDA, "launch adam_rows_probe");
    }
    CK(cudaEventRecord(ev[1], h->hi));
    CK(cudaEventRecord(ev[2], h->lo));
    CK(cudaStreamWaitEvent(h->hi, ev[2], 0));
    CK(cudaEventRecord(ev[3], h->hi));
    CK(cudaEventSynchronize(ev[3]));
    for (int i = 0; i < 3; ++i) CK(cudaEventElapsedTime(&out[3 * r + i], ev[0], ev[i + 1]));
  }
  for (auto& e : ev) cudaEventDestroy(e);
  return st;
}
#endif

#ifdef TGB_BWD_PHASE_PROBE
// Debug build only (tools/bwd_phase_probe.py): every later bf16 backward contraction on the handle's device records its
// tiles' phase stamps into `buf` (device memory, 16 x 8 bytes per tile; see g_bwd_probe in gemm_tc.cuh), until the
// next call.  Null stops the recording.
extern "C" TGB200_API int tgb200_debug_bwd_phase_probe(tgb200_mapper* h, void* buf) {
  if (!h) return fail(TGB200_ERR_INVALID, "bad argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpyToSymbol(g_bwd_probe, &buf, sizeof(buf)));
  return TGB200_OK;
}
#endif

// Spatial neighbour graph (squidpy's gr.spatial_neighbors): exact k-nearest and radius search over a uniform cell grid
// (see neighbors.cuh for the kernels and the stop bound).
namespace {
constexpr int64_t kNbMaxCellsPerAxis = int64_t(1) << 24;   // keeps the rounding of scaled coordinates below 1e-8 cells
constexpr int64_t kNbMaxCells = int64_t(1) << 28;

int64_t nb_cell_cap(int64_t n) { return std::min<int64_t>(2 * n + 64, kNbMaxCells); }

// Cells of width h, about `per_cell` points each over the non-degenerate axes' box, at least min_h wide, grown until
// the grid has at most `cap` cells and no axis more than kNbMaxCellsPerAxis.
nb::Grid nb_grid(const double lo[3], const double ext[3], int64_t n, double per_cell, double min_h, int64_t cap) {
  double log_vol = 0.0, max_ext = 0.0;
  int d_eff = 0;
  for (int a = 0; a < 3; ++a) {
    if (ext[a] > 0) { log_vol += std::log(ext[a]); ++d_eff; }
    max_ext = std::max(max_ext, ext[a]);
  }
  double h = d_eff ? std::exp((log_vol + std::log(per_cell / (double)n)) / d_eff) : 1.0;
  h = std::max(h, min_h);
  if (!(h > 0) || !std::isfinite(1.0 / h)) h = max_ext > 0 ? max_ext : 1.0;
  nb::Grid g{};
  for (;;) {
    const double inv = 1.0 / h;
    double total = 1.0;
    bool ok = true;
    for (int a = 0; a < 3; ++a) {
      const double c = std::floor(ext[a] * inv) + 1.0;
      ok &= c <= (double)kNbMaxCellsPerAxis;
      total *= c;
    }
    if (ok && total <= (double)cap) {
      g.inv_h = inv;
      for (int a = 0; a < 3; ++a) { g.lo[a] = lo[a]; g.nc[a] = (int)(std::floor(ext[a] * inv) + 1.0); }
      break;
    }
    h *= 1.25;
  }
  g.h_lo = (1.0 / g.inv_h) * (1.0 - 1e-9);
  if (!(g.h_lo > 1e-150)) g.h_lo = 0.0;        // distances that small underflow when squared: no early stop
  return g;
}

// One search's device state: the staged coordinates, the points in cell order and the cell offsets.
struct NbSearch {
  DevBuf<double> C, xs, ys, zs;
  DevBuf<int> orig, cell, count, bad;
  DevBuf<long long> start, tiles;
  DevBuf<unsigned long long> box;
  nb::Grid g{};
  int n = 0;
  nb::Points points() const { return nb::Points{xs.p, ys.p, zs.p, orig.p, start.p}; }
};

int64_t nb_scan_tiles(int64_t n) { return ceil_div(n, nb::kScanTile); }

// out[0..n] = exclusive prefix of in[0..n) and the total; tiles holds 2 (tiles + 1) values.
int nb_scan(const int* in, int64_t n, long long* out, long long* tiles, cudaStream_t s) {
  const int64_t nt = nb_scan_tiles(n);
  nb::k_nb_scan_tiles<<<(unsigned)nt, 256, 0, s>>>(in, n, out, tiles);
  CK(cudaGetLastError());
  lrng::k_scan_counts<<<1, 1024, 0, s>>>(tiles, (int)nt, tiles + nt + 1);
  CK(cudaGetLastError());
  nb::k_nb_scan_add<<<(unsigned)ceil_div(n + 1, nb::kThreads), nb::kThreads, 0, s>>>(out, n, tiles + nt + 1, (int)nt);
  CK(cudaGetLastError());
  return TGB200_OK;
}

// Device bytes of a search over n points before its output: staged and sorted points, cell ids, the cell histogram
// and offsets at the cell cap, the scan's tiles.
double nb_search_bytes(int64_t n, int dim) {
  const int64_t cells = nb_cell_cap(n);
  return 8.0 * n * dim + 32.0 * n + 4.0 * n + 12.0 * (cells + 1) + 16.0 * (nb_scan_tiles(std::max(cells, n) + 1) + 1);
}

// Stages the coordinates, checks them, sizes the grid and sorts the points into cell order.  `out_bytes`: the caller's
// output buffers, counted in the memory check.
int nb_build(const double* coords, int64_t n, int dim, double per_cell, double min_h, double out_bytes, int32_t device,
             cudaStream_t s, const char* what, NbSearch& S) {
  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  const double need = nb_search_bytes(n, dim) + out_bytes, avail = (double)free_b - 256.0 * (1 << 20);
  if (need > avail)
    return fail(TGB200_ERR_INVALID, "%s over %lld points in %d-D needs %.3f GiB on device %d (%.3f GiB of it for the "
                "output); %.3f GiB are free", what, (long long)n, dim, need / 1073741824.0, device,
                out_bytes / 1073741824.0, free_b / 1073741824.0);
  S.n = (int)n;
  CKS(S.C.alloc((size_t)n * dim, false));
  CK(cudaMemcpyAsync(S.C.p, coords, sizeof(double) * n * dim, cudaMemcpyDefault, s));
  unsigned long long box0[6];
  for (int a = 0; a < 3; ++a) { box0[2 * a] = ~0ull; box0[2 * a + 1] = 0ull; }
  CKS(S.box.alloc(6, false));
  CKS(S.bad.alloc(1, false));
  CK(cudaMemcpyAsync(S.box.p, box0, sizeof(box0), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(S.bad.p, 0, sizeof(int), s));
  const unsigned bb = (unsigned)std::min<int64_t>(ceil_div(n, nb::kThreads), 8 * (int64_t)n_sms);
  nb::k_nb_bbox<<<bb, nb::kThreads, 0, s>>>(S.C.p, (int)n, dim, S.box.p, S.bad.p);
  CK(cudaGetLastError());
  unsigned long long box[6];
  int bad = 0;
  CK(cudaMemcpyAsync(box, S.box.p, sizeof(box), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(&bad, S.bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (bad) return fail(TGB200_ERR_INVALID, "%s: a coordinate is not finite", what);
  double lo[3] = {0, 0, 0}, ext[3] = {0, 0, 0};
  for (int a = 0; a < dim; ++a) {
    lo[a] = nb::from_ordered_bits(box[2 * a]);
    ext[a] = nb::from_ordered_bits(box[2 * a + 1]) - lo[a];
    if (!std::isfinite(ext[a]))
      return fail(TGB200_ERR_INVALID, "%s: the coordinates of axis %d span more than the largest double", what, a);
  }
  S.g = nb_grid(lo, ext, n, per_cell, min_h, nb_cell_cap(n));
  const int64_t cells = (int64_t)S.g.nc[0] * S.g.nc[1] * S.g.nc[2];
  CKS(S.xs.alloc(n, false)); CKS(S.ys.alloc(n, false)); CKS(S.zs.alloc(n, false));
  CKS(S.orig.alloc(n, false)); CKS(S.cell.alloc(n, false));
  CKS(S.count.alloc(cells, false));
  CKS(S.start.alloc(cells + 1, false));
  CKS(S.tiles.alloc(2 * (nb_scan_tiles(std::max<int64_t>(cells, n) + 1) + 1), false));
  CK(cudaMemsetAsync(S.count.p, 0, sizeof(int) * cells, s));
  const unsigned pb = (unsigned)ceil_div(n, nb::kThreads);
  nb::k_nb_cells<<<pb, nb::kThreads, 0, s>>>(S.C.p, (int)n, dim, S.g, S.cell.p, S.count.p);
  CK(cudaGetLastError());
  CKS(nb_scan(S.count.p, cells, S.start.p, S.tiles.p, s));
  nb::k_nb_scatter<<<pb, nb::kThreads, 0, s>>>(S.C.p, (int)n, dim, S.cell.p, S.count.p, S.start.p, S.xs.p, S.ys.p, S.zs.p,
                                               S.orig.p);
  CK(cudaGetLastError());
  return TGB200_OK;
}

int nb_check(const double* coords, int64_t n, int32_t dim, int64_t min_n, const char* what) {
  if (!coords) return fail(TGB200_ERR_INVALID, "%s: null coordinates", what);
  if (dim != 2 && dim != 3) return fail(TGB200_ERR_INVALID, "%s: dim=%d, must be 2 or 3", what, dim);
  if (n < min_n || n > INT32_MAX)
    return fail(TGB200_ERR_INVALID, "%s: n=%lld points, must lie in [%lld, %d]", what, (long long)n, (long long)min_n,
                INT32_MAX);
  return TGB200_OK;
}
}  // namespace

extern "C" int tgb200_spatial_knn(const double* coords, int64_t n, int32_t dim, int32_t k, int32_t* indices_out,
                                  double* dist_out, int32_t device, void* stream) {
  const char* what = "k-nearest-neighbour search";
  CKS(nb_check(coords, n, dim, 2, what));
  if (!indices_out || !dist_out) return fail(TGB200_ERR_INVALID, "%s: null output", what);
  if (k < 1 || k > nb::kMaxK) return fail(TGB200_ERR_INVALID, "%s: k=%d, must lie in [1, %d]", what, k, nb::kMaxK);
  if (k >= n) return fail(TGB200_ERR_INVALID, "%s: k=%d needs more than k points, got n=%lld", what, k, (long long)n);
  cudaStream_t s = (cudaStream_t)stream;
  NbSearch S;
  CKS(nb_build(coords, n, dim, std::max(2.0, 0.5 * (k + 1)), 0.0, 12.0 * n * k, device, s, what, S));
  DevBuf<int> cols;
  DevBuf<double> dists;
  CKS(cols.alloc((size_t)n * k, false));
  CKS(dists.alloc((size_t)n * k, false));
  const unsigned pb = (unsigned)ceil_div(n, nb::kThreads);
  const nb::Points P = S.points();
  if (k <= 8) nb::k_nb_knn<8><<<pb, nb::kThreads, 0, s>>>(S.g, P, (int)n, k, cols.p, dists.p);
  else if (k <= 16) nb::k_nb_knn<16><<<pb, nb::kThreads, 0, s>>>(S.g, P, (int)n, k, cols.p, dists.p);
  else if (k <= 32) nb::k_nb_knn<32><<<pb, nb::kThreads, 0, s>>>(S.g, P, (int)n, k, cols.p, dists.p);
  else nb::k_nb_knn<64><<<pb, nb::kThreads, 0, s>>>(S.g, P, (int)n, k, cols.p, dists.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(indices_out, cols.p, sizeof(int) * n * k, cudaMemcpyDefault, s));
  CK(cudaMemcpyAsync(dist_out, dists.p, sizeof(double) * n * k, cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_spatial_radius(const double* coords, int64_t n, int32_t dim, double radius, int64_t* indptr_out,
                                     int32_t* indices_out, double* dist_out, int64_t capacity, int32_t device,
                                     void* stream) {
  const char* what = "radius search";
  CKS(nb_check(coords, n, dim, 1, what));
  if (!indptr_out) return fail(TGB200_ERR_INVALID, "%s: null indptr_out", what);
  if (!(radius >= 0) || !std::isfinite(radius))
    return fail(TGB200_ERR_INVALID, "%s: radius=%g, must be finite and non-negative", what, radius);
  if (capacity < 0 || (capacity > 0 && (!indices_out || !dist_out)))
    return fail(TGB200_ERR_INVALID, "%s: capacity=%lld needs indices_out and dist_out", what, (long long)capacity);
  cudaStream_t s = (cudaStream_t)stream;
  NbSearch S;
  // cells just wider than the radius: rings 0 and 1 hold every neighbour, and the bound after ring 1 exceeds it
  CKS(nb_build(coords, n, dim, 2.0, radius * (1.0 + 1e-5), 12.0 * (n + 1), device, s, what, S));
  DevBuf<int> count;
  DevBuf<long long> off;
  CKS(count.alloc(n, false));
  CKS(off.alloc(n + 1, false));
  const unsigned pb = (unsigned)ceil_div(n, nb::kThreads);
  const nb::Points P = S.points();
  nb::k_nb_radius<false><<<pb, nb::kThreads, 0, s>>>(S.g, P, (int)n, radius, count.p, nullptr, nullptr, nullptr);
  CK(cudaGetLastError());
  CKS(nb_scan(count.p, n, off.p, S.tiles.p, s));
  CK(cudaMemcpyAsync(indptr_out, off.p, sizeof(int64_t) * (n + 1), cudaMemcpyDefault, s));
  long long nnz = 0;
  CK(cudaMemcpyAsync(&nnz, off.p + n, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (nnz == 0 || nnz > capacity) return TGB200_OK;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  if (12.0 * nnz > (double)free_b - 256.0 * (1 << 20))
    return fail(TGB200_ERR_INVALID, "%s: %lld neighbour pairs need %.3f GiB on device %d; %.3f GiB are free", what, nnz,
                12.0 * nnz / 1073741824.0, device, free_b / 1073741824.0);
  DevBuf<int> cols;
  DevBuf<double> dists;
  CKS(cols.alloc(nnz, false));
  CKS(dists.alloc(nnz, false));
  nb::k_nb_radius<true><<<pb, nb::kThreads, 0, s>>>(S.g, P, (int)n, radius, nullptr, off.p, cols.p, dists.p);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(indices_out, cols.p, sizeof(int) * nnz, cudaMemcpyDefault, s));
  CK(cudaMemcpyAsync(dist_out, dists.p, sizeof(double) * nnz, cudaMemcpyDefault, s));
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}
