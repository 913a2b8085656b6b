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

template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  int alloc(size_t count, bool zero = true) {
    release();
    if (count == 0) return TGB200_OK;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e != cudaSuccess) { p = nullptr; return fail(TGB200_ERR_CUDA, "cudaMalloc(%zu B): %s", count * sizeof(T), cudaGetErrorString(e)); }
    n = count;
    if (zero) {
      e = cudaMemset(p, 0, count * sizeof(T));
      if (e != cudaSuccess) return fail(TGB200_ERR_CUDA, "cudaMemset: %s", cudaGetErrorString(e));
    }
    return TGB200_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
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

// one launch while recording is on (tgb200_profile_step / tgb200_debug_timeline): stream 0 caller, 1 hi, 2 lo, 3 sf
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
  // training-gene mask of the loss (tgb200_set_loss_genes): gene_act[k] in {0, 1} (Ke floats, device and host) when
  // `masked`; n_active of the K genes are in the loss
  bool masked = false;
  int n_active = 0;
  DevBuf<float> gene_act;
  std::vector<float> gene_act_host;
  DevBuf<float> gw;             // Ke: sparsity weight of each gene in the loss (k_gene_weights), for the validation
  // per-epoch validation in the loop (tgb200_set_validation): epoch e (counted from that call) is validated when
  // e % val_every == 0, into history columns 12-15 of its row
  int val_every = 0;
  int64_t val_epoch = 0;
  int64_t val_row = -1;         // fp32 / bf16x3: the row whose validation this iteration's forward computes (see loss_stage)
  bool val_fuse = false;        // tgb200_run, not its last iteration: a validation may wait for the next iteration's forward
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
  // Pipelining of the bf16 backward over cell chunks (rows [chunk_row[c], chunk_row[c+1]), multiples of 256):
  //   hi (high-priority stream): forward(c) ... loss ... backward contraction(c)        -- tensor-core bound
  //   lo (low-priority stream):  row-dot finalize(c), streaming Adam(c)                 -- HBM bound
  // Adam(c) runs under the contraction of chunk c+1 and, across the iteration boundary, under the next forward's
  // chunks; forward(c) of the next iteration waits only for Adam(c).  The caller's stream forks into hi at the
  // start of an API call and joins hi + lo at its end (tgb200_run joins once, after its last iteration).
  bool pipelined = false;
  int nchunks = 1, chunk_row[9] = {0};
  cudaStream_t hi = nullptr, lo = nullptr, sf = nullptr;     // sf: the NEXT iteration's forward chunks (see backward_bf16)
  cudaEvent_t ev_fork = nullptr, ev_join_hi = nullptr, ev_join_lo = nullptr, ev_join_sf = nullptr, ev_loss = nullptr;
  cudaEvent_t ev_g[8] = {}, ev_a[8] = {}, ev_f[8] = {};
  bool a_valid = false;         // ev_a[] were recorded by an earlier step_end and guard the rows of the next forward
  bool prefetch_next = false;   // tgb200_run, not its last iteration: issue the NEXT forward's chunks between this backward's chunks
  bool fwd_ahead = false;       // ... and they have been issued: the next step_begin skips its chunk loop
  bool defer_join = false;      // inside tgb200_run: no fork / join between its iterations
  bool serial = false;          // tgb200_profile_step: everything on the caller's stream, one kernel at a time
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
  h->records.push_back({name, s == h->hi ? 1 : (s == h->lo ? 2 : (s == h->sf ? 3 : 0)), e});
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

extern "C" int tgb200_create(const tgb200_config* cfg, tgb200_mapper** out) {
  if (!cfg || !out) return fail(TGB200_ERR_INVALID, "null argument");
  *out = nullptr;
  if (cfg->struct_size != (int32_t)sizeof(tgb200_config))
    return fail(TGB200_ERR_INVALID, "tgb200_config.struct_size=%d, expected %zu", cfg->struct_size, sizeof(tgb200_config));
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
  if (h->x3) A(h->dpf.alloc(nv, false));
  A(h->M.alloc(nv)); A(h->v.alloc(nv));
  if (h->bf16) A(h->mb.alloc(nv)); else A(h->m.alloc(nv));
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
  if (h->bf16) {
    // cell chunks of the pipelined backward: 4 from 32k cells up, 2 from 8k (a rank of an 8-way sharded 100k-cell run):
    // each chunk still fills the GPU several times over
    int nc = h->N >= 32768 ? 4 : (h->N >= 8192 ? 2 : 1);
    if (const char* e = getenv("TGB200_CHUNKS")) nc = atoi(e);
    if (nc < 1) nc = 1;
    if (nc > 8) nc = 8;
    if (h->constrained) nc = 1;              // the filter update couples all rows of an iteration
    while (nc > 1 && h->N / nc < 1024) --nc;
    h->nchunks = nc;
    for (int c = 0; c <= nc; ++c) h->chunk_row[c] = c == nc ? h->N : (int)round_up((int64_t)c * h->N / nc, 256);
  }
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

static int zero_moments(tgb200_mapper* h, cudaStream_t s) {
  if (h->bf16) CK(cudaMemsetAsync(h->mb.p, 0, h->mb.n * sizeof(__nv_bfloat16), s));
  else CK(cudaMemsetAsync(h->m.p, 0, h->m.n * sizeof(float), s));
  CK(cudaMemsetAsync(h->v.p, 0, h->v.n * sizeof(float), s));
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
    h->gene_act_host.swap(flags);
    CK(cudaMemcpyAsync(h->gene_act.p, h->gene_act_host.data(), sizeof(float) * h->Ke, cudaMemcpyHostToDevice, s));
  }
  if (h->have_expr) {
    k_row_norms<<<(unsigned)ceil_div(h->V, 8), 256, 0, s>>>(h->V, h->K, h->Ke, h->G.p, h->masked ? h->gene_act.p : nullptr, h->ngr.p);
    LAUNCH_CHECK("row_norms");
    CKS(gene_weights(h, s));
  }
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

// Per-epoch validation inside tgb200_run / step_end (Mapper.train(val_each=), mapping_optimizer.py:398-403).  The scratch
// of the validation's loss scalars is allocated here, on first use, never in the loop.
extern "C" int tgb200_set_validation(tgb200_mapper* h, int32_t every, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  if (every < 0) return fail(TGB200_ERR_INVALID, "every = %d < 0", every);
  if (h->in_step) return fail(TGB200_ERR_STATE, "set_validation inside a step");
  if (every > 0 && h->cfg.n_cells_global != h->N) return fail(TGB200_ERR_UNSUPPORTED, "validation on a sharded handle");
  CK(cudaSetDevice(h->cfg.device));
  if (every > 0) {
    if (!h->val_coef.p) CKS(h->val_coef.alloc(2 * (size_t)h->Ke + 2 * (size_t)h->V));
    if (!h->val_hist.p) CKS(h->val_hist.alloc(TGB200_HIST_COLS));
    if (!h->rowpart.p && !h->val_rowpart.p) CKS(h->val_rowpart.alloc((size_t)h->ncolchunk * h->V * 2));
  }
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
  CK(cudaMemsetAsync(h->M.p, 0, h->M.n * sizeof(float), s));
  CK(cudaMemcpy2DAsync(h->M.p, (size_t)h->ld * sizeof(float), M0, (size_t)h->V * sizeof(float),
                       (size_t)h->V * sizeof(float), h->N, cudaMemcpyDefault, s));
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
  const long long nq = (long long)h->N * (h->ld / 4);
  k_init_normal<<<(unsigned)ceil_div(nq, 256), 256, 0, s>>>(h->M.p, h->N, h->V, h->ld, seed, (long long)first_row);
  LAUNCH_CHECK("init_normal");
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
  CK(cudaMemsetAsync(h->M.p, 0, h->M.n * sizeof(float), s));
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
    for (int i = 0; i < nf; ++i) CK(cudaMemcpyAsync(&dev_vals[i], h->M.p + fl[i].idx, sizeof(float), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    patch_vals.resize(nf);
    for (int i = 0; i < nf; ++i) {
      patch_vals[i] = (float)polar_value_host(fl[i].w, fl[i].comp);
      if (std::memcmp(&patch_vals[i], &dev_vals[i], sizeof(float)) != 0) {
        CK(cudaMemcpyAsync(h->M.p + fl[i].idx, &patch_vals[i], sizeof(float), cudaMemcpyHostToDevice, s));
        ++n_changed;
      }
    }
    n_fixed = nf;
  }
  float cached = (float)start->gauss;
  if (hg && t_lo == 0) CK(cudaMemcpyAsync(h->M.p, &cached, sizeof(float), cudaMemcpyHostToDevice, s));   // normal 0
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
  const float* Mp = h->M.p + (size_t)row0 * h->ld;
  RowStat* st = h->stats.p + row0;
  // One CTA per row, the row cached in registers between the max / exp-sum / emit passes.  Wide rows use more threads with
  // fewer float4 slots each: registers/thread stay <= 40..64, so 48-64 warps stay resident per SM (256 x 12 slots held 24,
  // and the row pass was latency-bound at 0.46 of the HBM peak).  Rows wider than 6144 float4 re-read M.
#define SMX(T, ITEMS, MINB)                                                                         \
  k_softmax_rows<PT, T, ITEMS, MINB><<<nrows, T, 0, s>>>(Mp, h->ld, h->V, P, h->ld, st, rowaux, want_entropy, split)
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

// Streams of an API call: the caller's stream `s` forks into the handle's high-priority stream (which in turn feeds the
// low-priority one through per-chunk events) and joins both at the end.
static cudaStream_t work_stream(tgb200_mapper* h, cudaStream_t s) { return (h->pipelined && !h->serial) ? h->hi : s; }
static cudaStream_t update_stream(tgb200_mapper* h, cudaStream_t s) { return (h->pipelined && !h->serial) ? h->lo : s; }
static int fork_streams(tgb200_mapper* h, cudaStream_t s) {
  if (!h->pipelined || h->serial || h->defer_join) return TGB200_OK;
  CK(cudaEventRecord(h->ev_fork, s));
  CK(cudaStreamWaitEvent(h->hi, h->ev_fork, 0));
  return TGB200_OK;
}
static int join_streams(tgb200_mapper* h, cudaStream_t s) {
  if (!h->pipelined || h->serial || h->defer_join) return TGB200_OK;
  CK(cudaEventRecord(h->ev_join_hi, h->hi));
  CK(cudaStreamWaitEvent(s, h->ev_join_hi, 0));
  CK(cudaEventRecord(h->ev_join_lo, h->lo));
  CK(cudaStreamWaitEvent(s, h->ev_join_lo, 0));
  CK(cudaEventRecord(h->ev_join_sf, h->sf));
  CK(cudaStreamWaitEvent(s, h->ev_join_sf, 0));
  return TGB200_OK;
}

// bf16 mode, cells of chunk c: exact row statistics from the sums the update left (k_row_norm), the scaled forward operand,
// and -- when the forward is chunked -- this chunk's contribution to Y_ext.  `lseA` / `lseT` as they are for THAT forward.
static int forward_chunk(tgb200_mapper* h, cudaStream_t s, int c, int fresh, const float* lseA, float* lseT) {
  float* rowaux = needs_rowaux(h->cfg) ? h->rowaux.p : nullptr;
  if (!h->plan_fwd.ready)
    CKS(tc_forward_plan(h->tc, h->plan_fwd, h->Pb.p, (size_t)h->N * h->ld, h->Sxs.p, (size_t)h->N * h->Ke, 1, h->N, h->V, h->Ke, h->ld,
                        g_err, sizeof(g_err)));
  const int r0 = h->nchunks > 1 ? h->chunk_row[c] : 0, r1 = h->nchunks > 1 ? h->chunk_row[c + 1] : h->N;
  // rows of this chunk: the streaming Adam kernel of the previous iteration must have written their P and row sums
  if (h->a_valid && h->pipelined && !h->serial) CK(cudaStreamWaitEvent(s, h->ev_a[c], 0));
  k_row_norm<<<(unsigned)ceil_div(r1 - r0, 256), 256, 0, s>>>(fresh, h->zsum.p, h->pxsum.p, h->l1sum.p, h->l2sum.p,
                                                             lseA, lseT, h->inv_zt.p, h->stats.p, rowaux, r0, r1);
  LAUNCH_CHECK("row_norm");
  const long long nq = (long long)(r1 - r0) * (h->Ke / 4);
  k_scale_rows_bf16<<<(unsigned)ceil_div(nq, 256), 256, 0, s>>>(s_act(h), h->inv_zt.p, r0, r1, h->Ke, h->Sxs.p);
  LAUNCH_CHECK("scale_rows");
  if (h->nchunks > 1) {
    // chunk 0 overwrites the exchange buffer, the others add to it (same stream, fixed order): no partial planes to sum
    CKS(tc_forward_launch_rows(h->tc, h->plan_fwd, 1, h->Y.p, c > 0 ? 1 : 0, r0, r1, h->V, h->Ke, s, g_err, sizeof(g_err)));
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
      if (h->nchunks > 1) return TGB200_OK;
    } else {
      for (int c = 0; c < h->nchunks; ++c) CKS(forward_chunk(h, s, c, h->p_state == PState::fresh ? 1 : 0, h->lseA, h->lseT));
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
    if (!h->plan_fwd.ready) {
      const __nv_bfloat16* sB = h->bf16 ? h->Sxs.p : h->Sxb.p;
      CKS(tc_forward_plan(h->tc, h->plan_fwd, h->Pb.p, (size_t)h->N * h->ld, sB, (size_t)h->N * h->Ke, h->x3 ? 3 : 1, h->N, h->V, h->Ke,
                          h->ld, g_err, sizeof(g_err)));
    }
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

extern "C" int tgb200_step_begin(tgb200_mapper* h, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  cudaStream_t caller = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(check_ready(h));
  if (h->in_step) return fail(TGB200_ERR_STATE, "step_begin called twice without step_end");
  CKS(fork_streams(h, caller));
  cudaStream_t s = work_stream(h, caller);
  if (h->constrained) {
    // the filter logits were updated on the update stream at the end of the previous iteration
    if (h->a_valid && h->pipelined && !h->serial) CK(cudaStreamWaitEvent(s, h->ev_a[0], 0));
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
  if (needs_rowscalars(h->cfg) || h->constrained || val) {
    k_row_scalar_reduce<<<1, 1024, 0, s>>>(h->stats.p, needs_rowaux(h->cfg) ? h->rowaux.p : nullptr,
                                           h->constrained ? h->fsig.p : nullptr, h->N, h->Y.p + vk);
    LAUNCH_CHECK("row_scalar_reduce");
  }
  if (h->cfg.n_cells_global != h->N && h->fwd_splits > 1) {
    // sharded: the exchange buffer must hold this rank's complete partial sum
    k_sum_planes<<<(unsigned)ceil_div(vk, 256), 256, 0, s>>>(h->Ypart.p, h->fwd_splits, vk, h->Y.p);
    LAUNCH_CHECK("sum_planes");
  }
  CKS(join_streams(h, caller));
  h->in_step = true;
  return TGB200_OK;
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

// _val_loss_fn's parameters (:311-356, as tgb200_validation_terms sets them): gene-voxel and voxel-gene cosines with weight 1,
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
  p.val_log_v = logf((float)h->V); p.val_n = (float)h->N;
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
static int backward_bf16(tgb200_mapper* h, cudaStream_t s, cudaStream_t su, const AdamScalars& a) {
  if (!h->plan_dp.ready) {
    CKS(tc_dpstore_epi_plan(h->tc, h->plan_dp, h->Pb.p, h->dq.p, h->N, h->ld, g_err, sizeof(g_err)));
    CKS(tc_dpstore_plan(h->tc, h->plan_dp, h->Sxb.p, 0, h->dYb.p, 0, 1, h->N, h->V, h->Ke, g_err, sizeof(g_err)));
  }
  const bool two_streams = su != s;
  const bool prefetch = two_streams && h->prefetch_next && h->nchunks > 1 && !h->constrained;
  for (int c = 0; c < h->nchunks; ++c) {
    const int r0 = h->nchunks > 1 ? h->chunk_row[c] : 0, r1 = h->nchunks > 1 ? h->chunk_row[c + 1] : h->N;
    TcEpiDpStore epi{h->plan_dp.pt, h->plan_dp.dq, h->ld, h->rcenter.p, h->rpart.p, h->N};
    CKS(tc_dpstore_launch(h->tc, h->plan_dp, 1, epi, r0, r1, h->V, h->Ke, s, g_err, sizeof(g_err)));
    mark(h, s, "tc_gemm_bwd_dp");
    if (two_streams) {
      CK(cudaEventRecord(h->ev_g[c], s));
      CK(cudaStreamWaitEvent(su, h->ev_g[c], 0));
    }
    k_rowdot_finalize_staged<<<(unsigned)ceil_div(r1 - r0, 256), 256, 0, su>>>(h->rpart.p, h->r_parts, h->N, r0, r1, h->lseT, h->inv_zt.p,
                                                                               h->stats.p, h->rcenter.p, h->rdot.p, h->rowc.p);
    { cudaStream_t s = su; LAUNCH_CHECK("rowdot_finalize"); }
    if (h->constrained) CKS(filter_update(h, su, a));
    AdamRowsArgs ar{h->M.p, h->mb.p, h->v.p, h->dq.p, h->Pb.p, reinterpret_cast<const RowConst*>(h->rowc.p),
                    h->zsum.p, h->pxsum.p, h->l1sum.p, h->l2sum.p, h->ld, h->V, r0, r1,
                    h->cfg.lambda_r, h->cfg.lambda_l1, h->cfg.lambda_l2, a};
    if (adam_rows_launch(ar, su)) return fail(TGB200_ERR_CUDA, "launch adam_rows: %s", cudaGetErrorString(cudaGetLastError()));
    mark(h, su, "adam_rows");
    if (two_streams) CK(cudaEventRecord(h->ev_a[c], su));
    h->a_valid = two_streams;
    // The next iteration's forward for this chunk goes to a third stream as soon as its rows are updated: the backward
    // contractions G(c+1..) run ahead on `s` (they feed the update), the update stream is never without tensor-core work
    // beside it, and nothing queues behind a kernel that still waits for the update.
    // (lseT of this iteration is the offset the new P was written with = lseA of the next; the other buffer is free.)
    if (prefetch) {
      if (c == 0) CK(cudaStreamWaitEvent(h->sf, h->ev_loss, 0));      // the partial planes of Y_ext were consumed by this iteration's loss
      CKS(forward_chunk(h, h->sf, c, 0, h->lseT, h->lseA));            // waits for ev_a[c]
      CK(cudaEventRecord(h->ev_f[c], h->sf));
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
  CKS(tc_dpstore_launch(h->tc, h->plan_dp, 6, epi, 0, h->N, h->V, h->Ke, s, g_err, sizeof(g_err)));
  mark(h, s, "tc_gemm_bwd_dp");
  k_rowdot_finalize<<<(unsigned)ceil_div(h->N, 256), 256, 0, s>>>(h->rpart.p, h->r_parts, h->N, h->rdot.p);
  LAUNCH_CHECK("rowdot_finalize");
  if (h->constrained) CKS(filter_update(h, s, a));
  AdamRowsExactArgs ar{h->M.p, h->m.p, h->v.p, h->dpf.p, h->stats.p, h->rdot.p, h->ld, h->V, 0, h->N,
                       h->cfg.lambda_r, h->cfg.lambda_l1, h->cfg.lambda_l2, a};
  if (adam_rows_exact_launch(ar, s)) return fail(TGB200_ERR_CUDA, "launch adam_rows_exact: %s", cudaGetErrorString(cudaGetLastError()));
  mark(h, s, "adam_rows");
  return TGB200_OK;
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

// The separate validation forward: what tgb200_validation_terms runs on the device, into out[0..3] (device), on `s`.
// bf16 mode re-runs the exact row pass, so the per-row entropy exists whatever lambda_r is; P is then fresh and the next
// iteration starts from it, exactly as after tgb200_validation_terms.
static int validation_forward(tgb200_mapper* h, cudaStream_t s, float* out) {
  if (h->bf16) { h->p_state = PState::stale; h->fwd_ahead = false; }
  CKS(forward_pass(h, s, 1));
  LossParams p = val_loss_params(h, out);
  CKS(reduce_columns(h, s, p, true, 1));
  k_row_scalar_reduce<<<1, 1024, 0, s>>>(h->stats.p, nullptr, nullptr, h->N, h->Y.p + (size_t)h->V * h->Ke);
  LAUNCH_CHECK("row_scalar_reduce");
  k_loss_scalars<true><<<1, 1024, 0, s>>>(p, 1, h->nredchunk, h->val_hist.p);
  LAUNCH_CHECK("loss_scalars");
  return TGB200_OK;
}

static bool val_due(const tgb200_mapper* h) { return h->val_every > 0 && h->val_epoch % h->val_every == 0; }

extern "C" int tgb200_step_end(tgb200_mapper* h, float lr, void* stream) {
  if (!h) return fail(TGB200_ERR_INVALID, "null handle");
  cudaStream_t caller = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  if (!h->in_step) return fail(TGB200_ERR_STATE, "step_end without step_begin");
  CKS(ensure_history(h, h->hist_len + 1, caller));
  CKS(fork_streams(h, caller));              // the caller may have all-reduced the exchange buffer on its stream
  cudaStream_t s = work_stream(h, caller);
  float* hist_row = h->hist.p + (size_t)h->hist_len * TGB200_HIST_COLS;
  // sharded: the caller all-reduced Y (already the sum of every rank's partial planes)
  const bool sharded = h->cfg.n_cells_global != h->N;
  CKS(loss_stage(h, s, hist_row, !sharded));
  if (h->pipelined && !h->serial) CK(cudaEventRecord(h->ev_loss, s));

  const AdamScalars a = adam_scalars(h->cfg, h->step + 1, lr);
  cudaStream_t su = update_stream(h, caller);
  if (h->bf16) CKS(backward_bf16(h, s, su, a));
  else if (h->x3) CKS(backward_bf16x3(h, s, a));
  else CKS(backward_fp32(h, s, a));
  // the validation of this epoch, on the mapping its update produced (mapping_optimizer.py:398-403)
  if (val_due(h)) {
    // fp32 / bf16x3 inside tgb200_run: the next iteration's forward serves it.  Constrained mode keeps the separate forward,
    // which (as tgb200_validation_terms) still sees the filter of this epoch; the next forward sees the updated one.
    if (h->val_fuse && !h->bf16 && !h->constrained) {
      h->val_row = h->hist_len;
    } else {
      if (su != s) {                           // the row pass reads every row the update stream wrote
        CK(cudaEventRecord(h->ev_join_lo, su));
        CK(cudaStreamWaitEvent(s, h->ev_join_lo, 0));
      }
      CKS(validation_forward(h, s, val_out_of(h, h->hist_len)));
    }
  }
  if (h->val_every > 0) h->val_epoch++;
  CKS(join_streams(h, caller));
  h->step++;
  h->hist_len++;
  h->in_step = false;
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
  CKS(fork_streams(h, (cudaStream_t)stream));
  h->defer_join = true;                      // iterations chain through the handle's own streams and events
  int st = TGB200_OK;
  for (int i = 0; i < n_steps && st == TGB200_OK; ++i) {
    // a validated bf16 epoch runs its own row pass after the update: no next forward issued ahead of it
    h->prefetch_next = i + 1 < n_steps && !val_due(h);
    h->val_fuse = i + 1 < n_steps;
    st = tgb200_step_begin(h, stream);
    if (st == TGB200_OK && sharded) st = exchange_partials(h, work_stream(h, (cudaStream_t)stream));
    if (st == TGB200_OK) st = tgb200_step_end(h, lr, stream);
  }
  h->defer_join = false;
  h->prefetch_next = false;
  h->val_fuse = false;
  h->val_row = -1;                           // set only when an iteration follows, unless that iteration failed
  CKS(join_streams(h, (cudaStream_t)stream));
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
  if (M) CK(cudaMemcpy2DAsync(M, w, h->M.p, pitch, w, h->N, cudaMemcpyDefault, s));
  if (m && !h->bf16) CK(cudaMemcpy2DAsync(m, w, h->m.p, pitch, w, h->N, cudaMemcpyDefault, s));
  if (m && h->bf16) {         // bf16 first moment -> fp32 for the caller
    float* scratch;
    int blk;
    DevBuf<float> one_row;
    CKS(moment_scratch(h, one_row, &scratch, &blk));
    for (int r0 = 0; r0 < h->N; r0 += blk) {
      const int nr = h->N - r0 < blk ? h->N - r0 : blk;
      const long long n = (long long)nr * h->ld;
      k_bf16_to_f32<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(h->mb.p + (size_t)r0 * h->ld, scratch, n);
      LAUNCH_CHECK("bf16_to_f32");
      CK(cudaMemcpy2DAsync(m + (size_t)r0 * h->V, w, scratch, pitch, w, nr, cudaMemcpyDefault, s));
    }
  }
  if (v) CK(cudaMemcpy2DAsync(v, w, h->v.p, pitch, w, h->N, cudaMemcpyDefault, s));
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
  if (M) {
    CK(cudaMemcpy2DAsync(h->M.p, pitch, M, w, w, h->N, cudaMemcpyDefault, s)); h->have_mapping = true; h->p_state = PState::stale;
    h->fwd_ahead = false;
    if (h->bf16) CK(cudaMemsetAsync(h->rcenter.p, 0, h->rcenter.n * sizeof(float), s));
  }
  if (m && !h->bf16) CK(cudaMemcpy2DAsync(h->m.p, pitch, m, w, w, h->N, cudaMemcpyDefault, s));
  if (m && h->bf16) {         // fp32 from the caller -> bf16 (exact for values that came out of tgb200_get_state)
    float* scratch;
    int blk;
    DevBuf<float> one_row;
    CKS(moment_scratch(h, one_row, &scratch, &blk));
    for (int r0 = 0; r0 < h->N; r0 += blk) {
      const int nr = h->N - r0 < blk ? h->N - r0 : blk;
      const long long n = (long long)nr * h->ld;
      CK(cudaMemsetAsync(scratch, 0, (size_t)n * sizeof(float), s));            // pad columns stay zero
      CK(cudaMemcpy2DAsync(scratch, pitch, m + (size_t)r0 * h->V, w, w, nr, cudaMemcpyDefault, s));
      k_f32_to_bf16<<<(unsigned)ceil_div(n, 256), 256, 0, s>>>(scratch, h->mb.p + (size_t)r0 * h->ld, n);
      LAUNCH_CHECK("f32_to_bf16");
    }
  }
  if (v) CK(cudaMemcpy2DAsync(h->v.p, pitch, v, w, w, h->N, cudaMemcpyDefault, s));
  h->step = step;
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_project(tgb200_mapper* h, const float* X, int64_t n_cols, float* out, void* stream) {
  if (!h || !X || !out || n_cols <= 0) return fail(TGB200_ERR_INVALID, "bad argument");
  if (!h->have_mapping) return fail(TGB200_ERR_STATE, "no mapping set");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  // softmax(M)^T X, gene columns streamed through in chunks (tangram/utils.py:368)
  const int chunk = 2048;
  if (h->tcm) {
    // tensor-core modes: the forward contraction kernel with split-bf16 operands (three planes each, six partial
    // products, accumulation chains cut at 2048 cells) -- fp32-grade results whatever the training precision was
    const size_t pplane = (size_t)h->N * h->ld;
    DevBuf<__nv_bfloat16> Pown, Xb;
    __nv_bfloat16* Pp = h->Pb.p;                    // bf16x3 mode rewrites its P planes every iteration anyway
    if (!h->x3) { CKS(Pown.alloc(3 * pplane, false)); Pp = Pown.p; }   // bf16 mode: Pb carries the unnormalised P state
    CKS(launch_softmax_rows<float>(h, s, (float*)nullptr, 0, nullptr, Split3{Pp, pplane}));
    const int ldc = (int)round_up(n_cols < chunk ? n_cols : chunk, 64);
    int splits = tc_forward_splits(h->tc.num_sms, h->N, h->V, ldc);
    { const int c = tc_splits_for_chain(h->N, 2048); if (c > splits) splits = c; }
    const size_t xplane = (size_t)h->N * ldc, oplane = (size_t)h->V * ldc;
    DevBuf<float> Xc, Opart, Oc;
    CKS(Xc.alloc(xplane)); CKS(Xb.alloc(3 * xplane, false)); CKS(Opart.alloc((size_t)splits * oplane, false));
    if (splits > 1) CKS(Oc.alloc(oplane, false));
    for (int64_t c0 = 0; c0 < n_cols; c0 += chunk) {
      const int nc = (int)((n_cols - c0) < chunk ? (n_cols - c0) : chunk);
      if (nc < ldc) CK(cudaMemsetAsync(Xc.p, 0, xplane * sizeof(float), s));
      CK(cudaMemcpy2DAsync(Xc.p, (size_t)ldc * sizeof(float), X + c0, (size_t)n_cols * sizeof(float),
                           (size_t)nc * sizeof(float), h->N, cudaMemcpyDefault, s));
      k_split3<<<(unsigned)ceil_div(xplane / 4, 256), 256, 0, s>>>(Xc.p, Split3{Xb.p, xplane}, (long long)(xplane / 4));
      LAUNCH_CHECK("split3");
      CKS(tc_forward(h->tc, Pp, pplane, Xb.p, xplane, 6, Opart.p, h->N, h->V, ldc, h->ld, splits, s, g_err, sizeof(g_err)));
      const float* res = Opart.p;
      if (splits > 1) {
        k_sum_planes<<<(unsigned)ceil_div(oplane, 256), 256, 0, s>>>(Opart.p, splits, oplane, Oc.p);
        LAUNCH_CHECK("sum_planes");
        res = Oc.p;
      }
      CK(cudaMemcpy2DAsync(out + c0, (size_t)n_cols * sizeof(float), res, (size_t)ldc * sizeof(float),
                           (size_t)nc * sizeof(float), h->V, cudaMemcpyDefault, s));
    }
    CK(cudaStreamSynchronize(s));
    return TGB200_OK;
  }
  CKS(launch_softmax_rows<float>(h, s, h->Pf.p, 0, nullptr));
  const int ldc = (int)round_up(n_cols < chunk ? n_cols : chunk, 4);
  DevBuf<float> Xc, Oc;
  CKS(Xc.alloc((size_t)h->N * ldc)); CKS(Oc.alloc((size_t)h->V * ldc));
  for (int64_t c0 = 0; c0 < n_cols; c0 += chunk) {
    const int nc = (int)((n_cols - c0) < chunk ? (n_cols - c0) : chunk);
    CK(cudaMemsetAsync(Xc.p, 0, Xc.n * sizeof(float), s));
    CK(cudaMemcpy2DAsync(Xc.p, (size_t)ldc * sizeof(float), X + c0, (size_t)n_cols * sizeof(float),
                         (size_t)nc * sizeof(float), h->N, cudaMemcpyDefault, s));
    GemmArgs g;
    g.A = h->Pf.p; g.lda = h->ld; g.B = Xc.p; g.ldb = ldc; g.M = h->V; g.N = nc; g.K = h->N;
    g.k_per_split = (int)round_up(h->N, 16);
    EpiStorePartial epi{Oc.p, ldc, 0};
    dim3 grid((unsigned)ceil_div(nc, SG_BN), (unsigned)ceil_div(h->V, SG_BM), 1);
    k_gemm_simt<false, false, EpiStorePartial><<<grid, SG_THREADS, 0, s>>>(g, epi);
    LAUNCH_CHECK("simt_gemm_project");
    CK(cudaMemcpy2DAsync(out + c0, (size_t)n_cols * sizeof(float), Oc.p, (size_t)ldc * sizeof(float),
                         (size_t)nc * sizeof(float), h->V, cudaMemcpyDefault, s));
  }
  CK(cudaStreamSynchronize(s));
  return TGB200_OK;
}

extern "C" int tgb200_validation_terms(tgb200_mapper* h, float* out4, void* stream) {
  if (!h || !out4) return fail(TGB200_ERR_INVALID, "null argument");
  cudaStream_t s = (cudaStream_t)stream;
  CK(cudaSetDevice(h->cfg.device));
  CKS(check_ready(h));
  if (h->in_step) return fail(TGB200_ERR_STATE, "validation_terms inside a step");
  if (h->cfg.n_cells_global != h->N) return fail(TGB200_ERR_UNSUPPORTED, "validation_terms on a sharded handle");
  // _val_loss_fn (:311-356): a second forward on the train matrices.  bf16 mode: re-run the exact row pass so that the
  // per-row entropy exists whatever lambda_r is (in steady state it is only carried when the entropy term is on)
  if (h->bf16) { h->p_state = PState::stale; h->fwd_ahead = false; }
  CKS(forward_pass(h, s, 1));
  LossParams p = make_loss_params(h);
  DevBuf<float> rowpart, coefAr, coefBr, hist;
  CKS(rowpart.alloc((size_t)h->ncolchunk * h->V * 2)); CKS(coefAr.alloc(h->V)); CKS(coefBr.alloc(h->V));
  CKS(hist.alloc(TGB200_HIST_COLS));
  p.rowpart = rowpart.p; p.coefAr = coefAr.p; p.coefBr = coefBr.p;
  p.lam_g2 = 1.f; p.lam_g1 = 1.f; p.lam_nb = 0.f; p.lam_go = 0.f; p.lam_ct = 0.f; p.density_mode = 0;
  CKS(reduce_columns(h, s, p, true, 1));
  k_row_scalar_reduce<<<1, 1024, 0, s>>>(h->stats.p, nullptr, nullptr, h->N, h->Y.p + (size_t)h->V * h->Ke);
  LAUNCH_CHECK("row_scalar_reduce");
  k_loss_scalars<false><<<1, 1024, 0, s>>>(p, 1, h->nredchunk, hist.p);
  LAUNCH_CHECK("loss_scalars");
  // sparsity-weighted gene score needs per-gene cosines: recover them from coefA/coefB on the host
  std::vector<float> hrow(TGB200_HIST_COLS), cA(h->K), cB(h->K), Gh((size_t)h->V * h->Ke), tail(4);
  CK(cudaMemcpyAsync(hrow.data(), hist.p, sizeof(float) * TGB200_HIST_COLS, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(cA.data(), h->coefA.p, sizeof(float) * h->K, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(cB.data(), h->coefB.p, sizeof(float) * h->K, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(Gh.data(), h->G.p, sizeof(float) * Gh.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(tail.data(), h->Y.p + (size_t)h->V * h->Ke, sizeof(float) * 4, cudaMemcpyDeviceToHost, s));
  std::vector<float> ngc(h->K);
  CK(cudaMemcpyAsync(ngc.data(), h->ngc.p, sizeof(float) * h->K, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  // cos_k = coefB_k * K' * ny^2 with ny = 1/(coefA_k * K' * ng)  (lam_g1 = 1 here; the K' genes of the loss)
  double wsum = 0.0, acc = 0.0;
  const double Kd = h->n_active;
  for (int k = 0; k < h->K; ++k) {
    if (h->masked && h->gene_act_host[k] == 0.f) continue;
    long nz = 0;
    for (int j = 0; j < h->V; ++j) nz += Gh[(size_t)j * h->Ke + k] != 0.f;
    const double w = (double)nz / h->V;       // 1 - gene_sparsity (:330)
    const double ny = 1.0 / ((double)cA[k] * Kd * ngc[k]);
    const double cosk = (double)cB[k] * Kd * ny * ny;
    wsum += w; acc += cosk * w;
  }
  const float gv = hrow[1], vg = hrow[2];
  out4[0] = gv + vg;                                   // expression_sim (:328)
  out4[1] = gv;                                        // gv_sim (:326)
  out4[2] = (float)(acc / wsum);                       // sp_sparsity_weighted_gv_sim (:331)
  out4[3] = -(tail[0] / logf((float)h->V)) / h->N;     // entropy (:333)
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
  cudaEvent_t e0;
  CK(cudaEventCreate(&e0));
  CK(cudaStreamSynchronize(s));
  CK(cudaEventRecord(e0, s));
  // the step's launches are appended to the records; a timeline recording in progress keeps them
  const bool timeline = h->recording;
  const size_t first = h->records.size();
  h->recording = true;
  h->serial = true;                          // one stream, one kernel at a time: clean per-kernel durations
  int st = tgb200_step_begin(h, stream);
  if (st == TGB200_OK) st = tgb200_step_end(h, lr, stream);
  h->serial = false;
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
  CK(cudaMemcpy(tmp.data(), src, tmp.size() * sizeof(__nv_bfloat16), cudaMemcpyDeviceToHost));
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
  if (nm == "Y") { src = h->Y.p; cnt = vk; }
  else if (nm == "M") { src = h->M.p; cnt = nv; }
  else if (nm == "v") { src = h->v.p; cnt = nv; }
  else if (nm == "m") {
    if (h->bf16) return widened(h->mb.p, nv, 1);
    src = h->m.p; cnt = nv;
  }
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
    CK(cudaMemcpy(out_host, src, cnt * sizeof(float), cudaMemcpyDeviceToHost));
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

extern "C" int tgb200_agreement(const float* const* arrays, int32_t R, int64_t rows, int64_t cols, int64_t ld,
                                double* pearson_out, float* vote_out, float* cons_out, int32_t device, void* stream) {
  if (!arrays) return fail(TGB200_ERR_INVALID, "null argument");
  if (R < 1 || R > kAgrMaxRuns) return fail(TGB200_ERR_INVALID, "R=%d runs, supported 1..%d", R, kAgrMaxRuns);
  if (rows <= 0 || cols <= 0 || ld < cols || cols > INT32_MAX)
    return fail(TGB200_ERR_INVALID, "bad shape rows=%lld cols=%lld ld=%lld", (long long)rows, (long long)cols, (long long)ld);
  int n_sms = 0;
  CKS(use_sm90_device(device, &n_sms));
  AgrArgs a{};
  a.rows = rows; a.cols = cols; a.ld = ld;
  a.vec = ld % 4 == 0;
  for (int r = 0; r < R; ++r) {
    if (!arrays[r]) return fail(TGB200_ERR_INVALID, "array %d is null", r);
    char what[32];
    snprintf(what, sizeof(what), "array %d", r);
    CKS(require_device_memory(arrays[r], device, what));
    a.x[r] = arrays[r];
    if (reinterpret_cast<uintptr_t>(arrays[r]) % 16) a.vec = 0;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const bool per_row = vote_out || cons_out;
  const int NS = R + R * (R + 1) / 2;
  int per_sm = 0;
#define AGR_OCC(RR) \
  case RR: CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, per_row ? k_agreement<RR, true> : k_agreement<RR, false>, kAgrThreads, 0)); break;
  switch (R) { AGR_OCC(1) AGR_OCC(2) AGR_OCC(3) AGR_OCC(4) AGR_OCC(5) AGR_OCC(6) AGR_OCC(7) AGR_OCC(8) }
#undef AGR_OCC
  const int warps = kAgrThreads / kWarp;
  const int64_t need = ceil_div(rows, warps);
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(need, (int64_t)std::max(per_sm, 1) * n_sms));
  // scratch is O(R^2 grid + rows): the per-block partials, the shifts, the correlations, the per-row results
  DevBuf<double> shift, part, corr;
  DevBuf<float> vote, cons;
  CKS(shift.alloc(R, false)); CKS(part.alloc((size_t)grid * NS, false)); CKS(corr.alloc(R > 1 ? R * (R - 1) / 2 : 1, false));
  if (vote_out) CKS(vote.alloc(rows, false));
  if (cons_out) CKS(cons.alloc(rows, false));
  a.shift = shift.p; a.part = part.p; a.vote = vote.p; a.cons = cons.p;
  k_agreement_shift<<<R, kAgrThreads, 0, s>>>(a, shift.p);
  CK(cudaGetLastError());
  switch (R) {
    case 1: launch_agreement<1>(a, grid, per_row, s); break;
    case 2: launch_agreement<2>(a, grid, per_row, s); break;
    case 3: launch_agreement<3>(a, grid, per_row, s); break;
    case 4: launch_agreement<4>(a, grid, per_row, s); break;
    case 5: launch_agreement<5>(a, grid, per_row, s); break;
    case 6: launch_agreement<6>(a, grid, per_row, s); break;
    case 7: launch_agreement<7>(a, grid, per_row, s); break;
    default: launch_agreement<8>(a, grid, per_row, s); break;
  }
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

extern "C" int tgb200_project_map(const float* map, int64_t rows, int64_t cols, int64_t ld, const float* X, int64_t x_ld,
                                  const int64_t* indptr, const int32_t* indices, const float* data, int64_t nnz,
                                  int64_t n_genes, float* out, int64_t block_rows, int32_t device, void* stream) {
  if (!map || !out) return fail(TGB200_ERR_INVALID, "null argument");
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
  const int64_t ldm = round_up(cols, 64), ldx = round_up(n_genes, 64), cap = round_up(rows, kProjUnit);
  auto max_nnz = [&](int64_t B) {
    int64_t m = 0;
    for (int64_t r0 = 0; csr && r0 < rows; r0 += B) m = std::max(m, ip[std::min(rows, r0 + B)] - ip[r0]);
    return m;
  };
  // out, then per block: the mapping twice in fp32 (copy target, double-buffered) and once in three bf16 planes, X in three
  // planes and, double-buffered, in fp32 (dense) or as the block's CSR entries
  auto need = [&](int64_t B) {
    double b = 4.0 * cols * ldx + 2 * 4.0 * B * ldm + 6.0 * B * ldm + 6.0 * B * ldx;
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
    CKS(Mf[k].alloc((size_t)B * ldm, false));
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
    CK(cudaMemsetAsync(Mf[k].p, 0, sizeof(float) * Mf[k].n, s));
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
    if (nb < nb64) {                                           // the last k-block reads up to nb64 rows: zero the tail
      CK(cudaMemsetAsync(Mf[k].p + nb * ldm, 0, sizeof(float) * (nb64 - nb) * ldm, cp.s));
      if (!csr) CK(cudaMemsetAsync(Xf[k].p + nb * ldx, 0, sizeof(float) * (nb64 - nb) * ldx, cp.s));
    }
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
    const long long m4 = nb64 * ldm / 4;
    k_split3<<<(unsigned)ceil_div(m4, 256), 256, 0, s>>>(Mf[k].p, Split3{Mp.p, (size_t)B * ldm}, m4);
    CK(cudaGetLastError());
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
                                 (int)ldx, s, g_err, sizeof(g_err)));
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
