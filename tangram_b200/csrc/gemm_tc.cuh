// wgmma / TMA tensor-core contraction path (sm_90a): bf16 operands staged in shared memory by
// TMA (128B swizzle), wgmma.mma_async issued by two consumer warpgroups, fp32 accumulators in
// registers, fused epilogues straight from the accumulator fragments.
//
//   forward   Y_ext[z] = P[z]^T S_ext[z]        A = P  (MN-major), B = S_ext (MN-major), split over cells / cell chunks
//   backward  dP = S_ext dY_ext^T  -> stored (bf16 centred / fp32) + row-dot partials in the epilogue (A, B K-major).
//             The update itself is a streaming kernel (adam_rows.cuh).
//
// Persistent, warp-specialised kernel: one CTA per SM loops over 128 x 256 output tiles.
//   warpgroup 0     TMA producer (one thread): keeps the operand ring full across tile boundaries, so the loads of
//                   tile i+1 run while the consumers drain tile i
//   warpgroups 1-2  consumers: rows [0, 64) / [64, 128) of the tile, m64n256k16 wgmma into 128 fp32 registers per
//                   thread, then the epilogue on those registers
#pragma once
#include <cuda.h>
#include <cstdio>
#include "common.cuh"
#include "gemm_simt.cuh"

namespace tgb {

constexpr int TC_BM = 128;        // output rows per tile (two 64-row wgmma warpgroups)
constexpr int TC_BK = 64;         // one 128-byte swizzle row of bf16 per k-block
constexpr int TC_MMA_K = 16;
constexpr int TC_BN = 256;        // output columns per tile (wgmma N)
constexpr int TC_THREADS = 384;   // producer warpgroup + two consumer warpgroups
constexpr int TC_ACC = TC_BN / 2; // fp32 accumulator registers per consumer thread

// ---- PTX wrappers ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// L2 policy: operand tiles are re-read by many CTAs -> evict_last (CUTLASS TMA::CacheHintSm90::EVICT_LAST)
constexpr uint64_t kPolicyEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kPolicyEvictLast = 0x14F0000000000000ull;
constexpr uint64_t kPolicyEvictFirst = 0x12F0000000000000ull;
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// register budget of the two roles (warpgroup-wide): 128 x 40 + 256 x 232 <= 64K registers
__device__ __forceinline__ void setmaxnreg_producer() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;"); }
__device__ __forceinline__ void setmaxnreg_consumer() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;"); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across the asynchronous MMAs
__device__ __forceinline__ void acc_fence(float (&d)[TC_ACC]) {
#pragma unroll
  for (int i = 0; i < TC_ACC; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (64 x 256, fp32, registers) (+)= A[smem] * B[smem], bf16 x bf16; TA / TB: operand stored MN-major (transposed)
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
      "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
      "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
      "}, %128, %129, p, 1, 1, %131, %132;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA), "n"(TB));
}
// ---- descriptors ----------------------------------------------------------------------------
// Shared-memory matrix descriptor (cute/arch/mma_sm90_desc.hpp GmmaDescriptor): start>>4 [0,14),
// LBO>>4 [16,30), SBO>>4 [32,46), layout SWIZZLE_128B=1 [62,64).
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// Operand tile in shared memory, one pipeline stage.
//   K-major  (rows = MN index, 64 k-elements = 128 B per row):   ROWS x 128 B, SBO = 1024 B (8 rows)
//   MN-major (rows = k index,  64 mn-elements = 128 B per row):  ROWS/64 boxes of [64 k][128 B];
//            LBO = 8192 B (next 64-wide MN atom), SBO = 1024 B (next 8 k-rows)
// Either way the 64-row half `h` of a tile starts 8192 B in.
template <bool KMAJOR, int ROWS>
struct OperandTile {
  static constexpr int kBytes = ROWS * TC_BK * 2;
  static __device__ __forceinline__ void load(const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int mn0, int k0, uint64_t policy) {
    if (KMAJOR) {
      tma_load_2d(map, bar, dst, k0, mn0, policy);               // box {64 k, ROWS mn}
    } else {
#pragma unroll
      for (int b = 0; b < ROWS / 64; ++b) tma_load_2d(map, bar, dst + b * 8192, mn0 + b * 64, k0, policy);  // box {64 mn, 64 k}
    }
  }
  static __device__ __forceinline__ uint64_t desc(uint32_t saddr, int k_step /* 0..3 */) {
    if (KMAJOR) return make_smem_desc(saddr + k_step * (TC_MMA_K * 2), 16, 1024);
    return make_smem_desc(saddr + k_step * (TC_MMA_K * 128), 8192, 1024);
  }
};

// ---- epilogues ------------------------------------------------------------------------------
// run() gets one consumer thread's accumulator fragment of the m64n256 wgmma: for every 8-column group j, d[4j], d[4j+1]
// are columns (8j + 2 (lane % 4), +1) of row `row`, and d[4j+2], d[4j+3] the same columns of row `row + 8`.  A quad of
// lanes covers 8 consecutive columns of a row (one 32-byte sector of fp32).  prologue() is called by all 256 consumer
// threads (`ct`) before the tile's main loop.
// Work item w -> (row tile m, column tile n).  Row tiles are taken in groups of `group_m`; inside a group the order is
// column-major (all rows of the group for column 0, then column 1, ...).  The CTAs running at the same time then cover
// the whole group for a few columns: the group's A rows (group_m x 128 x K, re-read for every column) are a small,
// hot L2 footprint and each B column tile is used in one burst.  group_m = 1 is plain column-fastest order.
__device__ __forceinline__ void tile_mn(int w, int tiles_m, int tiles_n, int group_m, int& m, int& n) {
  const int per_group = group_m * tiles_n;
  const int g = w / per_group, r = w - g * per_group;
  const int rows = min(group_m, tiles_m - g * group_m);
  n = r / rows;
  m = g * group_m + (r - n * rows);
}
struct TileCoord {
  int m0, n0;        // first output row / column of the tile
  int tile_n;        // column-tile index
  int tiles_n;       // number of column tiles
  int split;         // k-split index
};

__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

struct TcEpiStore {
  float* C; int ldc; size_t split_stride; int M;
  int accumulate;        // 1: C += tile (cell chunks of the pipelined forward run one after the other: fixed summation order)
  __device__ __forceinline__ void prologue(const TileCoord&, int) const {}
  __device__ __forceinline__ void run(const float (&d)[TC_ACC], const TileCoord& t, int row, int lane) const {
    float* base = C + (size_t)t.split * split_stride;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      if (r >= M) continue;
#pragma unroll
      for (int j = 0; j < TC_BN / 8; ++j) {
        const int col = t.n0 + 8 * j + 2 * (lane & 3);
        if (col < ldc) {
          float2* dst = reinterpret_cast<float2*>(base + (size_t)r * ldc + col);
          float2 v = make_float2(d[4 * j + 2 * h], d[4 * j + 2 * h + 1]);
          if (accumulate) { const float2 o = *dst; v.x += o.x; v.y += o.y; }
          *dst = v;
        }
      }
    }
  }
};

// Store-only backward epilogue (bf16 throughput mode, "staged" backward): dP = S_ext dY_ext^T leaves the kernel as
// bf16, centred per row on the previous iteration's row-dot (dq_ij = bf16(dP_ij - c_i): the softmax-Jacobian only sees
// dP_ij - r_i, so the bf16 rounding is relative to the deviation from the row mean, not to dP itself), and the same
// epilogue accumulates this iteration's row-dot partials r'_i = sum_j Pt_ij dq_ij from the ROUNDED values (so that
// sum_j g_ij = 0 holds for what the streaming Adam kernel consumes).  The Pt segment of the tile is prefetched into L2
// before the main loop.
struct TcEpiDpStore {
  __nv_bfloat16* dq; const __nv_bfloat16* Pt; int ld;     // both [rows][ld]
  const float* center;                                    // c_i (per row)
  float* rpart;                                           // [tiles_n][M]
  int M;
  __device__ __forceinline__ void prologue(const TileCoord& t, int ct) const {
#pragma unroll
    for (int i = ct; i < TC_BM * (TC_BN / 64); i += 256) {      // 128-byte lines of the tile's Pt block
      const int row = t.m0 + (i >> 2), col = t.n0 + (i & 3) * 64;
      if (row < M && col < ld) prefetch_l2(Pt + (size_t)row * ld + col);
    }
  }
  __device__ __forceinline__ void run(const float (&d)[TC_ACC], const TileCoord& t, int row, int lane) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      const bool live = r < M;
      const float c = live ? center[r] : 0.f;
      const __nv_bfloat16* prow = Pt + (size_t)r * ld;
      __nv_bfloat16* drow = dq + (size_t)r * ld;
      float racc = 0.f;
#pragma unroll
      for (int j = 0; j < TC_BN / 8; ++j) {
        const int col = t.n0 + 8 * j + 2 * (lane & 3);
        if (live && col < ld) {
          const __nv_bfloat162 d2 = __floats2bfloat162_rn(d[4 * j + 2 * h] - c, d[4 * j + 2 * h + 1] - c);
          const __nv_bfloat162 p2 = *reinterpret_cast<const __nv_bfloat162*>(prow + col);
          racc = fmaf(__low2float(p2), __low2float(d2), racc);
          racc = fmaf(__high2float(p2), __high2float(d2), racc);
          *reinterpret_cast<__nv_bfloat162*>(drow + col) = d2;
        }
      }
      racc = quad_sum(racc);
      if (live && (lane & 3) == 0) rpart[(size_t)t.tile_n * M + r] = racc;
    }
  }
};

// The same store-only backward for the parity mode (bf16x3): dP leaves the kernel in fp32 (nothing to centre) and the
// row-dot partials use P reconstructed from its three bf16 planes (hi + mid + lo = the fp32 value the row pass computed).
struct TcEpiDpStoreF32 {
  float* dp; int ld;                       // [rows][ld] fp32
  const __nv_bfloat16* P3; size_t plane;   // three planes of [rows][ld] bf16
  float* rpart;                            // [tiles_n][M]
  int M;
  __device__ __forceinline__ void prologue(const TileCoord& t, int ct) const {
#pragma unroll
    for (int i = ct; i < 3 * TC_BM * (TC_BN / 64); i += 256) {
      const int pl = i / (TC_BM * (TC_BN / 64)), li = i - pl * (TC_BM * (TC_BN / 64));
      const int row = t.m0 + (li >> 2), col = t.n0 + (li & 3) * 64;
      if (row < M && col < ld) prefetch_l2(P3 + pl * plane + (size_t)row * ld + col);
    }
  }
  __device__ __forceinline__ void run(const float (&d)[TC_ACC], const TileCoord& t, int row, int lane) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = row + 8 * h;
      const bool live = r < M;
      const __nv_bfloat16* prow = P3 + (size_t)r * ld;
      float* drow = dp + (size_t)r * ld;
      float racc = 0.f;
#pragma unroll
      for (int j = 0; j < TC_BN / 8; ++j) {
        const int col = t.n0 + 8 * j + 2 * (lane & 3);
        if (live && col < ld) {
          const __nv_bfloat162 h2 = *reinterpret_cast<const __nv_bfloat162*>(prow + col);
          const __nv_bfloat162 m2 = *reinterpret_cast<const __nv_bfloat162*>(prow + plane + col);
          const __nv_bfloat162 l2 = *reinterpret_cast<const __nv_bfloat162*>(prow + 2 * plane + col);
          const float p0 = (__low2float(l2) + __low2float(m2)) + __low2float(h2);
          const float p1 = (__high2float(l2) + __high2float(m2)) + __high2float(h2);
          const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
          racc = fmaf(p0, v0, racc);
          racc = fmaf(p1, v1, racc);
          *reinterpret_cast<float2*>(drow + col) = make_float2(v0, v1);
        }
      }
      racc = quad_sum(racc);
      if (live && (lane & 3) == 0) rpart[(size_t)t.tile_n * M + r] = racc;
    }
  }
};

// Per-row constants of the backward epilogue: lse = exact log-sum-exp of the row (P_ij = exp(M_ij - lse)),
// r = row-dot, h = sum_j P log P (entropy term only).
struct __align__(16) RowConst { float lse, r, h, pad; };

__device__ __forceinline__ float fast_ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_sqrt(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// ---- split-precision operands -------------------------------------------------------------------
// Parity mode on tensor cores ("bf16x3"): every fp32 operand value x is stored as three bf16 planes
// hi + mid + lo (x reconstructed to ~2^-24), and a*b is accumulated in fp32 from the six partial products
// whose magnitude is >= 2^-24 relative: (l,h) (h,l) (m,m) (m,h) (h,m) (h,h), smallest first.  The kernel
// simply runs its k-loop once per pair into the same accumulator; with n_pairs == 1 only (h,h) runs
// (plain bf16 mode).
struct TcMaps { CUtensorMap m[3]; };
__device__ __constant__ int kPairA[6] = {2, 0, 1, 1, 0, 0};
__device__ __constant__ int kPairB[6] = {0, 2, 1, 0, 1, 0};

// ---- the kernel -------------------------------------------------------------------------------
// Work item w -> (split z, row tile, column tile), column tile fastest so that CTAs running at the
// same time share A rows and stream B through L2.
template <bool A_KMAJOR, bool B_KMAJOR, int STAGES, class Epi>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_gemm_tc(const __grid_constant__ TcMaps maps_a, const __grid_constant__ TcMaps maps_b, int n_pairs,
          int k_total, int k_per_split, int tiles_m, int tiles_n, int splits, int group_m, uint64_t policy_a,
          uint64_t policy_b, int tm_off, int k_off, const Epi epi) {
  using TileA = OperandTile<A_KMAJOR, TC_BM>;
  using TileB = OperandTile<B_KMAJOR, TC_BN>;
  constexpr int kStageBytes = TileA::kBytes + TileB::kBytes;
  constexpr int kTA = A_KMAJOR ? 0 : 1, kTB = B_KMAJOR ? 0 : 1;
  constexpr uint32_t kConsumerWarps = 8;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int total = tiles_m * tiles_n * splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps_a.m[0]);
    tma_prefetch_desc(&maps_b.m[0]);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_producer();
    if (threadIdx.x == 0) {
      uint32_t kbg = 0;                         // k-blocks issued so far (ring position)
      for (int w = blockIdx.x; w < total; w += gridDim.x) {
        const int z = w / (tiles_n * tiles_m);
        int tm_i, tn_i;
        tile_mn(w - z * tiles_n * tiles_m, tiles_m, tiles_n, group_m, tm_i, tn_i);
        const int n0 = tn_i * TC_BN, m0 = (tm_off + tm_i) * TC_BM;
        const int k_begin = k_off + z * k_per_split;
        const int k_end = min(k_total, k_begin + k_per_split);
        const int num_kb = (k_end - k_begin + TC_BK - 1) / TC_BK;
        for (int pr = 6 - n_pairs; pr < 6; ++pr) {
          const CUtensorMap* ma = &maps_a.m[kPairA[pr]];
          const CUtensorMap* mb = &maps_b.m[kPairB[pr]];
          for (int kb = 0; kb < num_kb; ++kb, ++kbg) {
            const int s = kbg % STAGES;
            const uint32_t ph = (kbg / STAGES) & 1;
            mbar_wait(&empty_bar[s], ph ^ 1);
            uint8_t* sa = smem + s * kStageBytes;
            uint8_t* sb = sa + TileA::kBytes;
            mbar_expect_tx(&full_bar[s], kStageBytes);
            const int k0 = k_begin + kb * TC_BK;
            TileA::load(ma, &full_bar[s], sa, m0, k0, policy_a);
            TileB::load(mb, &full_bar[s], sb, n0, k0, policy_b);
          }
        }
      }
    }
  } else {
    // ===== consumers: wgmma main loop, then the fused epilogue on the accumulator registers =====
    setmaxnreg_consumer();
    const int cw = wg - 1;                      // rows [64 cw, 64 cw + 64) of the tile
    const int ct = threadIdx.x - 128;
    const int row_in_tile = 64 * cw + 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);
    float acc[TC_ACC];
#pragma unroll
    for (int i = 0; i < TC_ACC; ++i) acc[i] = 0.f;
    uint32_t kbg = 0;
    for (int w = blockIdx.x; w < total; w += gridDim.x) {
      TileCoord t;
      t.split = w / (tiles_n * tiles_m);
      int tm_i;
      tile_mn(w - t.split * tiles_n * tiles_m, tiles_m, tiles_n, group_m, tm_i, t.tile_n);
      t.tiles_n = tiles_n;
      t.n0 = t.tile_n * TC_BN;
      t.m0 = (tm_off + tm_i) * TC_BM;
      const int k_begin = k_off + t.split * k_per_split;
      const int k_end = min(k_total, k_begin + k_per_split);
      const int total_kb = (k_end - k_begin + TC_BK - 1) / TC_BK * n_pairs;
#ifndef TGB_SKIP_EPI
      epi.prologue(t, ct);
#endif
      acc_fence(acc);
      for (int kb = 0; kb < total_kb; ++kb, ++kbg) {
        const int s = kbg % STAGES;
        const uint32_t ph = (kbg / STAGES) & 1;
        mbar_wait(&full_bar[s], ph);
        const uint32_t sa = smem_u32(smem + s * kStageBytes) + cw * 8192;
        const uint32_t sb = smem_u32(smem + s * kStageBytes) + TileA::kBytes;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / TC_MMA_K; ++k)
          wgmma_m64n256k16<kTA, kTB>(acc, TileA::desc(sa, k), TileB::desc(sb, k), (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();                        // the MMAs of the previous k-block have retired: release its stage
        if (kb > 0 && lane == 0) mbar_arrive(&empty_bar[(kbg - 1) % STAGES]);
      }
      wgmma_wait<0>();
      acc_fence(acc);
      if (total_kb > 0 && lane == 0) mbar_arrive(&empty_bar[(kbg - 1) % STAGES]);
#ifndef TGB_SKIP_EPI
      epi.run(acc, t, t.m0 + row_in_tile, lane);
#endif
    }
  }
}

// ---- host side --------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TcContext {
  PFN_encodeTiled encode = nullptr;
  int num_sms = 132;
  const void* smem_fn[16] = {};   // kernels whose dynamic shared-memory limit this handle has already raised
  int smem_bytes[16] = {};
};

static inline int tc_init(TcContext& tc, char* err, size_t n) {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
    snprintf(err, n, "cuTensorMapEncodeTiled not available from the driver (%s)", cudaGetErrorString(e));
    return -2;
  }
  tc.encode = (PFN_encodeTiled)fn;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&tc.num_sms, cudaDevAttrMultiProcessorCount, dev);
  return 0;
}

// 2D bf16 row-major [rows][cols] (row pitch ld elements): inner dim = cols.  box = {box_inner, box_outer}.
static inline int tc_make_map(TcContext& tc, CUtensorMap* map, const void* base, uint64_t cols, uint64_t rows,
                              uint64_t ld, uint32_t box_inner, uint32_t box_outer, char* err, size_t n) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = tc.encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    snprintf(err, n, "cuTensorMapEncodeTiled failed (%d) cols=%llu rows=%llu ld=%llu box=%ux%u", (int)r,
             (unsigned long long)cols, (unsigned long long)rows, (unsigned long long)ld, box_inner, box_outer);
    return -2;
  }
  return 0;
}

// cudaFuncSetAttribute once per (handle, kernel): it is a driver call, not something to repeat on every launch
template <class Kern>
static inline int tc_set_smem(TcContext& tc, Kern kern, int bytes, char* err, size_t n) {
  const void* key = reinterpret_cast<const void*>(kern);
  int slot = -1;
  for (int i = 0; i < 16; ++i) {
    if (tc.smem_fn[i] == key) { if (tc.smem_bytes[i] == bytes) return 0; slot = i; break; }
    if (tc.smem_fn[i] == nullptr && slot < 0) slot = i;
  }
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) { snprintf(err, n, "cudaFuncSetAttribute(smem=%d): %s", bytes, cudaGetErrorString(e)); return -2; }
  if (slot >= 0) { tc.smem_fn[slot] = key; tc.smem_bytes[slot] = bytes; }
  return 0;
}
static inline int tc_check_launch(const char* name, char* err, size_t n) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { snprintf(err, n, "launch %s: %s", name, cudaGetErrorString(e)); return -2; }
  return 0;
}

// 4 stages of 48 KB (128 x 64 A + 256 x 64 B, bf16): 193 KB of the 227 KB an H100 block may use
constexpr int TC_STAGES = 4;
constexpr int TC_SMEM = TC_STAGES * (TC_BM + TC_BN) * TC_BK * 2 + 1024;
static inline int tc_dp_row_parts(int V) { return (int)ceil_div(V, TC_BN); }
// (tile_mn's row-tile groups stay at 1: more CTAs pulling the same B tile at once hot-spot L2 slices.)
static inline int tc_splits(int num_sms, long long tiles, long long k_total, int min_k) {
  long long s = (2LL * num_sms + tiles - 1) / tiles;
  const long long max_s = (k_total + min_k - 1) / min_k;
  if (s > max_s) s = max_s;
  if (s < 1) s = 1;
  // make every split non-empty
  const long long kps = ((k_total + s - 1) / s + TC_BK - 1) / TC_BK * TC_BK;
  return (int)((k_total + kps - 1) / kps);
}
// Parity mode: the tensor core accumulates in fp32 with truncation, a bias that grows with the length of the
// accumulation chain.  Chains are therefore cut at `max_chain` contraction elements; the partial results are summed
// in fp32 (round-to-nearest) by the kernels that consume them.
static inline int tc_splits_for_chain(long long k_total, int max_chain) {
  long long s = (k_total + max_chain - 1) / max_chain;
  if (s < 1) s = 1;
  const long long kps = ((k_total + s - 1) / s + TC_BK - 1) / TC_BK * TC_BK;
  return (int)((k_total + kps - 1) / kps);
}
static inline int tc_forward_splits(int num_sms, int N, int V, int Ke) {
  return tc_splits(num_sms, (long long)ceil_div(V, TC_BM) * ceil_div(Ke, TC_BN), N, 512);
}
static inline int tc_kps(int k_total, int splits) {
  return (int)(round_up(ceil_div(k_total, splits), TC_BK));
}
static inline unsigned tc_grid(const TcContext& tc, long long total) {
  return (unsigned)(total < tc.num_sms ? total : tc.num_sms);
}

// Operand planes: plane p of an operand starts at base + p * plane_elems (bf16).  n_pairs = 1 uses plane 0 only.
static inline int tc_make_maps(TcContext& tc, TcMaps* maps, const __nv_bfloat16* base, size_t plane_elems, int n_planes,
                               uint64_t cols, uint64_t rows, uint64_t ld, uint32_t bi, uint32_t bo, char* err, size_t n) {
  for (int p = 0; p < 3; ++p) {
    const __nv_bfloat16* ptr = base + (size_t)(p < n_planes ? p : 0) * plane_elems;
    if (tc_make_map(tc, &maps->m[p], ptr, cols, rows, ld, bi, bo, err, n)) return -2;
  }
  return 0;
}

// The tensor maps of one contraction over fixed device buffers.  cuTensorMapEncodeTiled is a driver call: the handle
// encodes each plan once (the buffers never move) instead of on every launch.
struct TcPlan {
  TcMaps a, b;
  bool ready = false;
};

// Y_ext[z] (V x Ke) = P[cells of split z]^T S_ext[...]
static inline int tc_forward_plan(TcContext& tc, TcPlan& pl, const __nv_bfloat16* P, size_t p_plane, const __nv_bfloat16* Sx,
                                  size_t s_plane, int planes, int N, int V, int Ke, int ld, char* err, size_t n) {
  if (tc_make_maps(tc, &pl.a, P, p_plane, planes, V, N, ld, 64, 64, err, n)) return -2;      // A: MN-major (voxels contiguous), rows = cells
  if (tc_make_maps(tc, &pl.b, Sx, s_plane, planes, Ke, N, Ke, 64, 64, err, n)) return -2;    // B: MN-major (genes contiguous), rows = cells
  pl.ready = true;
  return 0;
}
static inline int tc_forward_launch(TcContext& tc, const TcPlan& pl, int n_pairs, float* out, int N, int V, int Ke, int splits,
                                    cudaStream_t s, char* err, size_t n) {
  auto kern = k_gemm_tc<false, false, TC_STAGES, TcEpiStore>;
  if (tc_set_smem(tc, kern, TC_SMEM, err, n)) return -2;
  TcEpiStore epi{out, Ke, (size_t)V * Ke, V, 0};
  const int tm = (int)ceil_div(V, TC_BM), tn = (int)ceil_div(Ke, TC_BN);
  kern<<<tc_grid(tc, (long long)tm * tn * splits), TC_THREADS, TC_SMEM, s>>>(pl.a, pl.b, n_pairs, N, tc_kps(N, splits), tm, tn,
                                                                             splits, 1, kPolicyEvictNormal, kPolicyEvictNormal, 0, 0, epi);
  return tc_check_launch("tc_gemm_fwd", err, n);
}
// cells [row0, row1) only (row0 a multiple of 64): `out` = or += this chunk's partial sum -- the host pipelines cell chunks
// behind the streaming Adam kernel; the chunks run one after the other on one stream, so the summation order is fixed
static inline int tc_forward_launch_rows(TcContext& tc, const TcPlan& pl, float* out, int accumulate, int row0, int row1, int V, int Ke,
                                         cudaStream_t s, char* err, size_t n) {
  auto kern = k_gemm_tc<false, false, TC_STAGES, TcEpiStore>;
  if (tc_set_smem(tc, kern, TC_SMEM, err, n)) return -2;
  TcEpiStore epi{out, Ke, (size_t)V * Ke, V, accumulate};
  const int tm = (int)ceil_div(V, TC_BM), tn = (int)ceil_div(Ke, TC_BN);
  kern<<<tc_grid(tc, (long long)tm * tn), TC_THREADS, TC_SMEM, s>>>(pl.a, pl.b, 1, row1, (int)round_up(row1 - row0, TC_BK), tm, tn,
                                                                    1, 1, kPolicyEvictNormal, kPolicyEvictNormal, 0, row0, epi);
  return tc_check_launch("tc_gemm_fwd", err, n);
}
// one-shot variant for temporary operands (tgb200_project)
static inline int tc_forward(TcContext& tc, const __nv_bfloat16* P, size_t p_plane, const __nv_bfloat16* Sx, size_t s_plane,
                             int n_pairs, float* out, int N, int V, int Ke, int ld, int splits, cudaStream_t s, char* err,
                             size_t n) {
  TcPlan pl;
  if (tc_forward_plan(tc, pl, P, p_plane, Sx, s_plane, n_pairs > 1 ? 3 : 1, N, V, Ke, ld, err, n)) return -2;
  return tc_forward_launch(tc, pl, n_pairs, out, N, V, Ke, splits, s, err, n);
}

// Staged backward: dq = bf16(S_ext dY_ext^T - centre) (bf16 mode) or dP in fp32 (bf16x3 mode, three operand planes, six
// partial products) to HBM + row-dot partials; the update itself is a streaming kernel (adam_rows.cuh).  Rows [row0, row1)
// only (row0 a multiple of 128): the host pipelines row chunks.
static inline int tc_dpstore_plan(TcContext& tc, TcPlan& pl, const __nv_bfloat16* Sxb, size_t s_plane, const __nv_bfloat16* dYb,
                                  size_t dy_plane, int planes, int N, int V, int Ke, char* err, size_t n) {
  if (tc_make_maps(tc, &pl.a, Sxb, s_plane, planes, Ke, N, Ke, 64, TC_BM, err, n)) return -2;
  if (tc_make_maps(tc, &pl.b, dYb, dy_plane, planes, Ke, V, Ke, 64, TC_BN, err, n)) return -2;
  pl.ready = true;
  return 0;
}
template <class Epi>
static inline int tc_dpstore_launch(TcContext& tc, const TcPlan& pl, int n_pairs, const Epi& epi, int row0, int row1, int V, int Ke,
                                    cudaStream_t s, char* err, size_t n) {
  const int tn = (int)ceil_div(V, TC_BN);
  auto kern = k_gemm_tc<true, true, TC_STAGES, Epi>;
  if (tc_set_smem(tc, kern, TC_SMEM, err, n)) return -2;
  const int tm0 = row0 / TC_BM, tm = (int)ceil_div(row1, TC_BM) - tm0;
  kern<<<tc_grid(tc, (long long)tm * tn), TC_THREADS, TC_SMEM, s>>>(pl.a, pl.b, n_pairs, Ke, Ke, tm, tn, 1, 1,
                                                                    kPolicyEvictNormal, kPolicyEvictLast, tm0, 0, epi);
  return tc_check_launch("tc_gemm_bwd_dp", err, n);
}

}  // namespace tgb
