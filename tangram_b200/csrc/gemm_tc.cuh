// wgmma / TMA tensor-core contraction path (sm_90a): bf16 operands staged in shared memory by
// TMA (128B swizzle), wgmma.mma_async issued by two consumer warpgroups, fp32 accumulators in
// registers, fused epilogues on the accumulator fragments (the bf16 backward's through a shared-memory tile).
//
//   forward   Y_ext[z] = P[z]^T S_ext[z]        A = P  (MN-major), B = S_ext (MN-major), split over cells / cell chunks
//   backward  dP = S_ext dY_ext^T  -> stored (bf16 centred / fp32) + row-dot partials in the epilogue (A, B K-major).
//             The update itself is a streaming kernel (adam_rows.cuh).
//
// Persistent, warp-specialised kernel: one CTA per SM, in clusters of two that loop over pairs of 128 x 256 output tiles
// sharing their B tile (each CTA loads half of it and multicasts it to both).
//   warpgroup 0     TMA producer (one thread): keeps the operand ring full across tile boundaries, so the loads of
//                   tile i+1 run while the consumers drain tile i
//   warpgroups 1-2  consumers: rows [0, 64) / [64, 128) of the tile, m64n256k16 wgmma into 128 fp32 registers per
//                   thread, then the epilogue on those registers (the bf16 backward's: packed at once, the rest of it
//                   deferred into the next tile's first k-blocks)
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
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster (this CTA included).  It only
// says that this thread's reads of a stage are done (wgmma.wait_group has retired them); the writes it allows are the
// peer's TMA, so no cluster-scope release fence is needed (that would be a MEMBAR.GPU per k-block).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar)), "r"(cta) : "memory");
}
// cluster coordinates, read where they are used (asm volatile: not held in a register across the loops)
__device__ __forceinline__ int cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return (int)r; }
__device__ __forceinline__ int cluster_index() { uint32_t r; asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r)); return (int)r; }
__device__ __forceinline__ int cluster_count() { uint32_t r; asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r)); return (int)r; }
// every thread of every CTA of the cluster; orders the shared-memory writes before it (barrier init) cluster-wide
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}

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
// the same box written to `dst` and signalled on `bar` at the same offsets in both CTAs of the cluster
__device__ __forceinline__ void tma_load_2d_pair(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5, %6;"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"((uint16_t)0x3), "l"(policy) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// shared -> global tensor store, completion tracked by the issuing thread's bulk groups
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], %4;"
      ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "l"(policy) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the committed stores have finished reading shared memory (their global writes may still be in flight)
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// generic-proxy writes to shared memory become visible to the async proxy (TMA) of this CTA
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
template <int ID>
__device__ __forceinline__ void named_bar_sync(int threads) {
  asm volatile("bar.sync %0, %1;" ::"n"(ID), "r"(threads) : "memory");
}
// four 8 x 8 b16 matrices; lane l addresses row (l % 8) of matrix l / 8 and receives, from every matrix, the two
// elements of row l / 4, columns 2 (l % 4), +1 -- the wgmma accumulator fragment layout
__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
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
// D = A[smem] * B[smem], the first MMA of a tile: D is an output only, so whatever it held before is dead to the compiler
template <int TA, int TB>
__device__ __forceinline__ void wgmma_m64n256k16_first(float (&d)[128], uint64_t a_desc, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, 0, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
      "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
      "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
      "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63,"
      "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79,"
      "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95,"
      "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111,"
      "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
      "}, %128, %129, p, 1, 1, %130, %131;\n\t}"
      : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3]), "=f"(d[4]), "=f"(d[5]), "=f"(d[6]), "=f"(d[7]),
        "=f"(d[8]), "=f"(d[9]), "=f"(d[10]), "=f"(d[11]), "=f"(d[12]), "=f"(d[13]), "=f"(d[14]), "=f"(d[15]),
        "=f"(d[16]), "=f"(d[17]), "=f"(d[18]), "=f"(d[19]), "=f"(d[20]), "=f"(d[21]), "=f"(d[22]), "=f"(d[23]),
        "=f"(d[24]), "=f"(d[25]), "=f"(d[26]), "=f"(d[27]), "=f"(d[28]), "=f"(d[29]), "=f"(d[30]), "=f"(d[31]),
        "=f"(d[32]), "=f"(d[33]), "=f"(d[34]), "=f"(d[35]), "=f"(d[36]), "=f"(d[37]), "=f"(d[38]), "=f"(d[39]),
        "=f"(d[40]), "=f"(d[41]), "=f"(d[42]), "=f"(d[43]), "=f"(d[44]), "=f"(d[45]), "=f"(d[46]), "=f"(d[47]),
        "=f"(d[48]), "=f"(d[49]), "=f"(d[50]), "=f"(d[51]), "=f"(d[52]), "=f"(d[53]), "=f"(d[54]), "=f"(d[55]),
        "=f"(d[56]), "=f"(d[57]), "=f"(d[58]), "=f"(d[59]), "=f"(d[60]), "=f"(d[61]), "=f"(d[62]), "=f"(d[63]),
        "=f"(d[64]), "=f"(d[65]), "=f"(d[66]), "=f"(d[67]), "=f"(d[68]), "=f"(d[69]), "=f"(d[70]), "=f"(d[71]),
        "=f"(d[72]), "=f"(d[73]), "=f"(d[74]), "=f"(d[75]), "=f"(d[76]), "=f"(d[77]), "=f"(d[78]), "=f"(d[79]),
        "=f"(d[80]), "=f"(d[81]), "=f"(d[82]), "=f"(d[83]), "=f"(d[84]), "=f"(d[85]), "=f"(d[86]), "=f"(d[87]),
        "=f"(d[88]), "=f"(d[89]), "=f"(d[90]), "=f"(d[91]), "=f"(d[92]), "=f"(d[93]), "=f"(d[94]), "=f"(d[95]),
        "=f"(d[96]), "=f"(d[97]), "=f"(d[98]), "=f"(d[99]), "=f"(d[100]), "=f"(d[101]), "=f"(d[102]), "=f"(d[103]),
        "=f"(d[104]), "=f"(d[105]), "=f"(d[106]), "=f"(d[107]), "=f"(d[108]), "=f"(d[109]), "=f"(d[110]), "=f"(d[111]),
        "=f"(d[112]), "=f"(d[113]), "=f"(d[114]), "=f"(d[115]), "=f"(d[116]), "=f"(d[117]), "=f"(d[118]), "=f"(d[119]),
        "=f"(d[120]), "=f"(d[121]), "=f"(d[122]), "=f"(d[123]), "=f"(d[124]), "=f"(d[125]), "=f"(d[126]), "=f"(d[127])
      : "l"(a_desc), "l"(b_desc), "n"(TA), "n"(TB));
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
  // MN rows [h ROWS/2, (h + 1) ROWS/2) of the tile, multicast to both CTAs of the cluster: in either layout they are the
  // 16 KB starting h ROWS/2 * 128 B in
  static __device__ __forceinline__ void load_half_pair(const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int mn0, int k0, int h,
                                                        uint64_t policy) {
    constexpr int HALF = ROWS / 2;
    if (KMAJOR) {
      tma_load_2d_pair(map, bar, dst + h * HALF * 128, k0, mn0 + h * HALF, policy);         // box {64 k, ROWS/2 mn}
    } else {
#pragma unroll
      for (int b = 0; b < HALF / 64; ++b)
        tma_load_2d_pair(map, bar, dst + h * HALF * 128 + b * 8192, mn0 + h * HALF + b * 64, k0, policy);
    }
  }
  static __device__ __forceinline__ uint64_t desc(uint32_t saddr, int k_step /* 0..3 */) {
    if (KMAJOR) return make_smem_desc(saddr + k_step * (TC_MMA_K * 2), 16, 1024);
    return make_smem_desc(saddr + k_step * (TC_MMA_K * 128), 8192, 1024);
  }
};

// ---- phase probe (debug build only) --------------------------------------------------------------
#ifdef TGB_BWD_PHASE_PROBE
// tools/bwd_phase_probe.py: for every (tile, consumer warpgroup) of the bf16 backward, thread 0 of the warpgroup writes
// clock64() at six points of the tile's life (kBwdProbe*), the SM it ran on and globaltimer at the first one, into
// g_bwd_probe[(tile * 2 + cw) * 8 + ...], tile = row tile * column tiles + column tile.  Null: nothing is recorded.
enum { kBwdProbeFull, kBwdProbeRetired, kBwdProbePtFull, kBwdProbeStmatrix, kBwdProbeStore, kBwdProbeRead, kBwdProbeSm, kBwdProbeNs };
__device__ unsigned long long* g_bwd_probe;
__device__ __forceinline__ void bwd_probe(long long tile, int cw, int what) {
  if (g_bwd_probe == nullptr || tile < 0 || (threadIdx.x & 127) != 0) return;
  unsigned long long* p = g_bwd_probe + (tile * 2 + cw) * 8;
  p[what] = clock64();
  if (what == kBwdProbeFull) {
    unsigned long long ns;
    uint32_t sm;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
    asm volatile("mov.u32 %0, %%smid;" : "=r"(sm));
    p[kBwdProbeSm] = sm;
    p[kBwdProbeNs] = ns;
  }
}
#define TGB_BWD_PROBE(tile, cw, what) bwd_probe(tile, cw, what)
#else
#define TGB_BWD_PROBE(tile, cw, what) ((void)0)
#endif

// ---- epilogues ------------------------------------------------------------------------------
// run() gets one consumer thread's accumulator fragment of the m64n256 wgmma: for every 8-column group j, d[4j], d[4j+1]
// are columns (8j + 2 (lane % 4), +1) of row `row`, and d[4j+2], d[4j+3] the same columns of row `row + 8`.  A quad of
// lanes covers 8 consecutive columns of a row (one 32-byte sector of fp32).  prologue() is called by all 256 consumer
// threads (`ct`) before the tile's main loop.
// An epilogue may also own kSmemBytes of shared memory after the operand ring (EpiSmem).  load() is then called by the
// producer thread during the tile's main loop (TcEpiDpStore: in two rounds, at fixed k-blocks) to fill it.
// Each consumer warpgroup `cw` owns one full / free mbarrier pair for its half; `parity` is the current phase of both.
// A deferred epilogue (kDeferred) has no run(): its tile's accumulators are packed into registers right after the last
// MMA, and the rest runs as kSteps steps interleaved with the next tile's first k-blocks (see k_gemm_tc).
struct EpiSmem {
  uint8_t* buf;          // 1024-byte aligned
  uint64_t* full;        // [2] arrive count 1 + transaction bytes: the producer's load of half cw has landed
  uint64_t* free;        // [2] arrive count 1: consumer warpgroup cw no longer needs its half
  uint32_t parity;
};
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
  static constexpr int kSmemBytes = 0;
  static constexpr bool kDeferred = false;
  float* C; int ldc; size_t split_stride; int M;
  int accumulate;        // 1: C += tile (cell chunks of the pipelined forward run one after the other: fixed summation order)
  __device__ __forceinline__ void prologue(const TileCoord&, int) const {}
  __device__ __forceinline__ void load(int, int, const EpiSmem&) const {}
  __device__ __forceinline__ void run(const float (&d)[TC_ACC], const TileCoord& t, int row, int lane, int, const EpiSmem&) const {
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
// sum_j g_ij = 0 holds for what the streaming Adam kernel consumes).
// The tile's Pt comes in by TMA in two rounds of 128 columns, each into a 128 x 128 bf16 shared-memory tile (per 64-row
// half two 64 x 64 boxes of 8 KB, 128-byte swizzle); the epilogue reads a round with ldmatrix, writes dq over it with
// stmatrix and each consumer warpgroup stores its half of the round with TMA.  Both streams use evict_first: they pass
// through L2 once, beside the dY_ext operand that every tile re-reads.  A 32 KB buffer (instead of one for the whole
// 64 KB tile) leaves room for a fourth operand stage.
// The epilogue is deferred: pack() turns the accumulators into the 64 bf16x2 values that become dq as soon as the tile's
// last MMA retires, so the next tile's MMAs can start at once, and step(0..7) then does the shared-memory half, each step
// right after one of the next tile's k-blocks (step_kb): per round, one 64-column box of ldmatrix / row-dot / stmatrix in
// each of two steps, the TMA store, and the release of the buffer one k-block later.  The row-dot sums the same rounded
// values in the same order as an epilogue run in one piece, so dq and rpart do not depend on the deferral.
struct TcEpiDpStore {
  static constexpr int kSmemBytes = TC_BM * (TC_BN / 2) * 2;
  static constexpr int kHalfBytes = kSmemBytes / 2;
  static constexpr int kBoxBytes = 64 * 128;
  static constexpr bool kDeferred = true;
  static constexpr int kSteps = 8;                        // per round: two boxes, the store, the release
  static constexpr int kRound1Kb = 10;                    // the second round's steps start after this k-block
  // k-block of the next tile after which step s runs: round 0 after k-blocks 0-3, round 1 after kRound1Kb..+3
  static __host__ __device__ constexpr int step_kb(int s) { return s < 4 ? s : kRound1Kb + s - 4; }
  // Producer: the previous tile's second round is loaded after the current tile's kLoadKb1-th k-block, the current
  // tile's first round after its kLoadKb0-th.  The rounds are released after k-blocks 3 and kRound1Kb + 3, and the
  // producer runs at most STAGES (4) k-blocks ahead of the consumers, so neither load waits for its release or holds up
  // the ring; the second round still lands well before its steps.
  static constexpr int kLoadKb1 = 8, kLoadKb0 = 18;
  CUtensorMap pt_map, dq_map;                             // Pt / dq [M][ld] bf16, box {64 columns, 64 rows}
  int ld;                                                 // a multiple of 64
  const float* center;                                    // c_i (per row)
  float* rpart;                                           // [tiles_n][M]
  int M;
  // boxes of the 64-row half starting at row r0 that hold data; with ld a multiple of 64 a box lies wholly inside
  // [0, ld) or wholly past it, and TMA clips the rows >= M of a partly filled one
  __device__ __forceinline__ int boxes(int r0, int n0) const { return r0 < M ? min(TC_BN / 64, (ld - n0) / 64) : 0; }
  // the tile's index among all tiles of the contraction (the phase probe's record)
  __device__ __forceinline__ long long tile_id(int m0, int tile_n) const { return (long long)(m0 / TC_BM) * ((ld + TC_BN - 1) / TC_BN) + tile_n; }
  // c of this thread's rows `row`, `row + 8`, read before the tile's main loop
  __device__ __forceinline__ void centres(int row, float (&c)[2]) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) c[h] = row + 8 * h < M ? center[row + 8 * h] : 0.f;
  }
  // v[2j + h] = bf16(d - c) of columns 8j + 2 (lane % 4), +1 of row `row + 8h`
  static __device__ __forceinline__ void pack(const float (&d)[TC_ACC], const float (&c)[2], uint32_t (&v)[TC_ACC / 2]) {
#pragma unroll
    for (int j = 0; j < TC_BN / 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const __nv_bfloat162 d2 = __floats2bfloat162_rn(d[4 * j + 2 * h] - c[h], d[4 * j + 2 * h + 1] - c[h]);
        v[2 * j + h] = *reinterpret_cast<const uint32_t*>(&d2);
      }
    }
  }
  // Step s (a constant once the caller's loop is unrolled) of the epilogue of the tile at (m0, tile_n), whose packed
  // values are v; racc carries the row-dot from step to step.
  __device__ __forceinline__ void step(int s, const uint32_t (&v)[TC_ACC / 2], float (&racc)[2], int m0, int tile_n, int row,
                                       int lane, int cw, EpiSmem& es) const {
    const int r0 = m0 + 64 * cw, n0 = tile_n * TC_BN;
    const int nb = boxes(r0, n0);
    const int round = s / 4, sr = s % 4;
    if (sr < 2) {
      const int b = 2 * round + sr;                       // the box: columns 64 b .. +64 of the tile
      // ldmatrix / stmatrix address of this lane: row (lane % 8) of matrix lane / 8, where matrices 0..3 are
      // (rows +0, columns 8j), (rows +8, 8j), (rows +0, 8j + 8), (rows +8, 8j + 8) of the warp's 16 rows
      const int mi = lane >> 3, rr = lane & 7;
      const int arow = ((row - r0) & ~15) + 8 * (mi & 1) + rr;
      const uint32_t half = smem_u32(es.buf + cw * kHalfBytes) + arow * 128;
      if (sr == 0) {
        mbar_wait(&es.full[cw], es.parity);
        if (round == 0) {
          TGB_BWD_PROBE(tile_id(m0, tile_n), cw, kBwdProbePtFull);
          racc[0] = racc[1] = 0.f;
        }
      }
      if (b < nb) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {                     // columns 64 b + 16 q .. +16: j = 8 b + 2 q, +1
          const uint32_t addr = half + sr * kBoxBytes + (((2 * q + (mi >> 1)) ^ rr) << 4);
          uint32_t p[4], o[4];
          ldmatrix_x4(addr, p);
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int j = 8 * b + 2 * q + e;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const __nv_bfloat162 d2 = *reinterpret_cast<const __nv_bfloat162*>(&v[2 * j + h]);
              const __nv_bfloat162 p2 = *reinterpret_cast<const __nv_bfloat162*>(&p[2 * e + h]);
              racc[h] = fmaf(__low2float(p2), __low2float(d2), racc[h]);
              racc[h] = fmaf(__high2float(p2), __high2float(d2), racc[h]);
              o[2 * e + h] = v[2 * j + h];
            }
          }
          stmatrix_x4(addr, o);
        }
      }
      if (b == TC_BN / 64 - 1) TGB_BWD_PROBE(tile_id(m0, tile_n), cw, kBwdProbeStmatrix);
    } else if (sr == 2) {
      fence_proxy_async_smem();
      if (cw == 0) named_bar_sync<1>(128); else named_bar_sync<2>(128);    // this warpgroup's stmatrix writes are done
      if ((threadIdx.x & 127) == 0) {
        for (int b = 2 * round; b < min(nb, 2 * round + 2); ++b)
          tma_store_2d(&dq_map, es.buf + cw * kHalfBytes + (b - 2 * round) * kBoxBytes, n0 + 64 * b, r0, kPolicyEvictFirst);
        bulk_commit();
      }
      if (round == 1) {
        TGB_BWD_PROBE(tile_id(m0, tile_n), cw, kBwdProbeStore);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float sum = quad_sum(racc[h]);
          if (row + 8 * h < M && (lane & 3) == 0) rpart[(size_t)tile_n * M + row + 8 * h] = sum;
        }
      }
    } else {
      if ((threadIdx.x & 127) == 0) {
        bulk_wait_read_all();                             // the half may be refilled once the stores have read it
        if (round == 1) TGB_BWD_PROBE(tile_id(m0, tile_n), cw, kBwdProbeRead);
        mbar_arrive(&es.free[cw]);
      }
      es.parity ^= 1;
    }
  }
  // round r (columns 128 r .. +128) of the tile's Pt into the buffer, once the consumers have released it; the caller
  // flips es.parity after each round
  __device__ __forceinline__ void load(int m0, int n0, int r, const EpiSmem& es) const {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mbar_wait(&es.free[h], es.parity ^ 1);
      const int nb = min(2, max(0, boxes(m0 + 64 * h, n0) - 2 * r));
      mbar_expect_tx(&es.full[h], nb * kBoxBytes);
      for (int b = 0; b < nb; ++b)
        tma_load_2d(&pt_map, &es.full[h], es.buf + h * kHalfBytes + b * kBoxBytes, n0 + 128 * r + 64 * b, m0 + 64 * h,
                    kPolicyEvictFirst);
    }
  }
};

// The same store-only backward for the parity mode (bf16x3): dP leaves the kernel in fp32 (nothing to centre) and the
// row-dot partials use P reconstructed from its three bf16 planes (hi + mid + lo = the fp32 value the row pass computed).
struct TcEpiDpStoreF32 {
  static constexpr int kSmemBytes = 0;
  static constexpr bool kDeferred = false;
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
  __device__ __forceinline__ void load(int, int, const EpiSmem&) const {}
  __device__ __forceinline__ void run(const float (&d)[TC_ACC], const TileCoord& t, int row, int lane, int, const EpiSmem&) const {
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
// Launched as clusters of two CTAs.  Work item w -> (split z, pair of row tiles (2i, 2i + 1), column tile), column tile
// fastest so that clusters running at the same time share A rows and stream B through L2; the CTA of cluster rank r
// computes row tile 2i + r.  Both tiles need the same B tile: each CTA's producer loads its own A and one half of B, and
// multicasts that half into both CTAs' stages, so a stage reaches each CTA's full barrier as one A + two B halves, and
// it is refilled only once the consumers of both CTAs have released it (each consumer warp arrives on both CTAs' empty
// barriers).  With an odd number of row tiles the last pairs have a phantom second tile: that CTA loads no A, stores
// nothing and skips its epilogue, but loads and multicasts its half of B and takes part in every barrier.
template <bool A_KMAJOR, bool B_KMAJOR, int STAGES, class Epi>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_gemm_tc(const __grid_constant__ TcMaps maps_a, const __grid_constant__ TcMaps maps_b, int n_pairs,
          int k_total, int k_per_split, int tiles_m, int tiles_n, int splits, int group_m, uint64_t policy_a,
          uint64_t policy_b, int tm_off, int k_off, const __grid_constant__ Epi epi) {
  using TileA = OperandTile<A_KMAJOR, TC_BM>;
  using TileB = OperandTile<B_KMAJOR, TC_BN>;
  constexpr int kStageBytes = TileA::kBytes + TileB::kBytes;
  constexpr int kTA = A_KMAJOR ? 0 : 1, kTB = B_KMAJOR ? 0 : 1;
  constexpr uint32_t kConsumerWarps = 8;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  __shared__ __align__(8) uint64_t full_bar[STAGES];
  __shared__ __align__(8) uint64_t empty_bar[STAGES];
  __shared__ __align__(8) uint64_t epi_full[2], epi_free[2];

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int tiles_mp = (tiles_m + 1) / 2;                 // row-tile pairs
  const int total = tiles_mp * tiles_n * splits;
  EpiSmem es{smem + STAGES * kStageBytes, epi_full, epi_free, 0};

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&maps_a.m[0]);
    tma_prefetch_desc(&maps_b.m[0]);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2 * kConsumerWarps); }
    if constexpr (Epi::kSmemBytes > 0) {
      for (int h = 0; h < 2; ++h) { mbar_init(&epi_full[h], 1); mbar_init(&epi_free[h], 1); }
    }
    fence_barrier_init();
  }
  cluster_sync();                               // the peer's barriers are initialised before the first multicast

  if (wg == 0) {
    // ===== TMA producer =====
    setmaxnreg_producer();
    if (threadIdx.x == 0) {
      uint32_t kbg = 0;                         // k-blocks issued so far (ring position)
      int prev_m0 = -1, prev_n0 = 0;            // a live tile whose epilogue buffer still needs its second round
      (void)prev_n0;
      for (int w = cluster_index(); w < total; w += cluster_count()) {
        const int z = w / (tiles_n * tiles_mp);
        int tp_i, tn_i;
        tile_mn(w - z * tiles_n * tiles_mp, tiles_mp, tiles_n, group_m, tp_i, tn_i);
        const int tm_i = 2 * tp_i + cluster_rank();
        const bool live = tm_i < tiles_m;
        const int n0 = tn_i * TC_BN, m0 = (tm_off + tm_i) * TC_BM;
        const int k_begin = k_off + z * k_per_split;
        const int k_end = min(k_total, k_begin + k_per_split);
        const int num_kb = (k_end - k_begin + TC_BK - 1) / TC_BK;
        for (int pr = 6 - n_pairs; pr < 6; ++pr) {
          const CUtensorMap* ma = &maps_a.m[kPairA[pr]];
          const CUtensorMap* mb = &maps_b.m[kPairB[pr]];
#pragma unroll 1   // unrolled, the multicast loads do not fit the producer's 40 registers
          for (int kb = 0; kb < num_kb; ++kb, ++kbg) {
            const int s = kbg % STAGES;
            const uint32_t ph = (kbg / STAGES) & 1;
            mbar_wait(&empty_bar[s], ph ^ 1);
            uint8_t* sa = smem + s * kStageBytes;
            uint8_t* sb = sa + TileA::kBytes;
            mbar_expect_tx(&full_bar[s], live ? kStageBytes : TileB::kBytes);
            const int k0 = k_begin + kb * TC_BK;
            if (live) TileA::load(ma, &full_bar[s], sa, m0, k0, policy_a);
            TileB::load_half_pair(mb, &full_bar[s], sb, n0, k0, cluster_rank(), policy_b);
#ifndef TGB_SKIP_EPI
            // not before: waiting for the consumers to release the buffer would hold up the ring
            if constexpr (Epi::kSmemBytes > 0) {
              if (pr == 6 - n_pairs) {
                if (prev_m0 >= 0 && kb + 1 == min(Epi::kLoadKb1, num_kb)) {
                  epi.load(prev_m0, prev_n0, 1, es);
                  es.parity ^= 1;
                  prev_m0 = -1;
                }
                if (live && kb + 1 == min(Epi::kLoadKb0, num_kb)) {
                  epi.load(m0, n0, 0, es);
                  es.parity ^= 1;
                }
              }
            }
#endif
          }
        }
        if (live) { prev_m0 = m0; prev_n0 = n0; }
      }
#ifndef TGB_SKIP_EPI
      if constexpr (Epi::kSmemBytes > 0) {
        if (prev_m0 >= 0) epi.load(prev_m0, prev_n0, 1, es);   // the CTA's last tile
      }
#endif
    }
  } else if constexpr (Epi::kDeferred) {
    // ===== consumers, deferred epilogue: tile i's accumulators are packed right after its last MMA, and the rest of its
    // epilogue runs as steps between tile i+1's first k-blocks, so the tensor pipe always has a k-block queued =====
    setmaxnreg_consumer();
    const int cw = wg - 1;
    const int row_in_tile = 64 * cw + 16 * ((threadIdx.x >> 5) & 3) + (lane >> 2);
    float acc[TC_ACC];
#pragma unroll
    for (int i = 0; i < TC_ACC; ++i) acc[i] = 0.f;
    uint32_t dq[TC_ACC / 2];                    // the pending tile's packed values
    float racc[2] = {0.f, 0.f};                 // its row-dot, carried from step to step
    int pend_m0 = -1, pend_tn = 0;              // the pending tile (-1: none)
    uint32_t kbg = 0;
    // one k-block of the current tile: its MMAs are issued and the previous k-block's stage is released
    auto kblock = [&](int kb, long long probe_tile) {
      const int s = kbg % STAGES;
      const uint32_t ph = (kbg / STAGES) & 1;
      mbar_wait(&full_bar[s], ph);
      if (kb == 0) TGB_BWD_PROBE(probe_tile, cw, kBwdProbeFull);
      const uint32_t sa = smem_u32(smem + s * kStageBytes) + cw * 8192;
      const uint32_t sb = smem_u32(smem + s * kStageBytes) + TileA::kBytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / TC_MMA_K; ++k) {
        if (kb == 0 && k == 0) wgmma_m64n256k16_first<kTA, kTB>(acc, TileA::desc(sa, k), TileB::desc(sb, k));
        else wgmma_m64n256k16<kTA, kTB>(acc, TileA::desc(sa, k), TileB::desc(sb, k), 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (kb > 0 && lane < 2) mbar_arrive_cluster(&empty_bar[(kbg - 1) % STAGES], lane);
      ++kbg;
    };
    for (int w = cluster_index(); w < total; w += cluster_count()) {
      const int split = w / (tiles_n * tiles_mp);
      int tp_i, tile_n;
      tile_mn(w - split * tiles_n * tiles_mp, tiles_mp, tiles_n, group_m, tp_i, tile_n);
      const int m0 = (tm_off + 2 * tp_i + cluster_rank()) * TC_BM;
      const bool live = m0 < (tm_off + tiles_m) * TC_BM;
      const int k_begin = k_off + split * k_per_split;
      const int k_end = min(k_total, k_begin + k_per_split);
      const int total_kb = (k_end - k_begin + TC_BK - 1) / TC_BK * n_pairs;
      const long long probe_tile = live ? epi.tile_id(m0, tile_n) : -1;
      (void)probe_tile;
      float c[2] = {0.f, 0.f};
      if (live) epi.centres(m0 + row_in_tile, c);
      acc_fence(acc);
      // a phantom tile runs its MMAs on a stale A: the stages are released on the same schedule in both CTAs.  Its
      // k-blocks still carry the previous tile's steps; a tile with fewer k-blocks than steps runs the rest after them.
      // Every tile has a first k-block (k_total >= 1), whose first MMA overwrites the accumulators: they are dead from
      // the pack to there, which leaves the registers for the packed values.
      constexpr int kPrefix = Epi::step_kb(Epi::kSteps - 1) + 1;
#pragma unroll
      for (int p = 0; p < kPrefix; ++p) {
        if (p == 0 || p < total_kb) kblock(p, probe_tile);
#pragma unroll
        for (int s = 0; s < Epi::kSteps; ++s)
          if (Epi::step_kb(s) == p && pend_m0 >= 0) epi.step(s, dq, racc, pend_m0, pend_tn, pend_m0 + row_in_tile, lane, cw, es);
      }
      for (int kb = kPrefix; kb < total_kb; ++kb) kblock(kb, probe_tile);
      wgmma_wait<0>();
      acc_fence(acc);
      if (live) TGB_BWD_PROBE(probe_tile, cw, kBwdProbeRetired);
      if (total_kb > 0 && lane < 2) mbar_arrive_cluster(&empty_bar[(kbg - 1) % STAGES], lane);
#ifndef TGB_SKIP_EPI
      Epi::pack(acc, c, dq);                    // also for a phantom tile: a conditional pack would keep the old values live
      pend_m0 = live ? m0 : -1;
      pend_tn = tile_n;
#endif
    }
    if (pend_m0 >= 0) {                         // the CTA's last tile
#pragma unroll
      for (int s = 0; s < Epi::kSteps; ++s) epi.step(s, dq, racc, pend_m0, pend_tn, pend_m0 + row_in_tile, lane, cw, es);
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
    for (int w = cluster_index(); w < total; w += cluster_count()) {
      TileCoord t;
      t.split = w / (tiles_n * tiles_mp);
      int tp_i;
      tile_mn(w - t.split * tiles_n * tiles_mp, tiles_mp, tiles_n, group_m, tp_i, t.tile_n);
      t.tiles_n = tiles_n;
      t.n0 = t.tile_n * TC_BN;
      t.m0 = (tm_off + 2 * tp_i + cluster_rank()) * TC_BM;
      const bool live = t.m0 < (tm_off + tiles_m) * TC_BM;
      const int k_begin = k_off + t.split * k_per_split;
      const int k_end = min(k_total, k_begin + k_per_split);
      const int total_kb = (k_end - k_begin + TC_BK - 1) / TC_BK * n_pairs;
#ifndef TGB_SKIP_EPI
      if (live) epi.prologue(t, ct);
#endif
      acc_fence(acc);
      // a phantom tile runs its MMAs on a stale A: the stages are released on the same schedule in both CTAs
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
        if (kb > 0 && lane < 2) mbar_arrive_cluster(&empty_bar[(kbg - 1) % STAGES], lane);
      }
      wgmma_wait<0>();
      acc_fence(acc);
      if (total_kb > 0 && lane < 2) mbar_arrive_cluster(&empty_bar[(kbg - 1) % STAGES], lane);
#ifndef TGB_SKIP_EPI
      if (t.m0 < (tm_off + tiles_m) * TC_BM) {   // live, recomputed: the accumulators leave no register to keep it in
        epi.run(acc, t, t.m0 + row_in_tile, lane, cw, es);
        es.parity ^= 1;
      }
#endif
    }
  }
  cluster_sync();                               // no CTA leaves while its peer may still arrive on its barriers
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
  int clusters[16] = {};          // ... and how many of their 2-CTA clusters fit on the device at once
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

// Launches k_gemm_tc as a persistent grid of 2-CTA clusters over `pairs` work items (pairs of row tiles x column tiles x
// splits): at most as many clusters as can be resident at once, which on H100 may leave some SMs idle (the GPCs do not
// all hold an even number of SMs that a cluster can use).  `keep_sms` SMs (rounded up to whole clusters, at least one
// cluster stays) are left to other work: the streaming update that runs beside a contraction of the bf16 chunk pipeline.
// Which CTA computes a tile never changes a tile's arithmetic, so the result is the same bits at every grid size.
// cudaFuncSetAttribute and the occupancy query are driver calls: they run once per (handle, kernel), not on every launch.
template <class Kern, class... Args>
static inline int tc_launch(TcContext& tc, Kern kern, int smem, long long pairs, int keep_sms, cudaStream_t s, const char* name,
                            char* err, size_t n, Args... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(TC_THREADS);
  cfg.dynamicSmemBytes = (size_t)smem;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const void* key = reinterpret_cast<const void*>(kern);
  int slot = -1;
  for (int i = 0; i < 16; ++i) {
    if (tc.smem_fn[i] == key) { slot = i; break; }
    if (tc.smem_fn[i] == nullptr && slot < 0) slot = i;
  }
  if (slot < 0) { snprintf(err, n, "launch %s: more than 16 tensor-core kernels", name); return -2; }
  if (tc.smem_fn[slot] != key || tc.smem_bytes[slot] != smem) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) { snprintf(err, n, "cudaFuncSetAttribute(smem=%d): %s", smem, cudaGetErrorString(e)); return -2; }
    cfg.gridDim = dim3(2);
    int c = 0;
    e = cudaOccupancyMaxActiveClusters(&c, kern, &cfg);
    if (e != cudaSuccess || c < 1) {
      snprintf(err, n, "launch %s: no 2-CTA cluster with %d B of shared memory fits (%s)", name, smem, cudaGetErrorString(e));
      return -2;
    }
    tc.smem_fn[slot] = key; tc.smem_bytes[slot] = smem; tc.clusters[slot] = c;
  }
  const int clusters = std::max(1, tc.clusters[slot] - (keep_sms + 1) / 2);
  cfg.gridDim = dim3((unsigned)(2 * (pairs < clusters ? pairs : clusters)));
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, args...);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) { snprintf(err, n, "launch %s: %s", name, cudaGetErrorString(e)); return -2; }
  return 0;
}

// Operand ring of up to 4 stages of 48 KB (128 x 64 A + 256 x 64 B, bf16), as many as fit beside the epilogue's buffer
// in the 227 KB an H100 block may use (1 KB of it kept for the alignment of the dynamic buffer, 1 KB for the static
// barriers): 4 stages (193 KB), also beside TcEpiDpStore's 32 KB (225 KB).
constexpr int TC_STAGE_BYTES = (TC_BM + TC_BN) * TC_BK * 2;
constexpr int TC_SMEM_LIMIT = 227 * 1024;
template <class Epi>
constexpr int tc_stages() {
  const int fit = (TC_SMEM_LIMIT - 2048 - Epi::kSmemBytes) / TC_STAGE_BYTES;
  return fit < 4 ? fit : 4;
}
template <class Epi>
constexpr int tc_smem() { return tc_stages<Epi>() * TC_STAGE_BYTES + Epi::kSmemBytes + 1024; }
constexpr int TC_SMEM = tc_smem<TcEpiStore>();     // the forward
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
// work items of one launch: pairs of row tiles x column tiles x splits
static inline long long tc_pairs(int tiles_m, int tiles_n, int splits) { return (long long)(tiles_m + 1) / 2 * tiles_n * splits; }

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
  CUtensorMap pt, dq;     // bf16 store-only backward: its epilogue's Pt input and dq output
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
  auto kern = k_gemm_tc<false, false, tc_stages<TcEpiStore>(), TcEpiStore>;
  TcEpiStore epi{out, Ke, (size_t)V * Ke, V, 0};
  const int tm = (int)ceil_div(V, TC_BM), tn = (int)ceil_div(Ke, TC_BN);
  return tc_launch(tc, kern, TC_SMEM, tc_pairs(tm, tn, splits), 0, s, "tc_gemm_fwd", err, n, pl.a, pl.b, n_pairs, N, tc_kps(N, splits),
                   tm, tn, splits, 1, kPolicyEvictNormal, kPolicyEvictNormal, 0, 0, epi);
}
// cells [row0, row1) only (row0 a multiple of 64): `out` = or += this chunk's partial sum -- the host pipelines cell chunks
// behind the streaming Adam kernel (and the projection adds its 512-cell chains); the chunks run one after the other
// on one stream, so the summation order is fixed
static inline int tc_forward_launch_rows(TcContext& tc, const TcPlan& pl, int n_pairs, float* out, int accumulate, int row0, int row1,
                                         int V, int Ke, int keep_sms, cudaStream_t s, char* err, size_t n) {
  auto kern = k_gemm_tc<false, false, tc_stages<TcEpiStore>(), TcEpiStore>;
  TcEpiStore epi{out, Ke, (size_t)V * Ke, V, accumulate};
  const int tm = (int)ceil_div(V, TC_BM), tn = (int)ceil_div(Ke, TC_BN);
  return tc_launch(tc, kern, TC_SMEM, tc_pairs(tm, tn, 1), keep_sms, s, "tc_gemm_fwd", err, n, pl.a, pl.b, n_pairs, row1,
                   (int)round_up(row1 - row0, TC_BK), tm, tn, 1, 1, kPolicyEvictNormal, kPolicyEvictNormal, 0, row0, epi);
}

// Staged backward: dq = bf16(S_ext dY_ext^T - centre) (bf16 mode) or dP in fp32 (bf16x3 mode, three operand planes, six
// partial products) to HBM + row-dot partials; the update itself is a streaming kernel (adam_rows.cuh).  Rows [row0, row1)
// only (row0 a multiple of 128): the host pipelines row chunks.
static inline int tc_dpstore_plan(TcContext& tc, TcPlan& pl, const __nv_bfloat16* Sxb, size_t s_plane, const __nv_bfloat16* dYb,
                                  size_t dy_plane, int planes, int N, int V, int Ke, char* err, size_t n) {
  if (tc_make_maps(tc, &pl.a, Sxb, s_plane, planes, Ke, N, Ke, 64, TC_BM, err, n)) return -2;
  if (tc_make_maps(tc, &pl.b, dYb, dy_plane, planes, Ke, V, Ke, 64, TC_BN / 2, err, n)) return -2;   // one half of a B tile
  pl.ready = true;
  return 0;
}
// TcEpiDpStore's Pt and dq, both [N][ld] bf16, in 64 x 64 boxes
static inline int tc_dpstore_epi_plan(TcContext& tc, TcPlan& pl, const __nv_bfloat16* Pt, const __nv_bfloat16* dq, int N, int ld,
                                      char* err, size_t n) {
  if (tc_make_map(tc, &pl.pt, Pt, ld, N, ld, 64, 64, err, n)) return -2;
  return tc_make_map(tc, &pl.dq, dq, ld, N, ld, 64, 64, err, n);
}
template <class Epi>
static inline int tc_dpstore_launch(TcContext& tc, const TcPlan& pl, int n_pairs, const Epi& epi, int row0, int row1, int V, int Ke,
                                    int keep_sms, cudaStream_t s, char* err, size_t n) {
  const int tn = (int)ceil_div(V, TC_BN);
  auto kern = k_gemm_tc<true, true, tc_stages<Epi>(), Epi>;
  constexpr int smem = tc_smem<Epi>();
  const int tm0 = row0 / TC_BM, tm = (int)ceil_div(row1, TC_BM) - tm0;
  return tc_launch(tc, kern, smem, tc_pairs(tm, tn, 1), keep_sms, s, "tc_gemm_bwd_dp", err, n, pl.a, pl.b, n_pairs, Ke, Ke, tm, tn, 1, 1,
                   kPolicyEvictNormal, kPolicyEvictLast, tm0, 0, epi);
}

}  // namespace tgb
