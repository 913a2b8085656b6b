// Streaming half of the staged backward (bf16 throughput mode): softmax-Jacobian + Adam + next iteration's P over
// M, m, v (fp32) and the bf16 dq = dP - centre written by the store-only backward contraction (TcEpiDpStore).
//
//   g_ij   = P_ij (dq_ij - r'_i - lam_r ((M_ij - lse_i) - h_i)) + lam_l1 sign(M_ij) + 2 lam_l2 M_ij     (SURVEY A.2)
//   m, v, M <- Adam(g)                                                (torch.optim.Adam, mapping_optimizer.py:373, :396)
//   Pt_ij  = exp(Mnew_ij - lse_i)  (bf16) and zt_i = sum_j Pt_ij      (the next forward's operand, see k_row_norm)
//
// Pure HBM streaming: 12 B/element in (M 4, m 2, v 4, dq 2), 12 B/element out (M 4, m 2, v 4, Pt 2).  One warp owns a row, so the row sums
// need no partial arrays and are deterministic; every lane moves full 32-byte sectors (two 16-byte accesses), 8 columns
// per lane and iteration, two iterations in flight.
#pragma once
#include "common.cuh"
#include "gemm_tc.cuh"

namespace tgb {

struct AdamRowsArgs {
  float* M; __nv_bfloat16* m; float* v;  // [rows][ld]; the first moment is stored in bf16 (2 + 2 B/element instead of 4 + 4)
  const __nv_bfloat16* dq;               // [rows][ld]
  __nv_bfloat16* Pt;                     // [rows][ld]
  const RowConst* rowc;                  // (lse, r', h) per row
  float* zsum; float* pxsum; float* l1sum; float* l2sum;   // per row; px/l1/l2 may be null
  int ld, V, row0, row1;
  float lam_r, lam_l1, lam_l2;
  AdamScalars a;
};

// 8 floats = one 32-byte sector as two 16-byte streaming (evict-first) accesses
__device__ __forceinline__ void ldg256f(const float* src, float (&x)[8]) {
  asm volatile("ld.global.cs.v4.f32 {%0,%1,%2,%3}, [%8];\n\t"
               "ld.global.cs.v4.f32 {%4,%5,%6,%7}, [%8+16];"
               : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3]), "=f"(x[4]), "=f"(x[5]), "=f"(x[6]), "=f"(x[7]) : "l"(src));
}
__device__ __forceinline__ void stg256f(float* dst, const float (&x)[8]) {
  asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};\n\t"
               "st.global.cs.v4.f32 [%0+16], {%5,%6,%7,%8};"
               ::"l"(dst), "f"(x[0]), "f"(x[1]), "f"(x[2]), "f"(x[3]), "f"(x[4]), "f"(x[5]), "f"(x[6]), "f"(x[7]) : "memory");
}
__device__ __forceinline__ uint4 ldg128_stream(const void* src) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(src));
  return r;
}

struct AdamRowsLoad { float x[8], m[8], v[8]; uint4 d, mq; };

__device__ __forceinline__ void unpack_bf8(const uint4& q, float (&f)[8]) {
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const __nv_bfloat162 b = *reinterpret_cast<const __nv_bfloat162*>(&w[e]);
    f[2 * e] = __low2float(b); f[2 * e + 1] = __high2float(b);
  }
}
__device__ __forceinline__ uint4 pack_bf8(const float (&f)[8]) {
  uint4 o;
  __nv_bfloat162 b;
  b = __floats2bfloat162_rn(f[0], f[1]); o.x = *reinterpret_cast<uint32_t*>(&b);
  b = __floats2bfloat162_rn(f[2], f[3]); o.y = *reinterpret_cast<uint32_t*>(&b);
  b = __floats2bfloat162_rn(f[4], f[5]); o.z = *reinterpret_cast<uint32_t*>(&b);
  b = __floats2bfloat162_rn(f[6], f[7]); o.w = *reinterpret_cast<uint32_t*>(&b);
  return o;
}

// PLAIN: default loss (no entropy / L1 / L2) -> no per-element branches, 4 MUFU per element.
#ifndef TGB_ADAM_MAXNREG
#define TGB_ADAM_MAXNREG 96     // two 8-column groups of M, m, v, dq in flight per lane without spills; 2 CTAs of 256 threads per SM
#endif
template <bool PLAIN>
__device__ __forceinline__ void adam_row(const AdamRowsArgs& p, int row, int lane) {
  const RowConst rc = p.rowc[row];
  const float lse_l2e = rc.lse * 1.4426950408889634f;
  const size_t base = (size_t)row * p.ld;
  float* Mr = p.M + base; __nv_bfloat16* mr = p.m + base; float* vr = p.v + base;
  const __nv_bfloat16* dr = p.dq + base;
  __nv_bfloat16* pr = p.Pt + base;

  const float k_nstep = -p.a.step_size;

  float zs = 0.f, pxs = 0.f, l1s = 0.f, l2s = 0.f;

  auto load = [&](int c, AdamRowsLoad& L) {
    ldg256f(Mr + c, L.x); L.mq = ldg128_stream(mr + c); ldg256f(vr + c, L.v);
    L.d = ldg128_stream(dr + c);
  };
  auto one = [&](float& x, float dq, float& m, float& v) -> float {     // general path, one element; returns Pt
    const float pcur = fast_ex2(fmaf(x, 1.4426950408889634f, -lse_l2e));
    float g = dq - rc.r;
    if (p.lam_r != 0.f) g -= p.lam_r * ((x - rc.lse) - rc.h);
    g *= pcur;
    if (p.lam_l1 != 0.f) g += p.lam_l1 * (float)((x > 0.f) - (x < 0.f));
    if (p.lam_l2 != 0.f) g += 2.f * p.lam_l2 * x;
    m = fmaf(g - m, p.a.one_minus_beta1, m);
    v = fmaf(p.a.one_minus_beta2 * g, g, v * p.a.beta2);
    const float denom = fmaf(fast_sqrt(v), p.a.inv_bc2_sqrt, p.a.eps);
    x = fmaf(-p.a.step_size * m, fast_rcp(denom), x);
    const float pt = fast_ex2(fmaf(x, 1.4426950408889634f, -lse_l2e));
    zs += pt;
    if (p.pxsum) pxs = fmaf(pt, x, pxs);
    if (p.l1sum) { l1s += fabsf(x); l2s = fmaf(x, x, l2s); }
    return pt;
  };
  auto process = [&](int c, AdamRowsLoad& L) {
    const uint32_t dw[4] = {L.d.x, L.d.y, L.d.z, L.d.w};
    unpack_bf8(L.mq, L.m);
    float pt[8];
    if (c + 8 <= p.V) {
      if (PLAIN) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const __nv_bfloat162 d2 = *reinterpret_cast<const __nv_bfloat162*>(&dw[e >> 1]);
          const float dq = (e & 1) ? __high2float(d2) : __low2float(d2);
          float& x = L.x[e];
          float& m = L.m[e];
          float& v = L.v[e];
          const float g = (dq + -rc.r) * fast_ex2(fmaf(x, 1.4426950408889634f, -lse_l2e));
          m = fmaf(g + -m, p.a.one_minus_beta1, m);                          // m + (g - m)(1-b1)
          v = fmaf(p.a.one_minus_beta2 * g, g, v * p.a.beta2);
          const float den = fmaf(fast_sqrt(v), p.a.inv_bc2_sqrt, p.a.eps);
          x = fmaf(k_nstep * m, fast_rcp(den), x);
          pt[e] = fast_ex2(fmaf(x, 1.4426950408889634f, -lse_l2e));
        }
        zs += ((pt[0] + pt[1]) + (pt[2] + pt[3])) + ((pt[4] + pt[5]) + (pt[6] + pt[7]));
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const __nv_bfloat162 d2 = *reinterpret_cast<const __nv_bfloat162*>(&dw[e]);
          pt[2 * e] = one(L.x[2 * e], __low2float(d2), L.m[2 * e], L.v[2 * e]);
          pt[2 * e + 1] = one(L.x[2 * e + 1], __high2float(d2), L.m[2 * e + 1], L.v[2 * e + 1]);
        }
      }
      stg256f(Mr + c, L.x); *reinterpret_cast<uint4*>(mr + c) = pack_bf8(L.m); stg256f(vr + c, L.v);
    } else if (c < p.V) {                   // the ragged group: columns >= V are padding (state stays zero, Pt = 0)
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const __nv_bfloat162 d2 = *reinterpret_cast<const __nv_bfloat162*>(&dw[e >> 1]);
        const float dq = (e & 1) ? __high2float(d2) : __low2float(d2);
        pt[e] = (c + e < p.V) ? one(L.x[e], dq, L.m[e], L.v[e]) : 0.f;
      }
      stg256f(Mr + c, L.x); *reinterpret_cast<uint4*>(mr + c) = pack_bf8(L.m); stg256f(vr + c, L.v);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) pt[e] = 0.f;
    }
    *reinterpret_cast<uint4*>(pr + c) = pack_bf8(pt);
  };

  // ld is a multiple of 64: every 8-column group of the row is inside the allocation
  int c = lane * 8;
  for (; c + 256 < p.ld; c += 512) {
    AdamRowsLoad A, B;
    load(c, A);
    load(c + 256, B);
    process(c, A);
    process(c + 256, B);
  }
  if (c < p.ld) {
    AdamRowsLoad A;
    load(c, A);
    process(c, A);
  }
  zs = warp_sum(zs);
  if (p.pxsum) pxs = warp_sum(pxs);
  if (p.l1sum) { l1s = warp_sum(l1s); l2s = warp_sum(l2s); }
  if (lane == 0) {
    p.zsum[row] = zs;
    if (p.pxsum) p.pxsum[row] = pxs;
    if (p.l1sum) { p.l1sum[row] = l1s; p.l2sum[row] = l2s; }
  }
}
template <bool PLAIN>
__global__ void __maxnreg__(TGB_ADAM_MAXNREG)
k_adam_rows(const AdamRowsArgs p) {
  const int row = p.row0 + blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row < p.row1) adam_row<PLAIN>(p, row, threadIdx.x & 31);
}
#ifdef TGB_OVERLAP_PROBE
// Debug build only (tools/overlap_probe.py): the same rows, warps and arithmetic as a persistent grid of 512-thread CTAs.
// Two of them (2 x 512 x 96 registers) do not fit one SM, so a grid of U CTAs runs on U distinct SMs.
template <bool PLAIN>
__global__ void __maxnreg__(TGB_ADAM_MAXNREG)
k_adam_rows_probe(const AdamRowsArgs p) {
  const int warps = blockDim.x >> 5;
  for (int row = p.row0 + blockIdx.x * warps + (threadIdx.x >> 5); row < p.row1; row += gridDim.x * warps)
    adam_row<PLAIN>(p, row, threadIdx.x & 31);
}
#endif

// ---- parity mode (bf16x3): the same streaming pass in the reference's arithmetic ---------------------------------------------
// IEEE expf / div / sqrt, torch's single-tensor Adam op order (adam_update), P from the row-pass statistics (softmax_prob) --
// element for element what the fp32 mode's fused epilogue (EpiAdam) computes, here fed by the fp32 dP the store-only
// contraction left in HBM.  16 B/element in (M, m, v, dP), 12 B/element out.
struct AdamRowsExactArgs {
  float* M; float* m; float* v;          // [rows][ld]
  const float* dp;                       // [rows][ld]
  const RowStat* stats; const float* rdot;
  int ld, V, row0, row1;
  float lam_r, lam_l1, lam_l2;
  AdamScalars a;
};

__global__ void __launch_bounds__(256)
k_adam_rows_exact(const AdamRowsExactArgs p) {
  const int lane = threadIdx.x & 31;
  const int row = p.row0 + blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= p.row1) return;
  const RowStat st = p.stats[row];
  const float r = p.rdot[row];
  const size_t base = (size_t)row * p.ld;
  float* Mr = p.M + base; float* mr = p.m + base; float* vr = p.v + base;
  const float* dr = p.dp + base;
  for (int c = lane * 8; c < p.V; c += 256) {        // groups entirely in the padding are never touched
    float x[8], m[8], v[8], d[8];
    ldg256f(Mr + c, x); ldg256f(mr + c, m); ldg256f(vr + c, v); ldg256f(dr + c, d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      if (c + e < p.V) {
        const float pr = softmax_prob(x[e], st);
        float g = d[e] - r;
        if (p.lam_r != 0.f) g -= p.lam_r * (((x[e] - st.mx) - st.log_z) - st.h);
        g *= pr;
        if (p.lam_l1 != 0.f) g += p.lam_l1 * (float)((x[e] > 0.f) - (x[e] < 0.f));
        if (p.lam_l2 != 0.f) g += 2.f * p.lam_l2 * x[e];
        x[e] = adam_update(x[e], g, m[e], v[e], p.a);
      }
    }
    stg256f(Mr + c, x); stg256f(mr + c, m); stg256f(vr + c, v);
  }
}

static inline int adam_rows_exact_launch(const AdamRowsExactArgs& a, cudaStream_t s) {
  const int rows = a.row1 - a.row0;
  if (rows <= 0) return 0;
  k_adam_rows_exact<<<(unsigned)ceil_div(rows, 8), 256, 0, s>>>(a);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

static inline int adam_rows_launch(const AdamRowsArgs& a, cudaStream_t s) {
  const int rows = a.row1 - a.row0;
  if (rows <= 0) return 0;
  const unsigned grid = (unsigned)ceil_div(rows, 8);
  const bool plain = a.lam_r == 0.f && a.lam_l1 == 0.f && a.lam_l2 == 0.f;
  if (plain) k_adam_rows<true><<<grid, 256, 0, s>>>(a);
  else k_adam_rows<false><<<grid, 256, 0, s>>>(a);
  return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

}  // namespace tgb
