// Bandwidth-bound kernels of the hot path: row softmax + statistics, loss reductions,
// loss scalars, dY assembly.  Coalesced float4 HBM loads + warp-shuffle reductions.
// Reference: tangram/mapping_optimizer.py:189-309 (_loss_fn).
#pragma once
#include "common.cuh"
#include "gemm_simt.cuh"       // adam_update (k_filter_update)
#include <curand_kernel.h>

namespace tgb {

// ------------------------------------------------------------------------------------
// Row pass: P = softmax(M, dim=1) (:201) + per-row statistics.
// One CTA per cell row; the row lives in registers (ITEMS float4 per thread) when it fits,
// otherwise it is re-read (L2-resident).  Also emits sum_j P log P (entropy, :224),
// sum|M| and sum M^2 (:228-231) when those terms are enabled.
// Pad columns [V, ldp) of P are written as zero so the GEMMs can read whole vectors.
// ------------------------------------------------------------------------------------
template <typename PT>
__device__ __forceinline__ void store_p4(PT* dst, float a, float b, float c, float d);
template <>
__device__ __forceinline__ void store_p4<float>(float* dst, float a, float b, float c, float d) {
  st_stream(reinterpret_cast<float4*>(dst), make_float4(a, b, c, d));
}
template <>
__device__ __forceinline__ void store_p4<__nv_bfloat16>(__nv_bfloat16* dst, float a, float b, float c, float d) {
  __nv_bfloat162 lo = __floats2bfloat162_rn(a, b), hi = __floats2bfloat162_rn(c, d);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&lo);
  u.y = *reinterpret_cast<uint32_t*>(&hi);
  *reinterpret_cast<uint2*>(dst) = u;
}

// Three bf16 planes hi + mid + lo of an fp32 value (parity mode on tensor cores): x - (hi + mid + lo) ~ 2^-24 |x|.
struct Split3 { __nv_bfloat16* base; size_t plane; };
__device__ __forceinline__ void split3(float x, __nv_bfloat16& h, __nv_bfloat16& m, __nv_bfloat16& l) {
  h = __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(h);
  m = __float2bfloat16_rn(r1);
  l = __float2bfloat16_rn(r1 - __bfloat162float(m));
}
__device__ __forceinline__ uint32_t pack_bf2(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
__device__ __forceinline__ void store_split4(const Split3& d, size_t off, float a, float b, float c, float e) {
  __nv_bfloat16 h[4], m[4], l[4];
  split3(a, h[0], m[0], l[0]); split3(b, h[1], m[1], l[1]); split3(c, h[2], m[2], l[2]); split3(e, h[3], m[3], l[3]);
  *reinterpret_cast<uint2*>(d.base + off) = make_uint2(pack_bf2(h[0], h[1]), pack_bf2(h[2], h[3]));
  *reinterpret_cast<uint2*>(d.base + d.plane + off) = make_uint2(pack_bf2(m[0], m[1]), pack_bf2(m[2], m[3]));
  *reinterpret_cast<uint2*>(d.base + 2 * d.plane + off) = make_uint2(pack_bf2(l[0], l[1]), pack_bf2(l[2], l[3]));
}
// src (fp32, n elements, n % 4 == 0) -> three bf16 planes
__global__ void k_split3(const float* __restrict__ src, Split3 dst, long long n4) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n4) return;
  const float4 v = reinterpret_cast<const float4*>(src)[q];
  store_split4(dst, (size_t)q * 4, v.x, v.y, v.z, v.w);
}

template <typename PT, int THREADS, int ITEMS, int MINB = 1>
__global__ void __launch_bounds__(THREADS, MINB)
k_softmax_rows(const float* __restrict__ M, int ldm, int V, PT* __restrict__ P, int ldp,
               RowStat* __restrict__ stats, float* __restrict__ rowaux /* [N][2] or null */,
               int want_entropy, Split3 split /* base == null: none */) {
  __shared__ float sh[32];
  const int row = blockIdx.x;
  const float* mrow = M + (size_t)row * ldm;
  const int nvec = ldp >> 2;  // float4 slots incl. pad (ldm == ldp)
  constexpr bool kCached = ITEMS > 0;
  constexpr int NI = kCached ? ITEMS : 1;
  float4 x[NI];

  float mx = -INFINITY, s1 = 0.f, s2 = 0.f;
  const bool aux = rowaux != nullptr;
  auto visit_max = [&](const float4& v, int c) {
    if (c + 3 < V) {                          // interior group: no per-element bounds checks
      mx = fmaxf(fmaxf(mx, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
      if (aux) {
        s1 += (fabsf(v.x) + fabsf(v.y)) + (fabsf(v.z) + fabsf(v.w));
        s2 += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
      }
    } else {
      if (c + 0 < V) { mx = fmaxf(mx, v.x); s1 += fabsf(v.x); s2 += v.x * v.x; }
      if (c + 1 < V) { mx = fmaxf(mx, v.y); s1 += fabsf(v.y); s2 += v.y * v.y; }
      if (c + 2 < V) { mx = fmaxf(mx, v.z); s1 += fabsf(v.z); s2 += v.z * v.z; }
      if (c + 3 < V) { mx = fmaxf(mx, v.w); s1 += fabsf(v.w); s2 += v.w * v.w; }
    }
  };
  if (kCached) {
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int q = threadIdx.x + i * THREADS;
      x[i] = (q < nvec) ? ld_stream(reinterpret_cast<const float4*>(mrow) + q) : make_float4(0, 0, 0, 0);
      if (q < nvec) visit_max(x[i], q * 4);
    }
  } else {
    for (int q = threadIdx.x; q < nvec; q += THREADS)
      visit_max(reinterpret_cast<const float4*>(mrow)[q], q * 4);
  }
  mx = block_reduce<true>(mx, sh);

  // e_j = exp(M_ij - max): computed ONCE per element.  Without the entropy term the cached row is overwritten by e (padding
  // = 0), so the emit pass below is a multiply; with it the pass needs M_ij - max again and recomputes (same bits either way:
  // P_ij = expf(M_ij - max) * (1 / Z) is softmax_prob()).
  float z = 0.f;
  auto exp4 = [&](const float4& v, int c) -> float4 {
    float4 e;
    if (c + 3 < V) {
      e = make_float4(expf(v.x - mx), expf(v.y - mx), expf(v.z - mx), expf(v.w - mx));
    } else {
      e.x = (c + 0 < V) ? expf(v.x - mx) : 0.f;
      e.y = (c + 1 < V) ? expf(v.y - mx) : 0.f;
      e.z = (c + 2 < V) ? expf(v.z - mx) : 0.f;
      e.w = (c + 3 < V) ? expf(v.w - mx) : 0.f;
    }
    return e;
  };
  const bool keep_e = kCached && !want_entropy;
  if (kCached) {
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int q = threadIdx.x + i * THREADS;
      if (q < nvec) {
        const float4 e = exp4(x[i], q * 4);
        z += (e.x + e.y) + (e.z + e.w);
        if (keep_e) x[i] = e;
      }
    }
  } else {
    for (int q = threadIdx.x; q < nvec; q += THREADS) {
      const float4 e = exp4(reinterpret_cast<const float4*>(mrow)[q], q * 4);
      z += (e.x + e.y) + (e.z + e.w);
    }
  }
  z = block_reduce<false>(z, sh);

  RowStat st;
  st.mx = mx;
  st.inv_z = 1.0f / z;
  st.log_z = logf(z);
  st.h = 0.f;

  float h = 0.f;
  PT* prow = P + (size_t)row * ldp;
  auto emit = [&](const float4& v, int q) {          // v = e (keep_e) or M
    const int c = q * 4;
    float p0, p1, p2, p3;
    if (keep_e) {
      p0 = v.x * st.inv_z; p1 = v.y * st.inv_z; p2 = v.z * st.inv_z; p3 = v.w * st.inv_z;
    } else {
      p0 = (c + 0 < V) ? softmax_prob(v.x, st) : 0.f;
      p1 = (c + 1 < V) ? softmax_prob(v.y, st) : 0.f;
      p2 = (c + 2 < V) ? softmax_prob(v.z, st) : 0.f;
      p3 = (c + 3 < V) ? softmax_prob(v.w, st) : 0.f;
      if (want_entropy) {
        if (c + 0 < V) h += p0 * ((v.x - mx) - st.log_z);
        if (c + 1 < V) h += p1 * ((v.y - mx) - st.log_z);
        if (c + 2 < V) h += p2 * ((v.z - mx) - st.log_z);
        if (c + 3 < V) h += p3 * ((v.w - mx) - st.log_z);
      }
    }
    if (P != nullptr) store_p4<PT>(prow + c, p0, p1, p2, p3);
    if (split.base != nullptr) store_split4(split, (size_t)row * ldp + c, p0, p1, p2, p3);
  };
  if (kCached) {
#pragma unroll
    for (int i = 0; i < NI; ++i) {
      const int q = threadIdx.x + i * THREADS;
      if (q < nvec) emit(x[i], q);
    }
  } else {
    for (int q = threadIdx.x; q < nvec; q += THREADS)
      emit(reinterpret_cast<const float4*>(mrow)[q], q);
  }
  if (want_entropy) h = block_reduce<false>(h, sh);
  if (rowaux != nullptr) {
    s1 = block_reduce<false>(s1, sh);
    s2 = block_reduce<false>(s2, sh);
  }
  if (threadIdx.x == 0) {
    st.h = h;
    stats[row] = st;
    if (rowaux != nullptr) { rowaux[2 * row] = s1; rowaux[2 * row + 1] = s2; }
  }
}

// Sum of per-row scalars (entropy, L1, L2) over this rank's rows -> 8-float tail of the
// exchange buffer.  Deterministic (fixed tree), one CTA.
// tail (8 floats): [0] sum_i h_i, [1] sum|M|, [2] sum M^2, [3] sum_i f_i, [4] sum_i (f_i - f_i^2)  (f: constrained mode),
// [5] sum_i h_i again when `val` (a sharded handle's validation entropy, read by k_loss_scalars<true>), else 0; [6], [7] 0.
// stats / rowaux / f may be null: their slots are then 0
constexpr int kTail = 8;
constexpr int kTailValEntropy = 5;
__global__ void __launch_bounds__(1024)
k_row_scalar_reduce(const RowStat* __restrict__ stats, const float* __restrict__ rowaux, const float* __restrict__ f,
                    int n_rows, int val, float* __restrict__ tail) {
  __shared__ float sh[32];
  float h = 0.f, a = 0.f, b = 0.f, fs = 0.f, fr = 0.f;
  for (int i = threadIdx.x; i < n_rows; i += blockDim.x) {
    if (stats) h += stats[i].h;
    if (rowaux) { a += rowaux[2 * i]; b += rowaux[2 * i + 1]; }
    if (f) { const float x = f[i]; fs += x; fr += x - x * x; }
  }
  h = block_reduce<false>(h, sh);
  a = block_reduce<false>(a, sh);
  b = block_reduce<false>(b, sh);
  fs = block_reduce<false>(fs, sh);
  fr = block_reduce<false>(fr, sh);
  if (threadIdx.x == 0) {
    tail[0] = h; tail[1] = a; tail[2] = b; tail[3] = fs; tail[4] = fr; tail[5] = val ? h : 0.f; tail[6] = 0.f; tail[7] = 0.f;
  }
}

// ---- constrained mode (MapperConstrained, mapping_optimizer.py:411-639): per-cell filter f = sigmoid(F) ----------
// S_f = f o S_ext is the operand of all three contractions (:519, :521); its "ones" column becomes f, so the
// filtered column sums (:513) come out of the forward GEMM like the plain ones do.
__global__ void k_filter_prepare(const float* __restrict__ F, const float* __restrict__ Sx, int n_rows, int Ke,
                                 float* __restrict__ f, float* __restrict__ Sf) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one float4 of S_ext each
  const int nvec = Ke >> 2;
  if (q >= (long long)n_rows * nvec) return;
  const int r = (int)(q / nvec);
  const float fi = 1.f / (1.f + expf(-F[r]));
  if ((int)(q % nvec) == 0) f[r] = fi;
  float4 v = reinterpret_cast<const float4*>(Sx)[q];
  v.x *= fi; v.y *= fi; v.z *= fi; v.w *= fi;
  reinterpret_cast<float4*>(Sf)[q] = v;
}
// dL/df_i = r_i / f_i (the row-dot of the contractions: Y is linear in f_i) + density/count/regulariser parts, and
// dL/dF_i = dL/df_i f_i (1 - f_i).  Formed without the division,
//   g_i = r_i (1 - f_i) + (fscal[0] + lam_c fscal[1] + lam_f (1 - 2 f_i)) f_i (1 - f_i),
// so a saturated cell (f_i exactly 0 or 1, r_i = 0) gets g_i = 0 and keeps its F, as F.grad = grad f (1 - f) does in the
// reference (:507), instead of 0 / 0.  Every rounding is pinned (no contraction) so a test can form the same g in fp32.
// Then torch's Adam step with the same scalars as M (one optimizer over [M, F], :607).
// fscal: [0] lambda_d * sum(d) / sum(f)   [1] sign(sum(f) - target_count)
__global__ void k_filter_update(int n_rows, const float* __restrict__ rdot, const float* __restrict__ f,
                                const float* __restrict__ fscal, float lam_c, float lam_f, AdamScalars a,
                                float* __restrict__ F, float* __restrict__ mF, float* __restrict__ vF) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  const float fi = f[i];
  const float omf = __fsub_rn(1.f, fi);
  const float c = __fadd_rn(__fadd_rn(fscal[0], __fmul_rn(lam_c, fscal[1])), __fmul_rn(lam_f, __fsub_rn(1.f, __fmul_rn(2.f, fi))));
  const float g = __fadd_rn(__fmul_rn(rdot[i], omf), __fmul_rn(c, __fmul_rn(fi, omf)));
  float m = mF[i], v = vF[i];
  F[i] = adam_update(F[i], g, m, v, a);
  mF[i] = m; vF[i] = v;
}
__global__ void k_sigmoid(const float* __restrict__ F, int n, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = 1.f / (1.f + expf(-F[i]));
}

// ------------------------------------------------------------------------------------
// Loss stage.  All of it lives on V x Ke data (tiny next to N x V).
// ------------------------------------------------------------------------------------
struct Csr {
  const int* indptr;
  const int* indices;
  const float* vals;
};

constexpr int kLossCols = 128;  // gene columns per CTA (= threads)

struct LossParams {
  int V, K, Ke, T, ct_off, density_mode;
  // Training-gene mask (tgb200_set_loss_genes): act[k] = 1 for the Kact genes the loss sees, 0 for the others; null
  // when every gene is in the loss (Kact == K).  The cosine terms then run over the active genes only, as on S[:, a].
  const float* act;
  int Kact;
  long long n_cells_global;
  float lam_g1, lam_d, lam_g2, lam_r, lam_l1, lam_l2, lam_nb, lam_ct, lam_go;
  const float* G;     // V x Ke, zero beyond K
  const float* d;     // V
  float* Y;           // V x Ke (+4 tail floats): predicted expression | density cols | ct cols
  const float* ngc;   // K   max(||G_.k||, eps)
  const float* ngr;   // V   max(||G_j.||, eps)
  Csr W, WT, F, FT, A, AT;
  const float* WG;    // V x Ke   W @ G   (constant, :236 recomputes it every iteration)
  const float* nwg;   // K
  const float* AG;    // V x Ke   (A+I) @ G
  const float* nag;   // K
  const float* sgnG;  // K   sign(colsum G)
  float* Z;           // V x Ke   W @ Y
  float* Zg;          // V x Ke   (A+I) @ Y
  float* H;           // V x T    1[R > 0]
  float* colpart;     // [nchunk][3][Ke]
  float* colpart_nb;  // [nchunk][2][Ke]
  float* colpart_go;  // [nchunk][2][Ke]
  float* rowpart;     // [ncolchunk][V][2]
  float* ctpart;      // [n ct blocks]
  int n_ct_blocks;
  float* coefA; float* coefB;     // Ke
  float* coefAn; float* coefBn;   // Ke
  float* coefAg; float* coefBg;   // Ke
  float* coefAr; float* coefBr;   // V
  float* densg;                   // V
  // constrained mode
  int constrained;
  float lam_c, lam_f, target_count;
  float* fscal;                   // [2] coefficients for k_filter_update
  // history columns 12-15: 0 with validation off, NaN on the rows a validation does not fill (tgb200_set_validation)
  float hist_fill;
  // validation (_val_loss_fn, mapping_optimizer.py:311-356): k_loss_scalars<true> also writes
  // val_out[0..3] = (gv + vg, gv, sum_k cos_k w_k / sum_k w_k, -(sum_i h_i / log V) / n_cells_global), sum_i h_i from
  // tail[val_ent] (on a sharded handle kTailValEntropy, over every rank's cells once the exchange buffer is summed)
  const float* gw;                // Ke   w_k: fraction of voxels where G[:, k] != 0 (0 outside the mask)
  float* val_out;
  float val_log_v, val_n;         // logf(V) as the host computes it, n_cells_global
  int val_ent;                    // tail slot of sum_i h_i
};

// Y = sum over split partials; per-gene <Y,G>, |Y|^2, colsum(Y) for this row chunk;
// per-voxel <Y,G>, |Y|^2 for this column chunk (only when lambda_g2 != 0).
// rows_per_block (<= kLossRowsMax) is chosen on the host so that small problems still fill the GPU
// and large ones (V = 50k) keep the partial arrays small.
constexpr int kLossRowsMax = 128;
constexpr int kLossVec = 4;                       // columns per thread (float4)
constexpr int kLossColsBlk = kLossCols * kLossVec;  // columns per CTA
// kMasked: the row statistics skip the genes outside p.act.  A template argument, not a test of p.act: the unmasked
// instantiation keeps its contracted multiply-adds, so its results do not depend on whether this kernel can mask.
template <bool kMasked>
__global__ void __launch_bounds__(kLossCols)
k_loss_reduce(LossParams p, const float* __restrict__ part, int nsplit, int row_stats, int rows_per_block) {
  __shared__ float shr[4][kLossRowsMax][2];
  const int k = blockIdx.x * kLossColsBlk + threadIdx.x * kLossVec;   // Ke is a multiple of 64: whole float4s
  const int j0 = blockIdx.y * rows_per_block;
  const size_t plane = (size_t)p.V * p.Ke;
  const bool in = k < p.Ke;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const bool writeY = nsplit > 1 || part != p.Y;
  float dot[4] = {0.f, 0.f, 0.f, 0.f}, ny2[4] = {0.f, 0.f, 0.f, 0.f}, ys[4] = {0.f, 0.f, 0.f, 0.f};
  const int nrows = min(rows_per_block, p.V - j0);
  for (int r = 0; r < nrows; ++r) {
    const int j = j0 + r;
    float a = 0.f, b = 0.f;
    if (in) {
      const size_t o = (size_t)j * p.Ke + k;
      float4 y = *reinterpret_cast<const float4*>(part + o);
      for (int z = 1; z < nsplit; ++z) {
        const float4 t = *reinterpret_cast<const float4*>(part + (size_t)z * plane + o);
        y.x += t.x; y.y += t.y; y.z += t.z; y.w += t.w;
      }
      if (writeY) *reinterpret_cast<float4*>(p.Y + o) = y;
      const float4 g = *reinterpret_cast<const float4*>(p.G + o);
      const float yv[4] = {y.x, y.y, y.z, y.w}, gv[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (k + e < p.K) {
          dot[e] += yv[e] * gv[e]; ny2[e] += yv[e] * yv[e]; ys[e] += yv[e];
          if (!kMasked || p.act[k + e] != 0.f) { a += yv[e] * gv[e]; b += yv[e] * yv[e]; }
        }
      }
    }
    if (row_stats) {
      a = warp_sum(a); b = warp_sum(b);
      if (lane == 0) { shr[wid][r][0] = a; shr[wid][r][1] = b; }
    }
  }
  if (in) {
    float* cp = p.colpart + (size_t)blockIdx.y * 3 * p.Ke;
    *reinterpret_cast<float4*>(cp + k) = make_float4(dot[0], dot[1], dot[2], dot[3]);
    *reinterpret_cast<float4*>(cp + p.Ke + k) = make_float4(ny2[0], ny2[1], ny2[2], ny2[3]);
    *reinterpret_cast<float4*>(cp + 2 * p.Ke + k) = make_float4(ys[0], ys[1], ys[2], ys[3]);
  }
  if (row_stats) {
    __syncthreads();
    for (int r = threadIdx.x; r < nrows; r += kLossCols) {
      float a = shr[0][r][0] + shr[1][r][0] + shr[2][r][0] + shr[3][r][0];
      float b = shr[0][r][1] + shr[1][r][1] + shr[2][r][1] + shr[3][r][1];
      float* rp = p.rowpart + ((size_t)blockIdx.x * p.V + (j0 + r)) * 2;
      rp[0] = a; rp[1] = b;
    }
  }
}

// out[c][k] = sum over row chunks of part[chunk][c][k]   (thread per gene, coalesced, deterministic order)
__global__ void k_col_finalize(const float* __restrict__ part, int nchunk, int ncomp, int Ke, float* __restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (k >= Ke) return;
  float s0 = 0.f, s1 = 0.f;
  int q = 0;
  for (; q + 2 <= nchunk; q += 2) {
    s0 += part[((size_t)q * ncomp + c) * Ke + k];
    s1 += part[((size_t)(q + 1) * ncomp + c) * Ke + k];
  }
  if (q < nchunk) s0 += part[((size_t)q * ncomp + c) * Ke + k];
  out[(size_t)c * Ke + k] = s0 + s1;
}

// Zout = Op @ Y (CSR, ~7 nnz/row) fused with the per-gene <Zout,REF>, |Zout|^2 partials.
// Replaces the dense (V x V) @ (V x K) SGEMMs at :235 and :171.
__global__ void __launch_bounds__(kLossCols)
k_spatial_colstats(int V, int K, int Ke, Csr op, const float* __restrict__ Y, const float* __restrict__ REF,
                   float* __restrict__ Zout, float* __restrict__ colpart2, int rows_per_block) {
  const int k = blockIdx.x * kLossCols + threadIdx.x;
  const int j0 = blockIdx.y * rows_per_block;
  const bool gene = k < K;
  float dot = 0.f, nz2 = 0.f;
  for (int r = 0; r < rows_per_block; ++r) {
    const int j = j0 + r;
    if (j >= V) break;
    if (gene) {
      float z = 0.f;
      for (int e = op.indptr[j]; e < op.indptr[j + 1]; ++e)
        z += op.vals[e] * Y[(size_t)op.indices[e] * Ke + k];
      const size_t o = (size_t)j * Ke + k;
      Zout[o] = z;
      dot += z * REF[o];
      nz2 += z * z;
    }
  }
  if (k < Ke) {
    float* cp = colpart2 + (size_t)blockIdx.y * 2 * Ke;
    cp[k] = dot; cp[Ke + k] = nz2;
  }
}

// Cell-type islands (:242-248): R = C - F C, hinge partial sums and H = 1[R > 0].
__global__ void __launch_bounds__(256)
k_ct_islands(LossParams p) {
  __shared__ float sh[32];
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float hinge = 0.f;
  if (idx < (long long)p.V * p.T) {
    const int j = (int)(idx / p.T), t = (int)(idx % p.T);
    const float c = p.Y[(size_t)j * p.Ke + p.ct_off + t];
    float fc = 0.f;
    for (int e = p.F.indptr[j]; e < p.F.indptr[j + 1]; ++e)
      fc += p.F.vals[e] * p.Y[(size_t)p.F.indices[e] * p.Ke + p.ct_off + t];
    const float R = c - fc;
    hinge = fmaxf(R, 0.f);
    p.H[idx] = R > 0.f ? 1.f : 0.f;
  }
  hinge = block_reduce<false>(hinge, sh);
  if (threadIdx.x == 0) p.ctpart[blockIdx.x] = hinge;
}

// One CTA: finishes every reduction, writes the history row and the dY coefficients.
// cos(x,y) = <x,y> / (max(|x|,eps) max(|y|,eps))   (torch semantics, :205-206)
// d mean_k cos / dY_jk = a_k G_jk - b_k Y_jk,  a_k = 1/(K ny ng),  b_k = cos_k/(K ny^2)
// Under a gene mask the means run over the Kact active genes and an inactive gene's coefficients are 0.
// kVal: the validation's instantiation (p.gw, p.val_out).  A template argument, not a test of p.gw: the training
// instantiation compiles without the validation's arithmetic, so its results do not depend on it.
template <bool kVal>
__global__ void __launch_bounds__(1024)
k_loss_scalars(LossParams p, int nchunk, int ncolchunk, float* __restrict__ hist_row) {
  __shared__ float sh[32];
  const int tid = threadIdx.x, nt = blockDim.x;
  const float nan = __int_as_float(0x7fc00000);
  const float Kf = (float)p.Kact;
  float gv = 0.f, nb = 0.f, go = 0.f, sw = 0.f, ws = 0.f;
  for (int k = tid; k < p.K; k += nt) {
    if (p.act != nullptr && p.act[k] == 0.f) {
      p.coefA[k] = 0.f; p.coefB[k] = 0.f;
      if (p.lam_nb > 0.f) { p.coefAn[k] = 0.f; p.coefBn[k] = 0.f; }
      if (p.lam_go > 0.f) { p.coefAg[k] = 0.f; p.coefBg[k] = 0.f; }
      continue;
    }
    float dot = 0.f, ny2 = 0.f, ys = 0.f;
    for (int c = 0; c < nchunk; ++c) {
      const float* cp = p.colpart + (size_t)c * 3 * p.Ke;
      dot += cp[k]; ny2 += cp[p.Ke + k]; ys += cp[2 * p.Ke + k];
    }
    const float ny = fmaxf(sqrtf(ny2), kCosEps), ng = p.ngc[k];
    const float cs = dot / (ny * ng);
    gv += cs;
    if constexpr (kVal) { sw += cs * p.gw[k]; ws += p.gw[k]; }
    p.coefA[k] = p.lam_g1 / (Kf * ny * ng);
    p.coefB[k] = p.lam_g1 * cs / (Kf * ny * ny);
    if (p.lam_nb > 0.f) {
      float d2 = 0.f, n2 = 0.f;
      for (int c = 0; c < nchunk; ++c) {
        const float* cp = p.colpart_nb + (size_t)c * 2 * p.Ke;
        d2 += cp[k]; n2 += cp[p.Ke + k];
      }
      const float nz = fmaxf(sqrtf(n2), kCosEps), nr = p.nwg[k];
      const float c2 = d2 / (nz * nr);
      nb += c2;
      p.coefAn[k] = p.lam_nb / (Kf * nz * nr);
      p.coefBn[k] = p.lam_nb * c2 / (Kf * nz * nz);
    }
    if (p.lam_go > 0.f) {
      // cos(G*(G), G*(Y)) with G*(X) = (A+I) X / colsum(X)  (:171): the per-gene scale
      // cancels in the cosine up to its sign, so only sign(colsum) survives.
      float d2 = 0.f, n2 = 0.f;
      for (int c = 0; c < nchunk; ++c) {
        const float* cp = p.colpart_go + (size_t)c * 2 * p.Ke;
        d2 += cp[k]; n2 += cp[p.Ke + k];
      }
      const float sgn = ((ys > 0.f) ? 1.f : -1.f) * p.sgnG[k];
      const float nz = fmaxf(sqrtf(n2), kCosEps), nr = p.nag[k];
      const float c2 = d2 / (nz * nr);
      go += sgn * c2;
      p.coefAg[k] = sgn * p.lam_go / (Kf * nz * nr);
      p.coefBg[k] = sgn * p.lam_go * c2 / (Kf * nz * nz);
    }
  }
  gv = block_reduce<false>(gv, sh) / Kf;
  nb = block_reduce<false>(nb, sh) / Kf;
  go = block_reduce<false>(go, sh) / Kf;
  if constexpr (kVal) {
    sw = block_reduce<false>(sw, sh);
    ws = block_reduce<false>(ws, sh);
  }

  float vg = 0.f;
  if (p.lam_g2 != 0.f) {
    for (int j = tid; j < p.V; j += nt) {
      float dot = 0.f, ny2 = 0.f;
      for (int c = 0; c < ncolchunk; ++c) {
        const float* rp = p.rowpart + ((size_t)c * p.V + j) * 2;
        dot += rp[0]; ny2 += rp[1];
      }
      const float ny = fmaxf(sqrtf(ny2), kCosEps), ng = p.ngr[j];
      const float cs = dot / (ny * ng);
      vg += cs;
      p.coefAr[j] = p.lam_g2 / ((float)p.V * ny * ng);
      p.coefBr[j] = p.lam_g2 * cs / ((float)p.V * ny * ny);
    }
    vg = block_reduce<false>(vg, sh) / (float)p.V;
  }

  // density KL (:212-221): KLDivLoss(sum)(log dhat, d) = sum xlogy(d,d) - d log dhat
  float kl = 0.f, dsum = 0.f;
  const float* tailp = p.Y + (size_t)p.V * p.Ke;
  const float fsum = tailp[3];                       // sum_i f_i (constrained mode)
  if (p.density_mode != 0) {
    for (int j = tid; j < p.V; j += nt) {
      const float cs = p.Y[(size_t)j * p.Ke + p.K] + p.Y[(size_t)j * p.Ke + p.K + 1];
      float dhat = (p.density_mode == 1) ? cs / (float)p.n_cells_global : cs;
      if (p.constrained) dhat = cs / fsum;           // :512-514  (f-weighted column sums / sum f)
      const float dj = p.d[j];
      kl += ((dj > 0.f) ? dj * logf(dj) : 0.f) - dj * logf(dhat);
      dsum += dj;
      p.densg[j] = -p.lam_d * dj / cs;
    }
    kl = block_reduce<false>(kl, sh);
    dsum = block_reduce<false>(dsum, sh);
  }

  float ct = 0.f;
  if (p.lam_ct > 0.f) {
    for (int b = tid; b < p.n_ct_blocks; b += nt) ct += p.ctpart[b];
    ct = block_reduce<false>(ct, sh) / ((float)p.V * (float)p.T);
  }

  if (tid == 0) {
    const float* tail = p.Y + (size_t)p.V * p.Ke;
    const float ent = -tail[0], l1 = tail[1], l2 = tail[2];
    float total = -p.lam_g1 * gv;
    if (p.lam_g2 != 0.f) total -= p.lam_g2 * vg;
    if (p.density_mode != 0) total += p.lam_d * kl;
    if (p.lam_r != 0.f) total += p.lam_r * ent;
    if (p.lam_l1 != 0.f) total += p.lam_l1 * l1;
    if (p.lam_l2 != 0.f) total += p.lam_l2 * l2;
    if (p.lam_ct > 0.f) total += p.lam_ct * ct;
    if (p.lam_nb > 0.f) total -= p.lam_nb * nb;
    if (p.lam_go > 0.f) total -= p.lam_go * go;
    float count_abs = 0.f, freg = 0.f;
    if (p.constrained) {                               // :528-532, :575
      const float cnt = fsum - p.target_count;
      count_abs = fabsf(cnt);
      freg = tail[4];
      total += p.lam_c * count_abs + p.lam_f * freg;
      p.fscal[0] = (p.density_mode != 0) ? p.lam_d * dsum / fsum : 0.f;
      p.fscal[1] = (float)((cnt > 0.f) - (cnt < 0.f));
    }
    hist_row[0] = total;
    hist_row[1] = gv;
    hist_row[2] = (p.lam_g2 != 0.f) ? vg : nan;
    hist_row[3] = (p.density_mode != 0 && p.lam_d != 0.f) ? kl : nan;
    hist_row[4] = (p.lam_r != 0.f) ? ent : nan;
    hist_row[5] = (p.lam_l1 != 0.f) ? l1 : nan;
    hist_row[6] = (p.lam_l2 != 0.f) ? l2 : nan;
    hist_row[7] = (p.lam_nb > 0.f) ? nb : nan;
    hist_row[8] = (p.lam_ct > 0.f) ? ct : nan;
    hist_row[9] = (p.lam_go > 0.f) ? go : nan;
    hist_row[10] = (p.constrained && p.lam_c != 0.f) ? count_abs : nan;
    hist_row[11] = (p.constrained && p.lam_f != 0.f) ? freg : nan;
    for (int i = 12; i < 16; ++i) hist_row[i] = p.hist_fill;
    if constexpr (kVal) {
      p.val_out[0] = gv + vg;                            // expression_sim (:328)
      p.val_out[1] = gv;                                 // gv_sim (:326)
      p.val_out[2] = sw / ws;                            // sp_sparsity_weighted_gv_sim (:329-331)
      p.val_out[3] = -(tail[p.val_ent] / p.val_log_v) / p.val_n;  // entropy (:333)
    }
  }
}

// dY_ext = dL/dY_ext (V x Ke): gene columns from the cosine terms (+ transposed SpMM of
// the spatial terms), density columns, cell-type columns.  Written in f32 and, for the
// tensor-core path, bf16.
__global__ void __launch_bounds__(kLossCols)
k_dy_assemble(LossParams p, float* __restrict__ dY, __nv_bfloat16* __restrict__ dYb, Split3 split) {
  const int k0 = (blockIdx.y * kLossCols + threadIdx.x) * kLossVec;     // four columns per thread
  const int j = blockIdx.x;                  // voxels on gridDim.x (2^31 - 1): gridDim.y stops at 65535, real sections have more spots
  if (k0 >= p.Ke) return;
  const size_t o = (size_t)j * p.Ke + k0;
  const float4 y4 = *reinterpret_cast<const float4*>(p.Y + o);
  const float4 g4 = *reinterpret_cast<const float4*>(p.G + o);
  const float yv[4] = {y4.x, y4.y, y4.z, y4.w}, gv[4] = {g4.x, g4.y, g4.z, g4.w};
  float out[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int k = k0 + e;
    float dy = 0.f;
    if (k < p.K) {
      if (p.act != nullptr && p.act[k] == 0.f) { out[e] = 0.f; continue; }   // a gene outside the loss: exactly 0
      const float y = yv[e], g = gv[e];
      dy = -(p.coefA[k] * g - p.coefB[k] * y);
      if (p.lam_g2 != 0.f) dy -= p.coefAr[j] * g - p.coefBr[j] * y;
      if (p.lam_nb > 0.f) {
        const float a = p.coefAn[k], b = p.coefBn[k];
        float acc = 0.f;
        for (int q = p.WT.indptr[j]; q < p.WT.indptr[j + 1]; ++q) {
          const size_t w = (size_t)p.WT.indices[q] * p.Ke + k;
          acc += p.WT.vals[q] * (a * p.WG[w] - b * p.Z[w]);
        }
        dy -= acc;
      }
      if (p.lam_go > 0.f) {
        const float a = p.coefAg[k], b = p.coefBg[k];
        float acc = 0.f;
        for (int q = p.AT.indptr[j]; q < p.AT.indptr[j + 1]; ++q) {
          const size_t w = (size_t)p.AT.indices[q] * p.Ke + k;
          acc += p.AT.vals[q] * (a * p.AG[w] - b * p.Zg[w]);
        }
        dy -= acc;
      }
    } else if (k < p.K + 2) {
      dy = (p.density_mode != 0) ? p.densg[j] : 0.f;
    } else if (k < p.ct_off + p.T && p.lam_ct > 0.f) {
      const int t = k - p.ct_off;
      float acc = p.H[(size_t)j * p.T + t];
      for (int q = p.FT.indptr[j]; q < p.FT.indptr[j + 1]; ++q)
        acc -= p.FT.vals[q] * p.H[(size_t)p.FT.indices[q] * p.T + t];
      dy = p.lam_ct * acc / ((float)p.V * (float)p.T);
    }
    out[e] = dy;
  }
  if (dY != nullptr) *reinterpret_cast<float4*>(dY + o) = make_float4(out[0], out[1], out[2], out[3]);
  if (dYb != nullptr) store_p4<__nv_bfloat16>(dYb + o, out[0], out[1], out[2], out[3]);
  if (split.base != nullptr) store_split4(split, o, out[0], out[1], out[2], out[3]);
}

// ------------------------------------------------------------------------------------
// One-time helpers (constants of the loss, input packing, init).
// ------------------------------------------------------------------------------------
__global__ void k_spmm(int V, int K, int Ke, Csr op, const float* __restrict__ X, float* __restrict__ Z) {
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  const int j = blockIdx.x;                  // voxels on gridDim.x: no 65535 limit
  if (k >= Ke) return;
  float z = 0.f;
  if (k < K)
    for (int e = op.indptr[j]; e < op.indptr[j + 1]; ++e) z += op.vals[e] * X[(size_t)op.indices[e] * Ke + k];
  Z[(size_t)j * Ke + k] = z;
}

// per-column clamped norm + sign of the column sum (thread per column)
__global__ void k_col_norms(int V, int K, int Ke, const float* __restrict__ X, float* __restrict__ nrm,
                            float* __restrict__ sgn) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  float s2 = 0.f, s = 0.f;
  for (int j = 0; j < V; ++j) { const float x = X[(size_t)j * Ke + k]; s2 += x * x; s += x; }
  nrm[k] = fmaxf(sqrtf(s2), kCosEps);
  if (sgn) sgn[k] = s > 0.f ? 1.f : -1.f;
}
// Sparsity weight of each gene (_val_loss_fn, mapping_optimizer.py:329-331): w_k = 1 - gene_sparsity_k = (voxels where
// G[:, k] != 0) / V, from an integer count (thread per column); 0 for a gene outside the mask `act` and on pad columns.
__global__ void k_gene_weights(int V, int K, int Ke, const float* __restrict__ G, const float* __restrict__ act,
                               float* __restrict__ w) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= Ke) return;
  int nz = 0;
  if (k < K && (act == nullptr || act[k] != 0.f))
    for (int j = 0; j < V; ++j) nz += G[(size_t)j * Ke + k] != 0.f;
  w[k] = (float)nz / (float)V;
}
// per-row clamped norm over the K gene columns, or over the active ones of a gene mask `act` (warp per row)
__global__ void k_row_norms(int V, int K, int Ke, const float* __restrict__ X, const float* __restrict__ act,
                            float* __restrict__ nrm) {
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= V) return;
  float s2 = 0.f;
  for (int k = threadIdx.x & 31; k < K; k += 32) {
    if (act != nullptr && act[k] == 0.f) continue;
    const float x = X[(size_t)j * Ke + k]; s2 += x * x;
  }
  s2 = warp_sum(s2);
  if ((threadIdx.x & 31) == 0) nrm[j] = fmaxf(sqrtf(s2), kCosEps);
}

// dst[r][0:cols] = src[r][0:cols] (dense, ld = cols) into a padded row-major buffer; pad untouched
__global__ void k_pack_rows(const float* __restrict__ src, int rows, int cols, float* __restrict__ dst, int ld,
                            int col_off) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)rows * cols) return;
  const int r = (int)(i / cols), c = (int)(i % cols);
  dst[(size_t)r * ld + col_off + c] = src[i];
}
// density columns of S_ext: cells mode (1, 0); clusters mode (w, 0) in fp32 or (hi, lo) split for bf16
__global__ void k_fill_density_cols(float* __restrict__ Sx, int rows, int ld, int col, const float* __restrict__ w,
                                    int split_bf16) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  float a = 1.f, b = 0.f;
  if (w != nullptr) {
    a = w[r];
    if (split_bf16) {
      const float hi = __bfloat162float(__float2bfloat16_rn(a));
      b = a - hi; a = hi;
    }
  }
  Sx[(size_t)r * ld + col] = a;
  Sx[(size_t)r * ld + col + 1] = b;
}
__global__ void k_f32_to_bf16(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __float2bfloat16_rn(src[i]);
}
__global__ void k_bf16_to_f32(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = __bfloat162float(src[i]);
}
// zero n 16-byte words, stream-ordered: the cudaMemsetAsync of optimizer state held in mapped host memory
__global__ void k_zero16(uint4* __restrict__ p, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = make_uint4(0, 0, 0, 0);
}
// M0 ~ N(0,1) on device (Philox4x32-10), pad columns zero.  Throughput runs only; the
// reference draw (:150) is a host MT19937 float64 draw and is uploaded via set_mapping.
__global__ void k_init_normal(float* __restrict__ M, int rows, int V, int ld, unsigned long long seed, long long first_row) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;  // one float4 each
  const int nvec = ld >> 2;
  if (q >= (long long)rows * nvec) return;
  const int r = (int)(q / nvec), c = (int)(q % nvec) * 4;
  curandStatePhilox4_32_10_t st;
  // subsequence = global float4 index: the draw does not depend on how the cells are sharded over ranks
  curand_init(seed, (unsigned long long)(q + first_row * nvec), 0, &st);
  float4 n = curand_normal4(&st);
  if (c + 0 >= V) n.x = 0.f;
  if (c + 1 >= V) n.y = 0.f;
  if (c + 2 >= V) n.z = 0.f;
  if (c + 3 >= V) n.w = 0.f;
  reinterpret_cast<float4*>(M + (size_t)r * ld)[c >> 2] = n;
}
// ---- tensor-core path: row normalisation carried across iterations -------------------------
// The streaming update of iteration t writes, for iteration t+1, Pt_ij = exp(Mnew_ij - lseA_i)
// (bf16) where lseA_i is the exact log-sum-exp of the OLD row, plus per-row sums of Pt
// (and Pt*M, |M|, M^2 when those terms are on).  This kernel turns them into the exact statistics
// of the new row:  zt_i = sum_j Pt_ij,  lseT_i = lseA_i + log zt_i,  P_ij = Pt_ij / zt_i,
// h_i = sum_j P log P = px_i / zt_i - lseT_i.   `fresh` = P was just produced by the row pass
// (already normalised: zt = 1, lseT = mx + log Z).
__global__ void k_row_norm(int fresh, const float* __restrict__ zsum, const float* __restrict__ pxsum,
                           const float* __restrict__ l1sum, const float* __restrict__ l2sum,
                           const float* __restrict__ lseA, float* __restrict__ lseT, float* __restrict__ inv_zt,
                           RowStat* __restrict__ stats, float* __restrict__ rowaux, int row0, int row1) {
  const int i = row0 + blockIdx.x * blockDim.x + threadIdx.x;   // rows [row0, row1)
  if (i >= row1) return;
  if (fresh) {
    const RowStat st = stats[i];
    lseT[i] = st.mx + st.log_z;
    inv_zt[i] = 1.f;
    return;   // stats[i].h and rowaux were written by the row pass
  }
  const float z = zsum[i];
  const float lt = lseA[i] + logf(z);
  lseT[i] = lt;
  inv_zt[i] = 1.f / z;
  RowStat st;
  st.mx = lt; st.inv_z = 1.f; st.log_z = 0.f;
  st.h = pxsum ? pxsum[i] / z - lt : 0.f;
  stats[i] = st;
  if (rowaux && l1sum) { rowaux[2 * i] = l1sum[i]; rowaux[2 * i + 1] = l2sum[i]; }
}
// Sxs[i][:] = bf16(Sx[i][:] * inv_zt[i]): the forward B operand carries the row normalisation
__global__ void k_scale_rows_bf16(const float* __restrict__ Sx, const float* __restrict__ inv_zt, int row0, int row1, int ld,
                                  __nv_bfloat16* __restrict__ out) {
  const int nvec = ld >> 2;
  const long long q = (long long)row0 * nvec + (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one float4 each, rows [row0, row1)
  if (q >= (long long)row1 * nvec) return;
  const int r = (int)(q / nvec);
  const float s = inv_zt[r];
  const float4 v = reinterpret_cast<const float4*>(Sx)[q];
  store_p4<__nv_bfloat16>(out + q * 4, v.x * s, v.y * s, v.z * s, v.w * s);
}
// Staged backward: the store-only contraction left partials of r'_i = sum_j Pt_ij (dP_ij - c_i); with P = Pt / zt:
//   rowc_i = (lseT_i, r'_i / zt_i, h_i, 0) for the streaming Adam kernel,  r_i = c_i + r'_i / zt_i  (full row-dot),
// and r_i becomes the centre of the next iteration's dq.  Rows [row0, row1).
__global__ void k_rowdot_finalize_staged(const float* __restrict__ rpart, int nparts, int n_rows, int row0, int row1,
                                         const float* __restrict__ lseT, const float* __restrict__ inv_zt,
                                         const RowStat* __restrict__ stats, float* __restrict__ center,
                                         float* __restrict__ r, float4* __restrict__ rowc) {
  const int i = row0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= row1) return;
  float s = 0.f;
  for (int p = 0; p < nparts; ++p) s += rpart[(size_t)p * n_rows + i];
  s *= inv_zt[i];
  const float full = center[i] + s;
  r[i] = full;
  center[i] = full;
  rowc[i] = make_float4(lseT[i], s, stats[i].h, 0.f);
}

// out = sum of `nplanes` partial planes (deterministic order); used before the NCCL exchange
__global__ void k_sum_planes(const float* __restrict__ part, int nplanes, size_t plane, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= plane) return;
  float s = 0.f;
  for (int z = 0; z < nplanes; ++z) s += part[(size_t)z * plane + i];
  out[i] = s;
}
// r_i = sum over partial arrays (deterministic order)
__global__ void k_rowdot_finalize(const float* __restrict__ rpart, int nparts, int n_rows, float* __restrict__ r) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  float s = 0.f;
  for (int p = 0; p < nparts; ++p) s += rpart[(size_t)p * n_rows + i];
  r[i] = s;
}

}  // namespace tgb
