// fp32 FFMA contraction path (parity mode: the reference contracts in fp32, TF32 off).
// One register-tiled 128x128x16 kernel, templated on operand majorness and a fused epilogue:
//   forward  Y_ext  = P^T  S_ext           (:202, + density/ct columns)      -> StorePartial
//   row-dot  r_i    = <S_ext_i, (P dY_ext)_i>   (softmax-Jacobian term)      -> RowDot
//   backward dP     = S_ext dY_ext^T, fused softmax-Jacobian + Adam (:395-396) -> AdamEpilogue
#pragma once
#include "common.cuh"

namespace tgb {

struct GemmArgs {
  const float* A;   // A_KMAJOR: [M][K] (lda) else [K][M] (lda)
  const float* B;   // B_KMAJOR: [N][K] (ldb) else [K][N] (ldb)
  int M, N, K;      // true extents
  int lda, ldb;     // leading dims (multiples of 4; pad regions hold zeros)
  int k_per_split;  // multiple of 16
};

constexpr int SG_BM = 128, SG_BN = 128, SG_BK = 16, SG_LD = 132, SG_THREADS = 256;

// Adam scalars of one step (torch/optim/adam.py single-tensor path, computed in double on the host)
struct AdamScalars {
  float beta1, beta2, one_minus_beta1, one_minus_beta2, step_size, bc2_sqrt, eps, inv_bc2_sqrt;
};

// torch.optim.Adam(foreach=False) on CUDA element for element, each rounding pinned to the one torch's kernels make:
// lerp_ is self + w (end - self) contracted to one FMA, addcmul_ is self + value (t1 t2), a division of a tensor by a
// Python scalar multiplies by fp32(1 / scalar), and addcdiv_ is self + value (t1 / t2) contracted to one FMA.
__device__ __forceinline__ float adam_update(float x, float g, float& m, float& v, const AdamScalars& a) {
  m = fmaf(g - m, a.one_minus_beta1, m);                                       // exp_avg.lerp_(grad, 1-beta1)
  v = fmaf(a.one_minus_beta2, __fmul_rn(g, g), __fmul_rn(v, a.beta2));         // mul_(beta2).addcmul_(g, g, 1-beta2)
  const float denom = __fadd_rn(__fmul_rn(sqrtf(v), a.inv_bc2_sqrt), a.eps);   // (sqrt(v) / sqrt(bc2)).add_(eps)
  return fmaf(-a.step_size, m / denom, x);                                     // addcdiv_(m, denom, -step_size)
}

// ---- epilogues --------------------------------------------------------------------
struct EpiStorePartial {
  float* C; int ldc; size_t split_stride;
  __device__ __forceinline__ void operator()(const float (&acc)[8][8], int m0, int n0, int ty, int tx,
                                             int M, int N) const {
    float* c = C + (size_t)blockIdx.z * split_stride;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      if (m >= M) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = n0 + h * 64 + tx * 4;
        if (n < ldc)
          *reinterpret_cast<float4*>(c + (size_t)m * ldc + n) =
              make_float4(acc[i][h * 4 + 0], acc[i][h * 4 + 1], acc[i][h * 4 + 2], acc[i][h * 4 + 3]);
      }
    }
  }
};

struct EpiRowDot {
  const float* S; int lds;   // S_ext [M rows][lds]
  float* rpart;              // [(split * gridDim.x + blockIdx.x)][M]
  __device__ __forceinline__ void operator()(const float (&acc)[8][8], int m0, int n0, int ty, int tx,
                                             int M, int N) const {
    float* out = rpart + ((size_t)blockIdx.z * gridDim.x + blockIdx.x) * M;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      float s = 0.f;
      if (m < M) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int n = n0 + h * 64 + tx * 4;
          if (n < lds) {
            const float4 sv = *reinterpret_cast<const float4*>(S + (size_t)m * lds + n);
            s += acc[i][h * 4 + 0] * sv.x + acc[i][h * 4 + 1] * sv.y + acc[i][h * 4 + 2] * sv.z +
                 acc[i][h * 4 + 3] * sv.w;
          }
        }
      }
      // the 16 threads that share this row are the lanes with equal (lane / 16)
      s += __shfl_xor_sync(0xffffffffu, s, 8);
      s += __shfl_xor_sync(0xffffffffu, s, 4);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      if (tx == 0 && m < M) out[m] = s;
    }
  }
};

// dM_ij = P_ij (dP_ij - r_i - lam_r (log P_ij - h_i)) + lam_l1 sign(M_ij) + 2 lam_l2 M_ij, then Adam.
struct EpiAdam {
  float* Mp; float* mp; float* vp; int ld; int V;  // state, N x ld
  const RowStat* stats; const float* rdot;
  float lam_r, lam_l1, lam_l2;
  AdamScalars a;
  __device__ __forceinline__ float one(float x, float dp, float& m, float& v, const RowStat& st, float r) const {
    const float p = softmax_prob(x, st);
    float g = dp - r;
    if (lam_r != 0.f) g -= lam_r * (((x - st.mx) - st.log_z) - st.h);
    g *= p;
    if (lam_l1 != 0.f) g += lam_l1 * (float)((x > 0.f) - (x < 0.f));
    if (lam_l2 != 0.f) g += 2.f * lam_l2 * x;
    return adam_update(x, g, m, v, a);
  }
  __device__ __forceinline__ void operator()(const float (&acc)[8][8], int m0, int n0, int ty, int tx,
                                             int M, int N) const {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
      if (row >= M) continue;
      const RowStat st = stats[row];
      const float r = rdot[row];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = n0 + h * 64 + tx * 4;
        if (n >= V) continue;
        const size_t o = (size_t)row * ld + n;
        float4 x = ld_stream(reinterpret_cast<const float4*>(Mp + o));
        float4 m = ld_stream(reinterpret_cast<const float4*>(mp + o));
        float4 v = ld_stream(reinterpret_cast<const float4*>(vp + o));
        x.x = one(x.x, acc[i][h * 4 + 0], m.x, v.x, st, r);
        if (n + 1 < V) x.y = one(x.y, acc[i][h * 4 + 1], m.y, v.y, st, r);
        if (n + 2 < V) x.z = one(x.z, acc[i][h * 4 + 2], m.z, v.z, st, r);
        if (n + 3 < V) x.w = one(x.w, acc[i][h * 4 + 3], m.w, v.w, st, r);
        st_stream(reinterpret_cast<float4*>(Mp + o), x);
        st_stream(reinterpret_cast<float4*>(mp + o), m);
        st_stream(reinterpret_cast<float4*>(vp + o), v);
      }
    }
  }
};

// ---- main loop --------------------------------------------------------------------
template <bool KMAJOR>
__device__ __forceinline__ void sg_load_tile(const float* __restrict__ X, int ld, int mn0, int mn_extent,
                                             int k0, int k_end, float4 (&reg)[2]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = t + i * SG_THREADS;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (KMAJOR) {              // source [MN][K]: 128 rows x 16 k, float4 along k
      const int row = idx >> 2, kq = (idx & 3) * 4;
      const int mn = mn0 + row, k = k0 + kq;
      if (mn < mn_extent && k < k_end) {
        v = *reinterpret_cast<const float4*>(X + (size_t)mn * ld + k);
        if (k + 1 >= k_end) v.y = 0.f;
        if (k + 2 >= k_end) v.z = 0.f;
        if (k + 3 >= k_end) v.w = 0.f;
      }
    } else {                   // source [K][MN]: 16 k rows x 128 contiguous, float4 along mn
      const int kk = idx >> 5, c = (idx & 31) * 4;
      const int k = k0 + kk, mn = mn0 + c;
      if (k < k_end && mn < ld) v = *reinterpret_cast<const float4*>(X + (size_t)k * ld + mn);
    }
    reg[i] = v;
  }
}
template <bool KMAJOR>
__device__ __forceinline__ void sg_store_tile(float (*sm)[SG_LD], const float4 (&reg)[2]) {
  const int t = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int idx = t + i * SG_THREADS;
    if (KMAJOR) {
      const int row = idx >> 2, kq = (idx & 3) * 4;
      sm[kq + 0][row] = reg[i].x; sm[kq + 1][row] = reg[i].y;
      sm[kq + 2][row] = reg[i].z; sm[kq + 3][row] = reg[i].w;
    } else {
      const int kk = idx >> 5, c = (idx & 31) * 4;
      *reinterpret_cast<float4*>(&sm[kk][c]) = reg[i];
    }
  }
}

template <bool A_KMAJOR, bool B_KMAJOR, class Epi>
__global__ void __launch_bounds__(SG_THREADS, 2)
k_gemm_simt(GemmArgs g, Epi epi) {
  __shared__ __align__(16) float As[2][SG_BK][SG_LD];
  __shared__ __align__(16) float Bs[2][SG_BK][SG_LD];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int n0 = blockIdx.x * SG_BN, m0 = blockIdx.y * SG_BM;
  const int k_begin = blockIdx.z * g.k_per_split;
  const int k_end = min(g.K, k_begin + g.k_per_split);

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  if (k_begin < k_end) {
    sg_load_tile<A_KMAJOR>(g.A, g.lda, m0, g.M, k_begin, k_end, ra);
    sg_load_tile<B_KMAJOR>(g.B, g.ldb, n0, g.N, k_begin, k_end, rb);
    sg_store_tile<A_KMAJOR>(As[0], ra);
    sg_store_tile<B_KMAJOR>(Bs[0], rb);
  }
  __syncthreads();
  int buf = 0;
  for (int k0 = k_begin; k0 < k_end; k0 += SG_BK) {
    const bool more = k0 + SG_BK < k_end;
    if (more) {
      sg_load_tile<A_KMAJOR>(g.A, g.lda, m0, g.M, k0 + SG_BK, k_end, ra);
      sg_load_tile<B_KMAJOR>(g.B, g.ldb, n0, g.N, k0 + SG_BK, k_end, rb);
    }
#pragma unroll
    for (int kk = 0; kk < SG_BK; ++kk) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (more) {
      sg_store_tile<A_KMAJOR>(As[buf ^ 1], ra);
      sg_store_tile<B_KMAJOR>(Bs[buf ^ 1], rb);
    }
    __syncthreads();
    buf ^= 1;
  }
  epi(acc, m0, n0, ty, tx, g.M, g.N);
}

}  // namespace tgb
