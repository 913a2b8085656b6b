// Shared device helpers for the tangram_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace tgb {

constexpr float kCosEps = 1e-8f;   // torch cosine_similarity eps (mapping_optimizer.py:205)
constexpr int kWarp = 32;

__host__ __device__ inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
__host__ __device__ inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide reductions; `sh` needs >= 32 floats.  Result is broadcast to all threads.
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* sh) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int nw = (blockDim.x + 31) >> 5;
  v = kMax ? warp_max(v) : warp_sum(v);
  __syncthreads();                 // protect sh reuse across consecutive calls
  if (lane == 0) sh[wid] = v;
  __syncthreads();
  float r = (lane < nw) ? sh[lane] : (kMax ? -INFINITY : 0.f);
  r = kMax ? warp_max(r) : warp_sum(r);
  return r;
}

// 128-bit streaming accesses: M/m/v/P are touched once per pass, keep them out of L1.
__device__ __forceinline__ float4 ld_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(float4* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Per-row softmax statistics written by the row pass and reused by backward.
struct __align__(16) RowStat {
  float mx;     // row max of M
  float inv_z;  // 1 / sum_j exp(M_ij - mx)
  float log_z;  // log of that sum
  float h;      // sum_j P_ij log P_ij   (only when lambda_r != 0, else 0)
};

// The one definition of P_ij used everywhere (forward operand, backward epilogue, output),
// so every kernel sees bit-identical probabilities.  Reference: softmax(M, dim=1), :201.
__device__ __forceinline__ float softmax_prob(float x, const RowStat& s) {
  return expf(x - s.mx) * s.inv_z;
}

template <typename T> struct PType;
template <> struct PType<float> {
  static __device__ __forceinline__ float from(float v) { return v; }
};
template <> struct PType<__nv_bfloat16> {
  static __device__ __forceinline__ __nv_bfloat16 from(float v) { return __float2bfloat16_rn(v); }
};

}  // namespace tgb
