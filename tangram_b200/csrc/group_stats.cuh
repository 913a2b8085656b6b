// Per-label column statistics of an expression matrix (the basic statistics of scanpy's rank_genes_groups and
// highly_variable_genes): for every label t and gene k the fp64 sum of y, the fp64 sum of y * y and the count of x != 0
// over the rows labelled t, in one streaming pass that reads every dense element or stored CSR entry once.  y is the
// element's value under a compile-time transform: GsValue::kIdentity, y = (double)x (rank_genes_groups), or
// GsValue::kExpm1, y = expm1(scale * (double)x) in fp64 (highly_variable_genes' seurat flavor, which undoes log1p).
// The count is always of the untransformed x (NaN counts).
//
// Summation order (part of the contract, so the bits do not depend on how the data arrives): each aligned range of
// kGsRange cells forms one chain per label -- that range's rows of the label, added in row order, starting from 0.0 --
// and the chains are added in range order, starting from 0.0.  Absent CSR entries and explicit zeros both add +0.0, so
// dense and CSR input of the same matrix give the same bits; so do host and device pointers and any block size.  Under
// kExpm1 an absent entry becomes expm1(scale * 0.0) = +-0.0, which adds nothing either, so the same holds.
//
// Work split: the host stable-sorts the labelled rows of each range by label (perm) and cuts them into runs of one label.
// k_group_stats: one CTA per (range, slab of kGsSlab genes); each thread owns four genes and walks the range's runs in
// batches of kGsRows rows, flushing its sums to a per-run partial at the end of each run.  For CSR, the CTA first scatters
// the batch's rows into a zeroed kGsRows x kGsSlab shared tile (one warp per row, the slab's first entry found by a
// 32-way search of the row's strictly increasing columns) and then runs exactly the dense accumulation on the tile.
// k_group_stats_fold adds each label's run partials into the outputs in range order.  No atomics.
#pragma once
#include "common.cuh"

namespace tgb {

constexpr int kGsThreads = 256;
constexpr int kGsSlab = 4 * kGsThreads;        // genes per CTA: four per thread
constexpr int kGsRange = 2048;                 // cells per summation chain
constexpr int kGsRows = kGsThreads / kWarp;    // rows per batch: one CSR row per warp

enum class GsValue { kIdentity, kExpm1 };

struct GsArgs {
  const float* x;                              // dense: row i of the block at x + i * ld
  long long ld;
  int vec;                                     // x 16-byte aligned and ld % 4 == 0: float4 loads
  const int64_t* indptr;                       // CSR: nb + 1 absolute offsets (the block's entries start at indptr[0])
  const int* indices;                          //   the block's entries
  const float* data;
  long long n_genes;
  const int* perm;                             // labelled rows of the block (offsets in it), each range's stably by label
  const int* run_start;                        // [n_runs + 1]: run k covers perm[run_start[k] .. run_start[k + 1])
  const int* range_runs;                       // [n_ranges + 1]: range r holds runs range_runs[r] .. range_runs[r + 1]
  double scale;                                // kExpm1: y = expm1(scale * x)
  double* psum;                                // [n_runs][n_genes] per-run partials
  double* psq;
  int* pcnt;
};

// Row `row` of the CSR block into the shared tile row `trow` (columns [s0, s0 + kGsSlab)), by one warp.  Columns out of
// order or out of range are caught by k_gs_csr_check; here they can only cause missed entries, never a stray write.
__device__ __forceinline__ void gs_scatter_row(const GsArgs& a, int row, int s0, float* trow, int lane) {
  const int64_t base = a.indptr[0], hi = a.indptr[row + 1] - base;
  int64_t lo = a.indptr[row] - base, top = hi;           // the first column >= s0 is at a position in [lo, top]
  while (top - lo > kWarp) {
    const int64_t step = (top - lo + kWarp - 1) / kWarp, p = lo + lane * step;
    const int k = __popc(__ballot_sync(0xffffffffu, p < top && a.indices[p] < s0));
    if (k == 0) break;                                   // lo itself holds a column >= s0
    const int64_t last_below = lo + (int64_t)(k - 1) * step;
    top = min(top, last_below + step);
    lo = last_below + 1;
  }
  const int s1 = s0 + kGsSlab;
  for (int64_t p = lo + lane;; p += kWarp) {
    const int c = p < hi ? a.indices[p] : INT_MAX;
    if (c >= s0 && c < s1) trow[c - s0] = a.data[p];
    if (!__all_sync(0xffffffffu, c < s1)) break;          // columns increase: nothing of this slab further on
  }
}

template <bool kCsr, GsValue kValue>
__global__ void __launch_bounds__(kGsThreads) k_group_stats(GsArgs a) {
  __shared__ __align__(16) float tile[kCsr ? kGsRows : 1][kCsr ? kGsSlab : 4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s0 = blockIdx.x * kGsSlab;
  const long long c0 = (long long)s0 + 4 * threadIdx.x;
  const int nv = c0 >= a.n_genes ? 0 : (int)min(4LL, a.n_genes - c0);      // valid genes of this thread
  const bool v4 = a.vec && nv == 4;
  int run = a.range_runs[blockIdx.y];
  const int run_end = a.range_runs[blockIdx.y + 1];
  if (run == run_end) return;                                             // no labelled row in this range
  const int p_end = a.run_start[run_end];
  int next = a.run_start[run + 1];                                        // where the current run ends
  double s[4] = {0.0, 0.0, 0.0, 0.0}, q[4] = {0.0, 0.0, 0.0, 0.0};
  int n[4] = {0, 0, 0, 0};
  for (int b0 = a.run_start[run]; b0 < p_end; b0 += kGsRows) {
    const int nb = min(kGsRows, p_end - b0);
    float v[kGsRows][4];
    if (kCsr) {
      __syncthreads();                                                    // the previous batch's tile is consumed
      float4* t4 = reinterpret_cast<float4*>(&tile[0][0]);
      for (int k = threadIdx.x; k < kGsRows * kGsSlab / 4; k += kGsThreads) t4[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      if (warp < nb) gs_scatter_row(a, a.perm[b0 + warp], s0, tile[warp], lane);
      __syncthreads();
#pragma unroll
      for (int u = 0; u < kGsRows; ++u) {
        if (u >= nb) break;
        const float4 t = *reinterpret_cast<const float4*>(&tile[u][4 * threadIdx.x]);
        v[u][0] = t.x; v[u][1] = t.y; v[u][2] = t.z; v[u][3] = t.w;
      }
    } else {
#pragma unroll
      for (int u = 0; u < kGsRows; ++u) {
        if (u >= nb) break;
        const float* src = a.x + (size_t)a.perm[b0 + u] * a.ld + c0;
        if (v4) {
          const float4 t = ld_stream(reinterpret_cast<const float4*>(src));
          v[u][0] = t.x; v[u][1] = t.y; v[u][2] = t.z; v[u][3] = t.w;
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) v[u][e] = e < nv ? __ldg(src + e) : 0.f;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < kGsRows; ++u) {
      if (u >= nb) break;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const double y = kValue == GsValue::kExpm1 ? expm1(a.scale * (double)v[u][e]) : (double)v[u][e];
        s[e] += y;
        q[e] = __fma_rn(y, y, q[e]);    // fused whatever -fmad says; for the identity y * y is exact, so unfused alike
        n[e] += v[u][e] != 0.f;                                           // NaN counts
      }
      if (b0 + u + 1 == next) {                                           // the run ends: flush its partial
        const size_t o = (size_t)run * a.n_genes + c0;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (e < nv) { a.psum[o + e] = s[e]; a.psq[o + e] = q[e]; a.pcnt[o + e] = n[e]; }
          s[e] = 0.0; q[e] = 0.0; n[e] = 0;
        }
        if (++run < run_end) next = a.run_start[run + 1];
      }
    }
  }
}

// One warp per row of the CSR block: flags a column outside [0, n_genes) or not strictly increasing within its row.
__global__ void __launch_bounds__(kGsThreads) k_gs_csr_check(const int64_t* indptr, const int* indices, int nb,
                                                              long long n_genes, int* bad) {
  const long long r = ((long long)blockIdx.x * kGsThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= nb) return;
  const int64_t base = indptr[0], p0 = indptr[r] - base, p1 = indptr[r + 1] - base;
  for (int64_t p = p0 + lane; p < p1; p += kWarp) {
    const int c = indices[p];
    if (c < 0 || c >= n_genes || (p > p0 && indices[p - 1] >= c)) *bad = 1;
  }
}

// sum[t, j] += the partials of label t's runs in range order (lab_runs[lab_ptr[t] .. lab_ptr[t + 1])), and so for sq and
// cnt.  Grid: (ceil(n_genes / kGsThreads), any); label t is taken by blockIdx.y, then strides by gridDim.y.
__global__ void __launch_bounds__(kGsThreads) k_group_stats_fold(const double* psum, const double* psq, const int* pcnt,
                                                                 const int* lab_ptr, const int* lab_runs, int n_labels,
                                                                 long long n_genes, double* sum, double* sq,
                                                                 long long* cnt) {
  const long long j = (long long)blockIdx.x * kGsThreads + threadIdx.x;
  if (j >= n_genes) return;
  for (int t = blockIdx.y; t < n_labels; t += gridDim.y) {
    const int k0 = lab_ptr[t], k1 = lab_ptr[t + 1];
    if (k0 == k1) continue;
    const size_t o = (size_t)t * n_genes + j;
    double s = sum[o], q = sq[o];
    long long n = cnt[o];
    for (int k = k0; k < k1; ++k) {
      const size_t i = (size_t)lab_runs[k] * n_genes + j;
      s += psum[i]; q += psq[i]; n += pcnt[i];
    }
    sum[o] = s; sq[o] = q; cnt[o] = n;
  }
}

}  // namespace tgb
