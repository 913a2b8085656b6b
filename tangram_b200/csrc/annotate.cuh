// Annotation transfer from cells onto space (tangram/utils.py:126-153, 205-285, 820-842) in one streaming pass over an
// N x V float32 mapping P whose rows carry int32 labels in [-1, T):
//   label sums   out[t, j] = sum_{i : label_i = t} P[i, j] in fp64 (the int64 one-hot GEMM of project_cell_annotations and
//                cell_type_mapping, which numpy evaluates in float64)
//   row argmax   per labelled row, the first column holding the row maximum, NaN counting as the maximum (np.argmax of
//                count_cell_annotations)
// Rows labelled -1 are skipped.  Every mapping element is read once (4 NV bytes).
//
// Work split: the host sorts the labelled rows by label (stable counting sort) into a row permutation and cuts each
// label's segment into items of at most kAnnChunk rows.  A CTA takes one (item, column slab of kAnnSlab columns), gathers
// the item's rows through the permutation, keeps four fp64 column sums per thread and one (value, column) maximum per row
// and slab.  The chunk is a constant, so the split depends only on the labels.
// Determinism: no atomics.  k_annotate_sums adds a label's item partials in item order; k_annotate_argmax takes each
// row's maximum over the slabs in slab order (lower slab on ties).  A re-run gives identical bits on any device.
#pragma once
#include "common.cuh"

namespace tgb {

constexpr int kAnnThreads = 256;
constexpr int kAnnSlab = 4 * kAnnThreads;      // columns per CTA: one float4 per thread
constexpr int kAnnChunk = 128;                 // rows per work item
constexpr int kAnnUnroll = 4;                  // rows in flight per thread

struct AnnArgs {
  const float* map;                            // rows x cols, leading dimension ld (elements)
  long long cols, ld;
  int vec;                                     // map 16-byte aligned and ld % 4 == 0: float4 loads
  const int* perm;                             // labelled rows, grouped by label, stable within a label
  const int* item_start;                       // [n_items + 1]: item k covers perm[item_start[k] .. item_start[k + 1])
  int n_items, n_slabs;
  double* part;                                // [n_items][cols] per-item column sums, or nullptr
  float* amax_val;                             // [n_labelled][n_slabs] per-slab row maximum, or nullptr
  int* amax_idx;                               //   and its column
};

template <bool kSums, bool kArgmax>
__global__ void __launch_bounds__(kAnnThreads) k_annotate(AnnArgs a) {
  constexpr int kWarps = kAnnThreads / kWarp;
  __shared__ int srow[kAnnChunk];
  __shared__ float wbest[kArgmax ? kAnnChunk : 1][kWarps];
  __shared__ int widx[kArgmax ? kAnnChunk : 1][kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long c0 = (long long)blockIdx.x * kAnnSlab + 4 * threadIdx.x;
  const int nv = c0 >= a.cols ? 0 : (int)min(4LL, a.cols - c0);        // valid columns of this thread
  const bool v4 = a.vec && nv == 4;
  for (int item = blockIdx.y; item < a.n_items; item += gridDim.y) {
    const int p0 = a.item_start[item], n = a.item_start[item + 1] - p0;
    __syncthreads();                                                  // srow / wbest of the previous item are consumed
    for (int k = threadIdx.x; k < n; k += kAnnThreads) srow[k] = a.perm[p0 + k];
    __syncthreads();
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    for (int r0 = 0; r0 < n; r0 += kAnnUnroll) {
      float v[kAnnUnroll][4];
#pragma unroll
      for (int u = 0; u < kAnnUnroll; ++u) {
        if (r0 + u >= n) break;
        const float* src = a.map + (size_t)srow[r0 + u] * a.ld + c0;
        if (v4) {
          const float4 q = ld_stream(reinterpret_cast<const float4*>(src));
          v[u][0] = q.x; v[u][1] = q.y; v[u][2] = q.z; v[u][3] = q.w;
        } else {
#pragma unroll
          for (int e = 0; e < 4; ++e) v[u][e] = e < nv ? __ldg(src + e) : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < kAnnUnroll; ++u) {
        if (r0 + u >= n) break;
        if (kSums) {
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[e] += (double)v[u][e];
        }
        if (kArgmax) {
          float best = -INFINITY;
          int bi = INT_MAX;
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (e < nv && argmax_prefer(v[u][e], (int)c0 + e, best, bi)) { best = v[u][e]; bi = (int)c0 + e; }
          warp_argmax(best, bi);
          if (lane == 0) { wbest[r0 + u][warp] = best; widx[r0 + u][warp] = bi; }
        }
      }
    }
    if (kSums) {
      double* dst = a.part + (size_t)item * a.cols + c0;
#pragma unroll
      for (int e = 0; e < 4; ++e) if (e < nv) dst[e] = acc[e];
    }
    if (kArgmax) {
      __syncthreads();
      for (int k = threadIdx.x; k < n; k += kAnnThreads) {             // warps hold increasing columns
        float best = wbest[k][0];
        int bi = widx[k][0];
#pragma unroll
        for (int w = 1; w < kWarps; ++w)
          if (argmax_prefer(wbest[k][w], widx[k][w], best, bi)) { best = wbest[k][w]; bi = widx[k][w]; }
        const size_t o = (size_t)(p0 + k) * a.n_slabs + blockIdx.x;
        a.amax_val[o] = best;
        a.amax_idx[o] = bi;
      }
    }
  }
}

// out[t, j] = sum of the partials of label t's items, in item order (labels without rows give 0).
// Grid: (ceil(cols / kAnnThreads), any); label t is taken by blockIdx.y, then strides by gridDim.y.
__global__ void __launch_bounds__(kAnnThreads) k_annotate_sums(const double* part, const int* label_items, int n_labels,
                                                               long long cols, double* out) {
  const long long j = (long long)blockIdx.x * kAnnThreads + threadIdx.x;
  if (j >= cols) return;
  for (int t = blockIdx.y; t < n_labels; t += gridDim.y) {
    double s = 0.0;
    for (int k = label_items[t]; k < label_items[t + 1]; ++k) s += part[(size_t)k * cols + j];
    out[(size_t)t * cols + j] = s;
  }
}

// argmax[perm[p]] = the column of the largest per-slab maximum of labelled row p, the lower slab on ties.
__global__ void __launch_bounds__(kAnnThreads) k_annotate_argmax(const float* val, const int* idx, const int* perm,
                                                                 long long n_labelled, int n_slabs, int* argmax) {
  for (long long p = (long long)blockIdx.x * kAnnThreads + threadIdx.x; p < n_labelled;
       p += (long long)gridDim.x * kAnnThreads) {
    const size_t o = (size_t)p * n_slabs;
    float best = val[o];
    int bi = idx[o];
    for (int s = 1; s < n_slabs; ++s)
      if (argmax_prefer(val[o + s], idx[o + s], best, bi)) { best = val[o + s]; bi = idx[o + s]; }
    argmax[perm[p]] = bi;
  }
}

}  // namespace tgb
