// Run-to-run agreement of R equally shaped arrays in one streaming pass (tangram/mapping_parameter_tuning.py:42-82, the
// metrics of the hyper-parameter tuner's trial): the fp64 sums and pairwise cross-product sums behind `pearson_corr`, and,
// per row, `vote_entropy` and `consensus_entropy` of the mapping cube.  Every element is read once (4 R bytes), nothing of
// size rows x cols is written.  The target is the HBM bound; DESIGN.md §6b has how close it gets.
//
// Determinism: one row per warp, rows dealt to warps in a fixed order, per-block partials in fp64 reduced by one block in
// block order (no float atomics), so a re-run on the same device gives identical bits.
// Cancellation: the cross products are taken about a per-array shift (the mean of a fixed strided sample), which makes the
// one-pass  sum(dx dy) - sum(dx) sum(dy) / n  as accurate as a two-pass centred sum when the shift is near the mean.
// Row shards (the sharded tuner trial): each shard returns its sample's sums and size (k_agreement_shift with sums = 1);
// the caller adds them over the shards, so every shard takes its cross products about the same shift, near the global
// mean; each shard's k_agreement partials are summed in block order (k_agreement_total), the caller adds those over the
// shards, and k_agreement_pearson finishes with the global element count.  One shard holding every row computes exactly
// what k_agreement_shift / k_agreement / k_agreement_finish compute.
#pragma once
#include "common.cuh"

namespace tgb {

constexpr int kAgrMaxRuns = 8;
constexpr int kAgrThreads = 256;          // 8 warps, one row per warp at a time
constexpr int kAgrSample = 4096;          // elements per array behind the shift

struct AgrArgs {
  const float* x[kAgrMaxRuns];            // R arrays, rows x cols, leading dimension ld (elements)
  long long rows, cols, ld;
  int vec;                                // every array 16-byte aligned and ld % 4 == 0: float4 loads
  const double* shift;                    // [R] (k_agreement_shift)
  double* part;                           // [gridDim.x][R + R(R+1)/2] per-block sums: sum dx_r, then sum dx_r dx_s (r <= s)
  float* vote;                            // [rows] vote entropy, or nullptr
  float* cons;                            // [rows] consensus entropy, or nullptr
};

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// shift[r] = mean of kAgrSample elements spread evenly over array r (grid = R blocks of kAgrThreads).  With sums != 0
// shift[r] is the sample's sum instead and shift[R] its size, for a caller that adds the samples of several row shards.
__global__ void __launch_bounds__(kAgrThreads) k_agreement_shift(AgrArgs a, double* shift, int sums) {
  __shared__ double sh[kAgrThreads];
  const float* x = a.x[0];
#pragma unroll
  for (int r = 1; r < kAgrMaxRuns; ++r)                               // static indexing keeps a.x in the parameter bank
    if (r == (int)blockIdx.x) x = a.x[r];
  const long long total = a.rows * a.cols;
  const int ns = total < kAgrSample ? (int)total : kAgrSample;
  double acc = 0.0;
  for (int k = threadIdx.x; k < ns; k += kAgrThreads) {
    const long long e = total / ns * k + (total % ns) * k / ns;       // floor(total k / ns) without overflow
    acc += (double)x[(e / a.cols) * a.ld + e % a.cols];
  }
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int w = kAgrThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) shift[blockIdx.x] = sums ? sh[0] : sh[0] / ns;
  if (sums && blockIdx.x == 0 && threadIdx.x == 0) shift[gridDim.x] = (double)ns;
}

template <int R, bool kRows>
struct AgrAcc {
  static constexpr int NP = R * (R + 1) / 2;
  double sx[R], sxy[NP];
  float best[R];
  int bidx[R];
  double csum, cplogp;                    // row sums of p = mean_r x_r and of p log p

  __device__ __forceinline__ void add(const float (&v)[R], const double (&sh)[R], int j) {
    double d[R];
#pragma unroll
    for (int r = 0; r < R; ++r) { d[r] = (double)v[r] - sh[r]; sx[r] += d[r]; }
    int k = 0;
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int s = r; s < R; ++s, ++k) sxy[k] = fma(d[r], d[s], sxy[k]);
    if (kRows) {
      float p = v[0];
#pragma unroll
      for (int r = 0; r < R; ++r) {
        // argmax_prefer's order, specialised to a lane that sees its columns in increasing order: a larger value or the
        // first NaN takes the place (!(v <= best) holds for a NaN v), nothing replaces a NaN, and an equal value keeps
        // the earlier column.  -inf is never taken: a lane that saw only -inf keeps bidx = INT_MAX (see below).
        if (!(v[r] <= best[r]) && best[r] == best[r]) { best[r] = v[r]; bidx[r] = j; }
        if (r > 0) p += v[r];
      }
      p = p / (float)R;                                               // numpy's float32 mean over the runs
      csum += (double)p;
      if (p > 0.f) cplogp += (double)(p * logf(p));                   // entr(0) = 0
    }
  }
};

// One pass over the R arrays.  Grid: any number of blocks (fixed for a device); warp w of block b takes rows
// b * 8 + w, then strides by gridDim.x * 8.
template <int R, bool kRows>
__global__ void __launch_bounds__(kAgrThreads) k_agreement(AgrArgs a) {
  constexpr int NP = R * (R + 1) / 2, NS = R + NP;
  __shared__ double wsum[kAgrThreads / kWarp][NS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  AgrAcc<R, kRows> acc;
  double sh[R];
#pragma unroll
  for (int r = 0; r < R; ++r) { acc.sx[r] = 0.0; sh[r] = a.shift[r]; }
#pragma unroll
  for (int k = 0; k < NP; ++k) acc.sxy[k] = 0.0;
  const long long cols = a.cols, cols4 = a.vec ? (cols & ~3LL) : 0;
  for (long long row = (long long)blockIdx.x * (kAgrThreads / kWarp) + warp; row < a.rows;
       row += (long long)gridDim.x * (kAgrThreads / kWarp)) {
    if (kRows) {
#pragma unroll
      for (int r = 0; r < R; ++r) { acc.best[r] = -INFINITY; acc.bidx[r] = INT_MAX; }
      acc.csum = 0.0; acc.cplogp = 0.0;
    }
    const size_t base = (size_t)row * a.ld;
    // software-pipelined: the next column block is in flight while this one is reduced
    float4 q[R], qn[R];
    if (4 * lane < cols4) {
#pragma unroll
      for (int r = 0; r < R; ++r) q[r] = ld_stream(reinterpret_cast<const float4*>(a.x[r] + base + 4 * lane));
    }
    for (long long c = 4 * lane; c < cols4; c += 4 * kWarp) {
      if (c + 4 * kWarp < cols4) {
#pragma unroll
        for (int r = 0; r < R; ++r) qn[r] = ld_stream(reinterpret_cast<const float4*>(a.x[r] + base + c + 4 * kWarp));
      }
      float v[R];
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = q[r].x;
      acc.add(v, sh, (int)c);
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = q[r].y;
      acc.add(v, sh, (int)c + 1);
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = q[r].z;
      acc.add(v, sh, (int)c + 2);
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = q[r].w;
      acc.add(v, sh, (int)c + 3);
#pragma unroll
      for (int r = 0; r < R; ++r) q[r] = qn[r];
    }
    for (long long c = cols4 + lane; c < cols; c += kWarp) {         // ragged tail / unaligned arrays
      float v[R];
#pragma unroll
      for (int r = 0; r < R; ++r) v[r] = __ldg(a.x[r] + base + c);
      acc.add(v, sh, (int)c);
    }
    if (kRows) {
      // argmax per run: largest value, first column on ties (np.argmax)
#pragma unroll
      for (int r = 0; r < R; ++r) {
        warp_argmax(acc.best[r], acc.bidx[r]);
        if (acc.bidx[r] == INT_MAX) acc.bidx[r] = 0;                 // every value -inf: np.argmax votes for column 0
      }
      const double s = warp_sum_d(acc.csum), plogp = warp_sum_d(acc.cplogp);
      if (lane == 0) {
        // one column: the reference divides by log(1) = 0, and the bracket of the consensus entropy need not round to
        // exactly 0, so both entropies are NaN by definition rather than 0 * inf or +-inf
        const double inv_log_cols = cols > 1 ? 1.0 / log((double)cols) : (double)NAN;
        if (a.vote) {
          // scipy.stats.entropy of the vote shares c / R, groups taken in column order as numpy sums them
          double h = 0.0, tot = 0.0;
          int prev = -1;
          for (int g = 0; g < R; ++g) {
            int col = INT_MAX, cnt = 0;
#pragma unroll
            for (int r = 0; r < R; ++r) if (acc.bidx[r] > prev && acc.bidx[r] < col) col = acc.bidx[r];
            if (col == INT_MAX) break;
#pragma unroll
            for (int r = 0; r < R; ++r) cnt += acc.bidx[r] == col;
            tot += (double)cnt / R;
            prev = col;
          }
          prev = -1;
          for (int g = 0; g < R; ++g) {
            int col = INT_MAX, cnt = 0;
#pragma unroll
            for (int r = 0; r < R; ++r) if (acc.bidx[r] > prev && acc.bidx[r] < col) col = acc.bidx[r];
            if (col == INT_MAX) break;
#pragma unroll
            for (int r = 0; r < R; ++r) cnt += acc.bidx[r] == col;
            const double p = (double)cnt / R / tot;
            h += -(p * log(p));
            prev = col;
          }
          a.vote[row] = (float)(h * inv_log_cols);
        }
        if (a.cons) a.cons[row] = (float)((log(s) - plogp / s) * inv_log_cols);     // entropy of p / sum(p)
      }
    }
  }
  // block partials: warp butterfly, then warps in order
#pragma unroll
  for (int r = 0; r < R; ++r) { const double t = warp_sum_d(acc.sx[r]); if (lane == 0) wsum[warp][r] = t; }
#pragma unroll
  for (int k = 0; k < NP; ++k) { const double t = warp_sum_d(acc.sxy[k]); if (lane == 0) wsum[warp][R + k] = t; }
  __syncthreads();
  if (threadIdx.x < NS) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kAgrThreads / kWarp; ++w) t += wsum[w][threadIdx.x];
    a.part[(size_t)blockIdx.x * NS + threadIdx.x] = t;
  }
}

// Threads [0, NS) of one block: tot[k] = sum of the per-block partials part[b][k] in block order.
__device__ __forceinline__ void agr_total(const double* part, int nblocks, int NS, double* tot) {
  if (threadIdx.x < NS) {
    double t = 0.0;
    for (int b = 0; b < nblocks; ++b) t += part[(size_t)b * NS + threadIdx.x];
    tot[threadIdx.x] = t;
  }
}

// One thread: np.corrcoef's pairwise correlations from the sums tot (sum dx_r, then sum dx_r dx_s for r <= s) of n
// elements per array, in np.tril_indices(R, -1) order: (1,0), (2,0), (2,1), (3,0), ...
__device__ __forceinline__ void agr_pearson(const double* tot, int R, double n, double* corr) {
  auto pidx = [R](int r, int s) { return R + r * R - r * (r - 1) / 2 + (s - r); };   // r <= s
  auto cov = [&](int r, int s) { return (tot[pidx(r, s)] - tot[r] * tot[s] / n) / (n - 1.0); };
  int k = 0;
  for (int i = 1; i < R; ++i)
    for (int j = 0; j < i; ++j, ++k) {
      double c = cov(j, i) / sqrt(cov(i, i)) / sqrt(cov(j, j));
      corr[k] = c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c);           // np.corrcoef clips to [-1, 1]
    }
}

// One block: sums the per-block partials in block order and forms the correlations (tgb200_agreement).
__global__ void k_agreement_finish(const double* part, int nblocks, int R, double n, double* corr) {
  __shared__ double tot[kAgrMaxRuns + kAgrMaxRuns * (kAgrMaxRuns + 1) / 2];
  agr_total(part, nblocks, R + R * (R + 1) / 2, tot);
  __syncthreads();
  if (threadIdx.x == 0) agr_pearson(tot, R, n, corr);
}

// The two halves of k_agreement_finish for row shards (tgb200_agreement_partials, tgb200_agreement_pearson): one block
// of at least R + R(R+1)/2 threads sums a shard's partials into tot; one thread forms the correlations from the sums
// of every shard.
__global__ void k_agreement_total(const double* part, int nblocks, int R, double* tot) {
  agr_total(part, nblocks, R + R * (R + 1) / 2, tot);
}

__global__ void k_agreement_pearson(const double* tot, int R, double n, double* corr) {
  if (threadIdx.x == 0) agr_pearson(tot, R, n, corr);
}

}  // namespace tgb
