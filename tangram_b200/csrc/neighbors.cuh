// Exact spatial neighbour search in fp64 (squidpy's gr.spatial_neighbors: k nearest and radius), over a uniform cell
// grid built on the device.
//
//   bbox     k_nb_bbox: per-axis min and max (order-preserving uint64 atomics) and a flag for non-finite coordinates
//   cells    k_nb_cells: each point's cell id and the per-cell histogram
//   scan     k_nb_scan_tiles + a scan of the tile totals + k_nb_scan_add: exclusive prefix of the histogram
//   scatter  k_nb_scatter: points into cell order (SoA x, y, z and the original index); the order within a cell is
//            whatever the atomics give, which the selection below makes irrelevant
//   query    k_nb_knn<K> / k_nb_radius<kFill>: one thread per point, in cell order, visits cells in growing Chebyshev
//            rings around its own cell and stops once no unvisited cell can hold a better candidate
//
// Distances are d = sqrt((dx*dx + dy*dy) + dz*dz) with dx = x_j - x_i, every operation rounded on its own (no FMA),
// so d is bit-identical to numpy's np.sqrt(((C[j] - C[i]) ** 2).sum()).  2-D points carry z = 0, which adds +0.0.
//
// The stop bound.  A point's scaled coordinate is t = fl(fl(x - lo) * inv_h) and its cell floor(t), clamped to the
// last cell.  After ring R, every unvisited point p lies beyond the ring on some axis a in a direction where cells
// remain, so t_p >= c_a + R + 1 (above) or t_p < c_a - R (below).  The scaled gap g = min over those (axis, direction)
// pairs of c_a + R + 1 - t_q or t_q - (c_a - R) therefore bounds t_p - t_q from below up to the rounding of both t,
// which is below 2.01 u (t_p + t_q) < 1e-8 cells while an axis has at most 2^24 cells.  The bound used is
// (g - 1e-6) * h_lo with h_lo = (1 / inv_h) (1 - 1e-9), below the true gap and below the computed distance of every
// unvisited point (d >= |fl(x_p - x_q)|).  The search stops when it holds k candidates and the k-th distance is
// strictly below that bound, so a point at exactly the bound is still visited and ties are ranked by index.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <limits.h>
#include <math.h>
#include <string.h>

#include "common.cuh"

namespace tgb {
namespace nb {

constexpr int kThreads = 128;            // query and helper kernels
constexpr int kScanItems = 8;            // per thread in k_nb_scan_tiles
constexpr int kScanTile = 256 * kScanItems;
constexpr int kMaxK = 64;                // largest k of the k-nearest query
constexpr double kGapMargin = 1e-6;      // cells, see the stop bound above

struct Grid {
  double lo[3];
  double inv_h;         // 1 / cell width
  double h_lo;          // (1 / inv_h) (1 - 1e-9): rounded-down cell width; 0 disables the early stop
  int nc[3];            // cells per axis (1 for a degenerate axis and for z of 2-D points)
};

// Sorted points: coordinates in cell order (SoA) and each one's original index.
struct Points {
  const double* x;
  const double* y;
  const double* z;
  const int* orig;
  const long long* start;   // cells + 1 offsets into the sorted points
};

__host__ __device__ __forceinline__ unsigned long long ordered_bits(double v) {
  unsigned long long b;
#ifdef __CUDA_ARCH__
  b = (unsigned long long)__double_as_longlong(v);
#else
  memcpy(&b, &v, 8);
#endif
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double from_ordered_bits(unsigned long long b) {
  b = (b >> 63) ? (b & 0x7fffffffffffffffull) : ~b;
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)b);
#else
  double v;
  memcpy(&v, &b, 8);
  return v;
#endif
}

// box[2a] = ordered min of axis a, box[2a + 1] = ordered max (initialised to ~0 and 0); *bad |= a coordinate is not finite.
__global__ void __launch_bounds__(kThreads) k_nb_bbox(const double* __restrict__ C, int n, int dim,
                                                       unsigned long long* __restrict__ box, int* __restrict__ bad) {
  double mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
  bool finite = true;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (a < dim) {
        const double v = C[(int64_t)i * dim + a];
        finite &= isfinite(v);
        mn[a] = fmin(mn[a], v);
        mx[a] = fmax(mx[a], v);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn[a] = fmin(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
      mx[a] = fmax(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
    }
  }
  finite = __all_sync(0xffffffffu, finite);
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (a < dim && mn[a] <= mx[a]) {   // this warp saw at least one point
        atomicMin(&box[2 * a], ordered_bits(mn[a]));
        atomicMax(&box[2 * a + 1], ordered_bits(mx[a]));
      }
    }
    if (!finite) atomicOr(bad, 1);
  }
}

__device__ __forceinline__ double scaled(double v, double lo, double inv_h) {
  return __dmul_rn(__dsub_rn(v, lo), inv_h);
}
__device__ __forceinline__ int cell_of(double t, int nc) { return min(nc - 1, (int)floor(t)); }

__device__ __forceinline__ void load_point(const double* __restrict__ C, int i, int dim, double& x, double& y,
                                           double& z) {
  x = C[(int64_t)i * dim];
  y = C[(int64_t)i * dim + 1];
  z = dim == 3 ? C[(int64_t)i * dim + 2] : 0.0;
}

// cell[i] = the cell of point i; count[cell] += 1.
__global__ void __launch_bounds__(kThreads) k_nb_cells(const double* __restrict__ C, int n, int dim, Grid g,
                                                        int* __restrict__ cell, int* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double x, y, z;
  load_point(C, i, dim, x, y, z);
  const int cx = cell_of(scaled(x, g.lo[0], g.inv_h), g.nc[0]);
  const int cy = cell_of(scaled(y, g.lo[1], g.inv_h), g.nc[1]);
  const int cz = cell_of(scaled(z, g.lo[2], g.inv_h), g.nc[2]);
  const int c = (cz * g.nc[1] + cy) * g.nc[0] + cx;
  cell[i] = c;
  atomicAdd(&count[c], 1);
}

// Exclusive prefix over tiles of kScanTile values: out[i] = sum of in[tile start .. i), tile_sum[t] = the tile's total.
__global__ void __launch_bounds__(256) k_nb_scan_tiles(const int* __restrict__ in, int64_t n,
                                                        long long* __restrict__ out, long long* __restrict__ tile_sum) {
  __shared__ long long warp_tot[8];
  const int64_t base = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * kScanItems;
  long long v[kScanItems], s = 0;
#pragma unroll
  for (int t = 0; t < kScanItems; ++t) {
    v[t] = base + t < n ? in[base + t] : 0;
    s += v[t];
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  long long inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long u = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += u;
  }
  if (lane == 31) warp_tot[w] = inc;
  __syncthreads();
  long long before = 0, total = 0;
  for (int k = 0; k < 8; ++k) {
    if (k < w) before += warp_tot[k];
    total += warp_tot[k];
  }
  long long run = before + inc - s;
#pragma unroll
  for (int t = 0; t < kScanItems; ++t) {
    if (base + t < n) out[base + t] = run;
    run += v[t];
  }
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// out[i] += tile_off[tile of i]; out[n] = the total.
__global__ void __launch_bounds__(kThreads) k_nb_scan_add(long long* __restrict__ out, int64_t n,
                                                           const long long* __restrict__ tile_off, int n_tiles) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] += tile_off[i / kScanTile];
  if (i == 0) out[n] = tile_off[n_tiles];
}

// Points into cell order; count[] (the histogram) is consumed.
__global__ void __launch_bounds__(kThreads) k_nb_scatter(const double* __restrict__ C, int n, int dim,
                                                          const int* __restrict__ cell, int* __restrict__ count,
                                                          const long long* __restrict__ start, double* __restrict__ xs,
                                                          double* __restrict__ ys, double* __restrict__ zs,
                                                          int* __restrict__ orig) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = cell[i];
  const long long p = start[c] + atomicSub(&count[c], 1) - 1;
  double x, y, z;
  load_point(C, i, dim, x, y, z);
  xs[p] = x;
  ys[p] = y;
  zs[p] = z;
  orig[p] = i;
}

__device__ __forceinline__ double dist(double qx, double qy, double qz, double px, double py, double pz) {
  const double dx = __dsub_rn(px, qx), dy = __dsub_rn(py, qy), dz = __dsub_rn(pz, qz);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

// One query's walk over the grid: its cell, its scaled coordinates, and the ring bookkeeping.
struct Walk {
  int c[3];
  double t[3];
  __device__ __forceinline__ Walk(const Grid& g, double x, double y, double z) {
    t[0] = scaled(x, g.lo[0], g.inv_h);
    t[1] = scaled(y, g.lo[1], g.inv_h);
    t[2] = scaled(z, g.lo[2], g.inv_h);
#pragma unroll
    for (int a = 0; a < 3; ++a) c[a] = cell_of(t[a], g.nc[a]);
  }
  // Lower bound on the computed distance of every point outside rings 0..R; +inf when no cell is left.
  __device__ __forceinline__ double bound(const Grid& g, int R) const {
    double gap = INFINITY;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (c[a] + R + 1 <= g.nc[a] - 1) gap = fmin(gap, (double)(c[a] + R + 1) - t[a]);
      if (c[a] - R - 1 >= 0) gap = fmin(gap, t[a] - (double)(c[a] - R));
    }
    if (gap == INFINITY) return INFINITY;
    return (gap - kGapMargin) * g.h_lo;
  }
  // Calls f(p) for every sorted point p in the cells at Chebyshev distance exactly R.
  template <class F>
  __device__ __forceinline__ void ring(const Grid& g, const Points& P, int R, F&& f) const {
    const int z0 = max(0, c[2] - R), z1 = min(g.nc[2] - 1, c[2] + R);
    const int y0 = max(0, c[1] - R), y1 = min(g.nc[1] - 1, c[1] + R);
    const int x0 = max(0, c[0] - R), x1 = min(g.nc[0] - 1, c[0] + R);
    for (int cz = z0; cz <= z1; ++cz) {
      for (int cy = y0; cy <= y1; ++cy) {
        const bool full = abs(cz - c[2]) == R || abs(cy - c[1]) == R;
        const int row = (cz * g.nc[1] + cy) * g.nc[0];
        // a full row of the ring, or only its two ends (one when R == 0 or when an end is outside the grid)
        for (int cx = full ? x0 : c[0] - R; cx <= (full ? x1 : c[0] + R); cx += full ? 1 : 2 * max(R, 1)) {
          if (cx < 0 || cx >= g.nc[0]) continue;
          const long long p1 = P.start[row + cx + 1];
          for (long long p = P.start[row + cx]; p < p1; ++p) f(p);
        }
      }
    }
  }
};

__device__ __forceinline__ bool nb_before(double d, int j, double bd, int bj) { return d < bd || (d == bd && j < bj); }

// k nearest neighbours of every point (j != i, ranked by (d, j)), each row written in column order:
// cols[i*k + t], dists[i*k + t].  K >= k slots in registers, ascending by (d, j); the K - k front slots hold (-1, -1)
// sentinels, so the k-th best is always slot K - 1 and no register is indexed at run time.  (The occupancy hint for
// K <= 16 is what keeps ptxas from spilling there; K = 32 and 64 use 172 and 254 registers.)
template <int K>
__global__ void __launch_bounds__(kThreads, K <= 16 ? 4 : 1) k_nb_knn(Grid g, Points P, int n, int k, int* __restrict__ cols,
                                                      double* __restrict__ dists) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const double qx = P.x[s], qy = P.y[s], qz = P.z[s];
  const int qi = P.orig[s];
  const Walk w(g, qx, qy, qz);
  double bd[K];
  int bj[K];
#pragma unroll
  for (int t = 0; t < K; ++t) {
    const bool pad = t < K - k;
    bd[t] = pad ? -1.0 : INFINITY;
    bj[t] = pad ? -1 : INT_MAX;
  }
  for (int R = 0;; ++R) {
    w.ring(g, P, R, [&](long long p) {
      const int j = P.orig[p];
      const double d = dist(qx, qy, qz, P.x[p], P.y[p], P.z[p]);
      if (j == qi || !nb_before(d, j, bd[K - 1], bj[K - 1])) return;
      double cd = d;
      int cj = j;
#pragma unroll
      for (int t = 0; t < K; ++t) {              // insertion: the candidate bubbles into place, the last slot drops
        if (nb_before(cd, cj, bd[t], bj[t])) {
          const double td = bd[t];
          const int tj = bj[t];
          bd[t] = cd; bj[t] = cj;
          cd = td; cj = tj;
        }
      }
    });
    const double lb = w.bound(g, R);
    if (lb == INFINITY || (bj[K - 1] != INT_MAX && bd[K - 1] < lb)) break;
  }
  // bitonic sort of the slots by column; the sentinels (-1) stay in front
#pragma unroll
  for (int size = 2; size <= K; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
#pragma unroll
      for (int t = 0; t < K; ++t) {
        const int u = t ^ stride;
        if (u > t && ((bj[t] > bj[u]) == ((t & size) == 0))) {
          const double td = bd[t]; bd[t] = bd[u]; bd[u] = td;
          const int tj = bj[t]; bj[t] = bj[u]; bj[u] = tj;
        }
      }
    }
  }
  int* out_c = cols + (int64_t)qi * k;
  double* out_d = dists + (int64_t)qi * k;
#pragma unroll
  for (int t = 0; t < K; ++t) {
    if (t >= K - k) {
      out_c[t - (K - k)] = bj[t];
      out_d[t - (K - k)] = bd[t];
    }
  }
}

// Every j != i with d <= r.  Count pass (kFill false): count[i] = the row's length.  Fill pass: the row at row_off[i],
// in search order.
template <bool kFill>
__global__ void __launch_bounds__(kThreads) k_nb_radius(Grid g, Points P, int n, double r, int* __restrict__ count,
                                                         const long long* __restrict__ row_off, int* __restrict__ cols,
                                                         double* __restrict__ dists) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const double qx = P.x[s], qy = P.y[s], qz = P.z[s];
  const int qi = P.orig[s];
  const Walk w(g, qx, qy, qz);
  long long at = kFill ? row_off[qi] : 0;
  int m = 0;
  for (int R = 0;; ++R) {
    w.ring(g, P, R, [&](long long p) {
      const int j = P.orig[p];
      const double d = dist(qx, qy, qz, P.x[p], P.y[p], P.z[p]);
      if (j == qi || !(d <= r)) return;
      if (kFill) {
        cols[at] = j;
        dists[at] = d;
        ++at;
      } else {
        ++m;
      }
    });
    if (!(w.bound(g, R) <= r)) break;
  }
  if (!kFill) count[qi] = m;
}

}  // namespace nb
}  // namespace tgb
