// Handle-free projection out = map^T X (tangram/utils.py:366-368) from a CSR X: one block of CSR rows straight into the
// three bf16 planes (hi + mid + lo, split3) that the split-bf16 forward contraction reads, with no fp32 dense slab in
// between.  A dense row block goes through k_split3 instead; both give the same planes for the same values.
#pragma once
#include "common.cuh"
#include "kernels_elem.cuh"   // Split3, split3

namespace tgb {

constexpr int kProjThreads = 256;

struct CsrSplitArgs {
  const int64_t* indptr;    // nb + 1 row offsets of this block, absolute (the block's entries start at indptr[0])
  const int* indices;       // the block's entries
  const float* data;
  int nb;                   // rows that hold entries
  int rows;                 // rows written: [nb, rows) become zero (the ragged tail of the last 64-row k-block)
  int n_genes;
  int ldx;                  // row pitch of the planes, a multiple of 64
  Split3 dst;
  int* bad;                 // set to 1 on a column outside [0, n_genes) or not strictly increasing within its row
};

// One warp per row: zero the row in all three planes, then scatter its entries.  A rejected entry is skipped, so nothing
// is written out of bounds, and raises the flag; no two lanes write the same element (columns strictly increase).
__global__ void __launch_bounds__(kProjThreads) k_csr_split3(CsrSplitArgs a) {
  const int r = (int)(((long long)blockIdx.x * kProjThreads + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= a.rows) return;
  const size_t row = (size_t)r * a.ldx;
  const uint4 z = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
  for (int pl = 0; pl < 3; ++pl) {
    uint4* dst = reinterpret_cast<uint4*>(a.dst.base + pl * a.dst.plane + row);
    for (int q = lane; q < a.ldx / 8; q += kWarp) dst[q] = z;
  }
  if (r >= a.nb) return;
  __syncwarp();                                       // the row's zeros land before its entries
  const int64_t base = a.indptr[0], p0 = a.indptr[r] - base, p1 = a.indptr[r + 1] - base;
  for (int64_t p = p0 + lane; p < p1; p += kWarp) {
    const int c = a.indices[p];
    if (c < 0 || c >= a.n_genes || (p > p0 && a.indices[p - 1] >= c)) { *a.bad = 1; continue; }
    __nv_bfloat16 h, m, l;
    split3(a.data[p], h, m, l);
    a.dst.base[row + c] = h;
    a.dst.base[a.dst.plane + row + c] = m;
    a.dst.base[2 * a.dst.plane + row + c] = l;
  }
}

}  // namespace tgb
