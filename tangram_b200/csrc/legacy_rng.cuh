// numpy's legacy normal stream (np.random.seed + np.random.normal, RandomState's polar method on MT19937) drawn on the
// device, bit-identical to the host draw it replaces (reference mapping_optimizer.py:147-157).
//
// Attempt a of the polar method consumes words 4a .. 4a+3 of the MT19937 output stream (counted from numpy's `pos`):
//   d = ((w0 >> 5) * 2^26 + (w1 >> 6)) / 2^53, likewise from w2, w3;  x = 2 d - 1;  r2 = x1 x1 + x2 x2
// and is accepted if 0 < r2 < 1; accepted attempt number k then yields normals 2k and 2k+1 (after a cached one):
// f x2 and f x1 with f = sqrt(-2 log(r2) / r2).  Everything up to the acceptance test is exact, so which attempts are
// accepted is pure integer arithmetic on the words and parallelises as a prefix count:
//   jump   block start states: the stream is cut into draw blocks of kWordsPerCta words (kBlocksPerCta MT19937
//          blocks); k_mt_jump applies jump polynomials x^J mod phi (mt19937_jump.h) to whole 624-word windows
//   count  k_legacy_pass<false>: each CTA regenerates its block's words and counts the accepted attempts
//   scan   k_scan_counts: exclusive prefix of the counts
//   emit   k_legacy_pass<true>: regenerate again, rank each accepted attempt, write float32(f x2), float32(f x1)
// The only inexact step is log: CUDA's and glibc's may differ in the last bit, so values whose fp64 result lies close
// to a float32 rounding midpoint are flagged and recomputed on the host with libm (tgb200_init_mapping_legacy).
#pragma once
#include "common.cuh"

namespace tgb {
namespace lrng {

constexpr int kN = 624, kM = 397;
constexpr int kBlocksPerCta = 512;                               // MT19937 blocks per draw block
constexpr long long kWordsPerCta = (long long)kN * kBlocksPerCta;
constexpr int kAttemptsPerMt = kN / 4;                           // 156
constexpr long long kAttemptsPerCta = kWordsPerCta / 4;
constexpr int kPolyWords = 312;                                  // x^J mod phi: degree < 19937
constexpr int kSeqWords = kPolyWords * 64 + kN;                  // k_mt_jump's output sequence x_0 .. x_{19967+623}
constexpr size_t kJumpSmem = kSeqWords * sizeof(uint32_t);
// A value is recomputed on the host when its fp64 result is within this many fp64 ulps of a float32 rounding
// midpoint (the 29 low mantissa bits against 2^28).  Derivation: CUDA's log (max 1 ulp) and glibc's log (< 1 ulp)
// differ by at most 2 ulp, i.e. 2^-51 relative.  -2 log is exact; the correctly rounded /r2 adds 2^-53 on each side
// (relative difference < 1.5 * 2^-51); sqrt halves that and adds 2^-53 per side (< 1.25 * 2^-51); the product with x
// adds 2^-53 per side: |v_dev - v_host| < 1.75 * 2^-51 |v| < 2^-50 |v|.  With 2^e <= |v| < 2^(e+1) an fp64 ulp is
// 2^(e-52), so the two values are less than 8 ulps apart; the float32 results can only differ if a midpoint lies
// between them.  32 keeps a 4x margin.  |v| >= 2^-78 (|x| >= 2^-52, f > 2^-26), far above float32's subnormals, so the
// 29-bit rule holds for every nonzero value.
constexpr long long kFlagUlps = 32;

struct Flagged { long long idx; uint32_t w[4]; int comp; int pad; };   // comp 0: f x2, 1: f x1
struct EndRecord { long long attempt; uint32_t w[4]; };

__host__ __device__ __forceinline__ uint32_t twist(uint32_t a, uint32_t b, uint32_t c) {
  const uint32_t y = (a & 0x80000000u) | (b & 0x7fffffffu);
  return c ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}

__device__ __forceinline__ uint32_t temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  return y ^ (y >> 18);
}

// numpy's mt19937_gen over a CTA of 624 threads, in place: the twist's three dependency phases (i < 227 reads the old
// block only; 227 <= i < 454 reads new words i - 227; the rest reads new words i - 227 and, for i = 623, new word 0)
__device__ __forceinline__ void gen_block(uint32_t* key, int i) {
  uint32_t v = 0;
  if (i < kN - kM) v = twist(key[i], key[i + 1], key[i + kM]);
  __syncthreads();
  if (i < kN - kM) key[i] = v;
  __syncthreads();
  if (i >= kN - kM && i < 2 * (kN - kM)) v = twist(key[i], key[i + 1], key[i + kM - kN]);
  __syncthreads();
  if (i >= kN - kM && i < 2 * (kN - kM)) key[i] = v;
  __syncthreads();
  if (i >= 2 * (kN - kM)) v = twist(key[i], key[i == kN - 1 ? 0 : i + 1], key[i + kM - kN]);
  __syncthreads();
  if (i >= 2 * (kN - kM)) key[i] = v;
  __syncthreads();
}

// dst[s] = p(F) src[s] for s < count (F: one word step; windows with their oldest word first), one CTA of 624 threads
// per state.  The CTA writes the output sequence x_0, x_1, ... of src into shared memory (227 new words per round:
// x_{k+624} needs x_{k+397}) and thread j forms word j of the result as XOR of x_{i+j} over the coefficients c_i = 1:
// the sum Horner's rule evaluates, without its 19937 serial steps.
__global__ void __launch_bounds__(kN) k_mt_jump(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst,
                                                const uint64_t* __restrict__ poly) {
  extern __shared__ uint32_t x[];
  __shared__ uint64_t pc[kPolyWords];
  const int j = threadIdx.x;
  x[j] = src[(size_t)blockIdx.x * kN + j];
  if (j < kPolyWords) pc[j] = poly[j];
  __syncthreads();
  for (int c = 0; c + kN < kSeqWords; c += kN - kM) {
    const int k = c + j;
    if (j < kN - kM && k + kN < kSeqWords) x[k + kN] = twist(x[k], x[k + 1], x[k + kM]);
    __syncthreads();
  }
  uint32_t acc = 0;
  for (int w = 0; w < kPolyWords; ++w) {
    uint64_t bits = pc[w];
    const uint32_t* xs = x + w * 64 + j;
    while (bits) {
      acc ^= xs[__ffsll((long long)bits) - 1];
      bits &= bits - 1;
    }
  }
  dst[(size_t)blockIdx.x * kN + j] = acc;
}

struct DrawParams {
  const uint32_t* key0;        // numpy's key: block B, exact
  const uint32_t* starts;      // starts[b] (b >= 1): window at the start of MT block B + b kBlocksPerCta - 1
  int pos0;                    // numpy's pos: the stream starts at word pos0 of block B (624: at block B + 1)
  int b_first;                 // draw block of CTA 0
  long long* counts;           // count pass: accepted attempts per draw block
  const long long* offs;       // emit pass: accepted attempts before each draw block
  long long t_lo, t_hi;        // stream normals written: [t_lo, t_hi) -> M element t - t_lo
  int has_gauss;               // normal 0 is numpy's cached value (written by the host)
  int V, ld;
  float* M;                    // elements [0, split) of the mapping (row * ld + column)
  float* Mh;                   // elements from split on (host state: rows [R, N) in pinned host memory)
  long long split;
  long long a_end;             // accepted attempt that ends the draw: its attempt index and words go to *end
  EndRecord* end;
  Flagged* flags;
  int* n_flags;
  int flag_cap;
};

// Draw block b = b_first + blockIdx.x covers stream words [pos0 + b L, pos0 + (b+1) L) of block B's start, L a
// multiple of 4, so no attempt straddles two CTAs: MT blocks k = 0 .. kBlocksPerCta of the CTA, attempts t >= pos0/4
// of block 0 and t < pos0/4 of block kBlocksPerCta.  An attempt may reach up to 3 words into the next MT block;
// those words depend on the current block only and are computed next to it.
template <bool kEmit>
__global__ void __launch_bounds__(kN) k_legacy_pass(DrawParams p) {
  __shared__ uint32_t key[kN];
  __shared__ uint32_t tw[kN + 4];
  __shared__ int wsum[5];
  __shared__ int cta_count;
  const int i = threadIdx.x;
  const int b = p.b_first + blockIdx.x;
  const int t0 = p.pos0 >> 2, off = p.pos0 & 3;
  key[i] = b == 0 ? p.key0[i] : p.starts[(size_t)b * kN + i];
  if (i == 0) cta_count = 0;
  __syncthreads();
  if (b != 0) gen_block(key, i);                       // the jumped window's oldest word is not exact: regenerate
  long long base = kEmit ? p.offs[b] : 0;               // accepted attempts before the current MT block
  const long long attempt0 = (long long)b * kAttemptsPerCta - t0;   // attempt index of (MT block 0, t = 0)
  int cnt = 0;
  const int k_last = t0 ? kBlocksPerCta : kBlocksPerCta - 1;
  for (int k = 0; k <= k_last; ++k) {
    tw[i] = temper(key[i]);
    if (i < 3) tw[kN + i] = temper(twist(key[i], key[i + 1], key[i + kM]));
    __syncthreads();
    const int lo = k == 0 ? t0 : 0, hi = k == kBlocksPerCta ? t0 : kAttemptsPerMt;
    bool acc = false;
    double x1 = 0.0, x2 = 0.0, r2 = 0.0;
    if (i >= lo && i < hi) {
      const uint32_t* w = tw + off + 4 * i;
      const double d1 = __ddiv_rn(__dadd_rn(__dmul_rn((double)(w[0] >> 5), 67108864.0), (double)(w[1] >> 6)),
                                  9007199254740992.0);
      const double d2 = __ddiv_rn(__dadd_rn(__dmul_rn((double)(w[2] >> 5), 67108864.0), (double)(w[3] >> 6)),
                                  9007199254740992.0);
      x1 = __dadd_rn(__dmul_rn(2.0, d1), -1.0);
      x2 = __dadd_rn(__dmul_rn(2.0, d2), -1.0);
      r2 = __dadd_rn(__dmul_rn(x1, x1), __dmul_rn(x2, x2));      // no FMA: numpy rounds both products
      acc = r2 < 1.0 && r2 != 0.0;
    }
    if (!kEmit) {
      cnt += acc;
    } else {
      unsigned bal = 0;
      const int lane = i & 31, warp = i >> 5;
      if (i < 160) bal = __ballot_sync(0xffffffffu, acc);          // attempts live in warps 0..4
      if (i < 160 && lane == 0) wsum[warp] = __popc(bal);
      __syncthreads();
      int before = 0, total = 0;
#pragma unroll
      for (int w = 0; w < 5; ++w) {
        before += w < warp ? wsum[w] : 0;
        total += wsum[w];
      }
      if (acc) {
        const long long a = base + before + __popc(bal & ((1u << lane) - 1u));
        const long long t = p.has_gauss + 2 * a;                   // normals t (f x2) and t + 1 (f x1)
        const uint32_t* w = tw + off + 4 * i;
        if (a == p.a_end) {
          p.end->attempt = attempt0 + 156LL * k + i;
          for (int q = 0; q < 4; ++q) p.end->w[q] = w[q];
        }
        if (t + 1 >= p.t_lo && t < p.t_hi) {
          const double f = __dsqrt_rn(__ddiv_rn(__dmul_rn(-2.0, log(r2)), r2));
#pragma unroll
          for (int comp = 0; comp < 2; ++comp) {
            const long long tc = t + comp;
            if (tc < p.t_lo || tc >= p.t_hi) continue;
            const double v = __dmul_rn(f, comp ? x1 : x2);
            const long long e = tc - p.t_lo, row = e / p.V;
            const long long idx = row * p.ld + (e - row * p.V);
            (idx < p.split ? p.M + idx : p.Mh + (idx - p.split))[0] = __double2float_rn(v);
            const long long low = __double_as_longlong(v) & ((1LL << 29) - 1);
            if (llabs(low - (1LL << 28)) <= kFlagUlps) {
              const int slot = atomicAdd(p.n_flags, 1);
              if (slot < p.flag_cap) {
                Flagged& fl = p.flags[slot];
                fl.idx = idx;
                fl.comp = comp;
                for (int q = 0; q < 4; ++q) fl.w[q] = w[q];
              }
            }
          }
        }
      }
      base += total;
    }
    if (k < k_last) {
      __syncthreads();                                  // tw and wsum are read; the twist may overwrite key
      gen_block(key, i);
    }
  }
  if (!kEmit) {
    if (cnt) atomicAdd(&cta_count, cnt);                // integer sum: the order does not matter
    __syncthreads();
    if (i == 0) p.counts[b] = cta_count;
  }
}

// offs[b] = sum of counts[c] for c < b, offs[n] = the total.  One CTA: each thread sums a contiguous run, thread 0
// scans the run totals, each thread writes its run.  Integer sums: the result does not depend on the launch shape.
__global__ void __launch_bounds__(1024) k_scan_counts(const long long* __restrict__ counts, int n,
                                                      long long* __restrict__ offs) {
  __shared__ long long part[1024];
  const int per = (n + blockDim.x - 1) / blockDim.x;
  const int lo = min(n, (int)threadIdx.x * per), hi = min(n, lo + per);
  long long s = 0;
  for (int b = lo; b < hi; ++b) s += counts[b];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long run = 0;
    for (unsigned t = 0; t < blockDim.x; ++t) {
      const long long v = part[t];
      part[t] = run;
      run += v;
    }
    offs[n] = run;
  }
  __syncthreads();
  s = part[threadIdx.x];
  for (int b = lo; b < hi; ++b) {
    offs[b] = s;
    s += counts[b];
  }
}

}  // namespace lrng
}  // namespace tgb
