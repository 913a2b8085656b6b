// MT19937 skip-ahead on the host: the characteristic polynomial phi of the generator's word recurrence (Berlekamp-Massey
// over its own output), jump polynomials x^J mod phi (square-and-multiply on 64-bit-word GF(2) polynomials), and their
// application to a state by Horner's rule -- the method of Haramoto, Matsumoto, Nishimura, Panneton and L'Ecuyer,
// "Efficient jump ahead for F2-linear random number generators" (INFORMS J. Computing, 2008).
//
// A state is numpy's: key[624] (the last generated block x_B .. x_B+623) and pos (the index of the next word to hand out;
// 624 = the block is used up and the next call regenerates it).  The word recurrence is
//   x_{k+624} = x_{k+397} ^ A((x_k & 0x80000000) | (x_{k+1} & 0x7fffffff))
// so the 19937 live bits of a state are the top bit of its oldest word and the 623 words after it.  A jump acts on those
// live bits only: the low 31 bits of the oldest word of a jumped window are not determined by it, and the code below
// never hands out a jumped window's oldest word without regenerating it first.
#pragma once

#include <chrono>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <vector>

namespace mtj {

constexpr int kN = 624, kM = 397;
constexpr int kDeg = 19937;                     // degree of phi
constexpr int kPolyWords = (kDeg + 63) / 64;    // 312: a polynomial of degree <= 19967, phi itself included
constexpr uint32_t kMatrixA = 0x9908b0dfu, kUpper = 0x80000000u, kLower = 0x7fffffffu;

// x_{k+624} from x_k (a), x_{k+1} (b), x_{k+397} (c)
inline uint32_t twist(uint32_t a, uint32_t b, uint32_t c) {
  const uint32_t y = (a & kUpper) | (b & kLower);
  return c ^ (y >> 1) ^ ((y & 1u) ? kMatrixA : 0u);
}

inline uint32_t temper(uint32_t y) {
  y ^= y >> 11;
  y ^= (y << 7) & 0x9d2c5680u;
  y ^= (y << 15) & 0xefc60000u;
  return y ^ (y >> 18);
}

// the next block, in place (numpy's mt19937_gen: 624 word steps with the window's oldest word at key[0])
inline void gen_block(uint32_t* key) {
  int i = 0;
  for (; i < kN - kM; ++i) key[i] = twist(key[i], key[i + 1], key[i + kM]);
  for (; i < kN - 1; ++i) key[i] = twist(key[i], key[i + 1], key[i + kM - kN]);
  key[kN - 1] = twist(key[kN - 1], key[0], key[kM - 1]);
}

inline bool coef(const uint64_t* p, int i) { return (p[i >> 6] >> (i & 63)) & 1u; }

// Polynomials of degree < kDeg in kPolyWords words, and the arithmetic modulo phi.
struct Field {
  std::vector<uint64_t> phi;              // kPolyWords words, degree kDeg
  std::vector<uint64_t> shifted;          // 64 copies of phi << s, kPolyWords + 1 words each
  double ms = 0.0;                        // host time it took to find phi

  Field() {
    const auto t0 = std::chrono::steady_clock::now();
    phi = berlekamp_massey();
    shifted.assign(64 * (kPolyWords + 1), 0);
    for (int s = 0; s < 64; ++s) {
      uint64_t* q = &shifted[s * (kPolyWords + 1)];
      for (int w = 0; w < kPolyWords; ++w) {
        q[w] ^= phi[w] << s;
        if (s) q[w + 1] ^= phi[w] >> (64 - s);
      }
    }
    ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  }

  // phi from 2 * kDeg output bits (bit 0 of the words x_624, x_625, ... of the generator seeded with 5489).  The
  // recurrence's characteristic polynomial is primitive, so every nonzero bit sequence it produces has phi as its
  // minimal polynomial; Berlekamp-Massey finds the connection polynomial C(x) = x^kDeg phi(1/x).
  static std::vector<uint64_t> berlekamp_massey() {
    const int n2 = 2 * kDeg;
    const int nw = n2 / 64 + 4;
    uint32_t key[kN];
    uint32_t seed = 5489u;                          // numpy's mt19937_seed
    for (int i = 0; i < kN; ++i) {
      key[i] = seed;
      seed = 1812433253u * (seed ^ (seed >> 30)) + (uint32_t)i + 1u;
    }
    std::vector<uint64_t> r(nw, 0);                 // the sequence reversed: bit j is s_{n2-1-j}
    for (int k = 0; k < n2; ++k) {
      if (k % kN == 0) gen_block(key);
      const int j = n2 - 1 - k;
      r[j >> 6] |= (uint64_t)(key[k % kN] & 1u) << (j & 63);
    }
    std::vector<uint64_t> C(nw, 0), B(nw, 0), T;
    C[0] = B[0] = 1;
    int L = 0, m = 1;
    for (int n = 0; n < n2; ++n) {
      // discrepancy: sum_{i=0..L} c_i s_{n-i} = sum_i c_i r_{base+i}
      const int base = n2 - 1 - n, w0 = base >> 6, sh = base & 63;
      uint64_t acc = 0;
      for (int w = 0; w <= L / 64; ++w) {
        uint64_t rw = r[w0 + w] >> sh;
        if (sh) rw |= r[w0 + w + 1] << (64 - sh);
        acc ^= C[w] & rw;
      }
      if (!(__builtin_popcountll(acc) & 1)) { ++m; continue; }
      const bool grow = 2 * L <= n;
      if (grow) T = C;
      const int ws = m >> 6, bs = m & 63;            // C ^= B << m
      for (int w = 0; w + ws < nw; ++w) {
        if (!B[w]) continue;
        C[w + ws] ^= B[w] << bs;
        if (bs && w + ws + 1 < nw) C[w + ws + 1] ^= B[w] >> (64 - bs);
      }
      if (grow) { L = n + 1 - L; B.swap(T); m = 1; } else { ++m; }
    }
    std::vector<uint64_t> p(kPolyWords, 0);
    if (L != kDeg) return {};                        // cannot happen for MT19937; the caller checks
    for (int i = 0; i <= L; ++i)
      if (coef(C.data(), L - i)) p[i >> 6] |= 1ull << (i & 63);
    return p;
  }

  bool ok() const { return !phi.empty(); }

  // p (2 * kPolyWords + 2 words, degree < 2 kDeg) mod phi, in place
  void reduce(uint64_t* p) const {
    for (int w = 2 * kPolyWords - 1; w >= kDeg / 64; --w) {
      for (;;) {
        uint64_t v = p[w];
        if (w == kDeg / 64) v &= ~0ull << (kDeg & 63);
        if (!v) break;
        const int s = w * 64 + (63 - __builtin_clzll(v)) - kDeg;
        const uint64_t* q = &shifted[(s & 63) * (kPolyWords + 1)];
        uint64_t* d = p + (s >> 6);
        for (int k = 0; k < kPolyWords + 1; ++k) d[k] ^= q[k];
      }
    }
  }

  void square(std::vector<uint64_t>& a) const {
    std::vector<uint64_t> t(2 * kPolyWords + 2, 0);
    for (int w = 0; w < kPolyWords; ++w) {
      t[2 * w] = spread((uint32_t)a[w]);
      t[2 * w + 1] = spread((uint32_t)(a[w] >> 32));
    }
    reduce(t.data());
    a.assign(t.begin(), t.begin() + kPolyWords);
  }

  void times_x(std::vector<uint64_t>& a) const {
    for (int w = kPolyWords - 1; w > 0; --w) a[w] = (a[w] << 1) | (a[w - 1] >> 63);
    a[0] <<= 1;
    if (coef(a.data(), kDeg))
      for (int w = 0; w < kPolyWords; ++w) a[w] ^= phi[w];
  }

  // x^J mod phi
  std::vector<uint64_t> x_pow(unsigned __int128 J) const {
    std::vector<uint64_t> a(kPolyWords, 0);
    a[0] = 1;
    int b = 127;
    while (b >= 0 && !((J >> b) & 1u)) --b;
    for (; b >= 0; --b) {
      square(a);
      if ((J >> b) & 1u) times_x(a);
    }
    return a;
  }

  static uint64_t spread(uint32_t v) {
    uint64_t x = v;
    x = (x | (x << 16)) & 0x0000ffff0000ffffull;
    x = (x | (x << 8)) & 0x00ff00ff00ff00ffull;
    x = (x | (x << 4)) & 0x0f0f0f0f0f0f0f0full;
    x = (x | (x << 2)) & 0x3333333333333333ull;
    x = (x | (x << 1)) & 0x5555555555555555ull;
    return x;
  }
};

// computed once per process, on first use
inline const Field& field() {
  static const Field f;
  return f;
}

// Horner: out = p(F) s, F the single word step, s and out windows with their oldest word at index 0.
inline void horner(const uint64_t* p, const uint32_t* s, uint32_t* out) {
  uint32_t acc[kN] = {0};
  int a = 0;                                      // index of acc's oldest word (acc is circular)
  int top = kDeg - 1;
  while (top >= 0 && !coef(p, top)) --top;
  for (int i = top; i >= 0; --i) {
    const int a1 = a + 1 == kN ? 0 : a + 1, am = a + kM >= kN ? a + kM - kN : a + kM;
    acc[a] = twist(acc[a], acc[a1], acc[am]);
    a = a1;
    if (coef(p, i)) {
      for (int k = 0; k < kN - a; ++k) acc[a + k] ^= s[k];
      for (int k = kN - a; k < kN; ++k) acc[a + k - kN] ^= s[k];
    }
  }
  for (int k = 0; k < kN; ++k) out[k] = acc[(a + k) % kN];
}

// The state after n = n_minus_1 + 1 more words (1 <= n <= 2^128): (key, pos) as numpy's MT19937 holds it after
// random_raw(n).  pos is 0 .. 624; the result's pos is 1 .. 624.
inline void jump(const uint32_t* key, int pos, unsigned __int128 n_minus_1, uint32_t* key_out, int* pos_out) {
  if (n_minus_1 < (unsigned)(kN - pos)) {         // no regeneration on the way
    std::memmove(key_out, key, kN * sizeof(uint32_t));
    *pos_out = pos + (int)n_minus_1 + 1;
    return;
  }
  // The last of the g >= 1 regenerated blocks is B + g with pos + n = 624 g + pos'.  The window at the start of
  // block B + g - 1 is J = 624 (g - 1) = n - 624 - pos' + pos words on; one regeneration from there makes every word
  // of block B + g exact.
  const int pos1 = (int)((pos + (int)(n_minus_1 % kN)) % kN) + 1;
  const unsigned __int128 J = n_minus_1 - (unsigned)(kN - 1 + pos1 - pos);
  uint32_t tmp[kN];
  if (J) horner(field().x_pow(J).data(), key, tmp);
  else std::memcpy(tmp, key, sizeof(tmp));
  gen_block(tmp);
  std::memcpy(key_out, tmp, sizeof(tmp));
  *pos_out = pos1;
}

}  // namespace mtj
