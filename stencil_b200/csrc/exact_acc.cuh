// The exact accumulator of the exact reductions (DESIGN.md section 2.6.1), shared by reduce_exact.cu and krylov.cu.
//
// A thread keeps, per sum, a floating-point expansion of kExFpe doubles grown by TwoSum (ex_add); what does not fit goes
// to the CTA's fixed-point accumulator ExShared by 64-bit shared atomics (ex_add_shared).  At the end of a tile each warp
// merges its 32 expansions into lane 0 (ex_warp_merge), which adds them to the accumulator; the tile's counters are then
// summed over the tiles of an item and carried into the canonical sb_exact_sum words (ex_carry).
#pragma once

#include "reduce.cuh"

namespace sb {

struct ExShared {
  unsigned long long digit[2][kExDigits]; // int64 counters of 32-bit digits, added to modulo 2^64
  unsigned flags[2];
};

// Adds the double t exactly to accumulator w of the CTA: inf and NaN set flags; a finite t = m * 2^(p - 1074) (m < 2^53)
// is m << (p mod 32), at most 85 bits, added as three unsigned 32-bit chunks (negated for t < 0) to digits p / 32 ...
__device__ __forceinline__ void ex_add_shared(ExShared *sh, int w, double t) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(t);
  const unsigned ex = unsigned(b >> 52) & 0x7ffu;
  const unsigned long long frac = b & ((1ull << 52) - 1);
  if (ex == 0x7ffu) {
    atomicOr(&sh->flags[w], frac ? SB_EXACT_NAN : (b >> 63) ? SB_EXACT_NEG_INF : SB_EXACT_POS_INF);
    return;
  }
  const unsigned long long m = ex ? frac | (1ull << 52) : frac;
  if (!m) return;
  const unsigned p = ex ? ex - 1 : 0, s = p & 31u, d = p >> 5;
  const unsigned long long lo = m << s, hi = s ? m >> (64u - s) : 0ull;
  const unsigned long long neg = (b >> 63) ? ~0ull : 0ull; // c -> (c ^ neg) - neg negates for t < 0
  unsigned long long *dg = sh->digit[w] + d;
  atomicAdd(dg, ((lo & 0xffffffffull) ^ neg) - neg);
  atomicAdd(dg + 1, ((lo >> 32) ^ neg) - neg);
  if (hi) atomicAdd(dg + 2, (hi ^ neg) - neg);
}

// t into the expansion f by TwoSum, level by level; the last error term, a term of magnitude >= 2^990 (the levels then
// stay below 2^1018 for any chain a tile makes, so no TwoSum overflows), inf and NaN go to the CTA's accumulator.
__device__ __forceinline__ void ex_add(double (&f)[kExFpe], double t, ExShared *sh, int w) {
  if (!(fabs(t) < 0x1p990)) {
    ex_add_shared(sh, w, t);
    return;
  }
#pragma unroll
  for (int i = 0; i < kExFpe; ++i) {
    const double s = __dadd_rn(f[i], t);
    const double bp = __dadd_rn(s, -f[i]);
    const double e = __dadd_rn(__dadd_rn(f[i], -__dadd_rn(s, -bp)), __dadd_rn(t, -bp));
    f[i] = s;
    t = e;
  }
  if (t != 0.0) ex_add_shared(sh, w, t);
}

// The expansions fa (accumulator 0) and fb (accumulator 1) of a warp merged into lane 0's: lane l + o into lane l for
// (l mod 2o) == 0 (exact in any order).  Every lane of the warp calls it.
__device__ __forceinline__ void ex_warp_merge(double (&fa)[kExFpe], double (&fb)[kExFpe], ExShared *sh, unsigned lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    double gv[kExFpe], gq[kExFpe];
#pragma unroll
    for (int i = 0; i < kExFpe; ++i) {
      gv[i] = __shfl_down_sync(0xffffffffu, fa[i], o);
      gq[i] = __shfl_down_sync(0xffffffffu, fb[i], o);
    }
    if (0 == (lane & unsigned(2 * o - 1))) {
#pragma unroll
      for (int i = 0; i < kExFpe; ++i) {
        ex_add(fa, gv[i], sh, 0);
        ex_add(fb, gq[i], sh, 1);
      }
    }
  }
}

// Accumulator w's digit counters, summed over the tiles as kGroups partial sums of their low 32 bits (lo) and of their
// signed high parts (hi), carried into the canonical two's complement words of e (flags are the caller's).
template <int kGroups, int kCols>
__device__ __forceinline__ void ex_carry(const long long (&lo)[kGroups][kCols], const long long (&hi)[kGroups][kCols], int w, sb_exact_sum &e) {
  __int128 c = 0;
  unsigned long long word = 0;
  for (int k = 0; k < kExDigits; ++k) {
    __int128 v = c;
    for (int g = 0; g < kGroups; ++g) v += __int128(lo[g][w * kExDigits + k]) + (k ? __int128(hi[g][w * kExDigits + k - 1]) : 0);
    const unsigned long long d = (unsigned long long)(v & 0xffffffff);
    c = v >> 32;
    word = (k & 1) ? word | (d << 32) : d;
    if (k & 1) e.word[k >> 1] = word;
  }
}

} // namespace sb
