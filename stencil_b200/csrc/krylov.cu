// Krylov vector kernels (see krylov.cuh and the sb_krylov_* entries of include/stencil_b200.h).
#include "exact_acc.cuh"
#include "krylov.cuh"

namespace sb {
namespace {

template <typename T, int N> struct KVec { using type = T; };
template <> struct KVec<float, 4> { using type = float4; };
template <> struct KVec<double, 2> { using type = double2; };

// every multiply and add of the rule rounded to nearest on its own (no FMA contraction)
__device__ __forceinline__ float t_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double t_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float t_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double t_add(double a, double b) { return __dadd_rn(a, b); }

__device__ __forceinline__ double kry_inf() { return __longlong_as_double(0x7ff0000000000000ll); }
__device__ __forceinline__ unsigned long long kry_bits(double x) { return (unsigned long long)__double_as_longlong(x); }
// sb_reduce_exact_combine's min / max, which do not depend on the order of the operands: a NaN wins (of two, the larger
// bit pattern); of +0 and -0 min takes -0 and max +0
__device__ __forceinline__ double kry_min(double a, double b) {
  if (a != a || b != b) return (a != a && b != b) ? (kry_bits(a) > kry_bits(b) ? a : b) : (a != a ? a : b);
  if (a != b) return a < b ? a : b;
  return signbit(a) ? a : b;
}
__device__ __forceinline__ double kry_max(double a, double b) {
  if (a != a || b != b) return (a != a && b != b) ? (kry_bits(a) > kry_bits(b) ? a : b) : (a != a ? a : b);
  if (a != b) return a > b ? a : b;
  return signbit(a) ? b : a;
}

struct KryAcc {
  double mn[2], mx[2];
  double f[2][kExFpe];
  ExShared *sh;
};

template <int D> __device__ __forceinline__ void kry_term(KryAcc &a, double v) {
  a.mn[D] = kry_min(a.mn[D], v);
  a.mx[D] = kry_max(a.mx[D], v);
  ex_add(a.f[D], v, a.sh, D);
}

// the buffers a mode reads and writes (bit k: buffer k); a buffer read and not written goes through the read-only cache
__host__ __device__ constexpr unsigned kry_reads(int m) {
  return m == kKryDot1 ? 3u : m == kKryDot2 ? 7u : m == kKryCopy ? 2u : m == kKryXpby ? 3u : m == kKryBicgP ? 7u : m == kKryUpdateC ? 31u : 15u;
}
__host__ __device__ constexpr unsigned kry_writes(int m) {
  return m == kKryCopy || m == kKryXpby || m == kKryBicgP ? 1u : m == kKryUpdate || m == kKryUpdateC ? 5u : 0u;
}

// N consecutive cells at byte offset `off` of every buffer: loaded, then the rule, then stored
template <typename T, int MODE, int N> struct KryChunk {
  using V = typename KVec<T, N>::type;
  T v[5][N];
  __device__ __forceinline__ void load(char *const *p, long long off) {
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      if (!((kry_reads(MODE) >> k) & 1u)) continue;
      const V *q = reinterpret_cast<const V *>(p[k] + off);
      V w;
      if ((kry_writes(MODE) >> k) & 1u)
        w = *q;
      else
        w = __ldg(q);
#pragma unroll
      for (int e = 0; e < N; ++e) v[k][e] = reinterpret_cast<const T *>(&w)[e];
    }
  }
  __device__ __forceinline__ void apply(T s, T t, KryAcc &a) {
#pragma unroll
    for (int e = 0; e < N; ++e) {
      if (MODE == kKryBicgP) {
        // p = r + T(beta) * (p - T(omega) * v)
        v[0][e] = t_add(v[1][e], t_mul(s, t_add(v[0][e], -t_mul(t, v[2][e]))));
      } else if (MODE == kKryUpdateC) {
        v[0][e] = t_add(v[0][e], t_mul(s, v[1][e]));
        v[2][e] = t_add(v[2][e], -t_mul(s, v[3][e]));
        const double r = double(v[2][e]);
        kry_term<0>(a, __dmul_rn(r, r));
        kry_term<1>(a, __dmul_rn(double(v[4][e]), r));
      } else if (MODE == kKryDot1) {
        kry_term<0>(a, __dmul_rn(double(v[0][e]), double(v[1][e])));
      } else if (MODE == kKryDot2) {
        const double x = double(v[0][e]);
        kry_term<0>(a, __dmul_rn(x, double(v[1][e])));
        kry_term<1>(a, __dmul_rn(x, double(v[2][e])));
      } else if (MODE == kKryCopy) {
        v[0][e] = v[1][e];
      } else if (MODE == kKryXpby) {
        v[0][e] = t_add(v[1][e], t_mul(s, v[0][e]));
      } else {
        v[0][e] = t_add(v[0][e], t_mul(s, v[1][e]));
        v[2][e] = t_add(v[2][e], -t_mul(s, v[3][e]));
        const double r = double(v[2][e]);
        kry_term<0>(a, __dmul_rn(r, r));
      }
    }
  }
  __device__ __forceinline__ void store(char *const *p, long long off) const {
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      if (!((kry_writes(MODE) >> k) & 1u)) continue;
      V w;
#pragma unroll
      for (int e = 0; e < N; ++e) reinterpret_cast<T *>(&w)[e] = v[k][e];
      *reinterpret_cast<V *>(p[k] + off) = w;
    }
  }
};

// The tiles of the box, any CTA any tile.  Per tile: the rows by groups of G lanes (head and tail cells one by one, the
// body in 16-byte vectors when WIDE, IF per buffer in flight per lane); with dots, the expansions merged per warp into
// the CTA's accumulator, which goes to the tile's partial with min / max and is cleared for the next tile.
template <typename T, int MODE, bool WIDE>
__global__ void __launch_bounds__(kRedThreads, 2) krylov_kernel(const KryParams P, const double s_, const double t_, KryPartial *__restrict__ part) {
  constexpr int ND = kry_dots(MODE);
  constexpr int N = WIDE ? 16 / int(sizeof(T)) : 1;
  // vectors per buffer in flight per lane: UPDATE with c holds five buffers and two accumulators, and with four it
  // would spill under the two-CTA register cap
  constexpr int IF = MODE == kKryUpdateC ? 2 : 4;
  __shared__ ExShared sh;
  __shared__ double warp_mn[2][kRedThreads / 32], warp_mx[2][kRedThreads / 32];
  if (ND) {
    for (int k = threadIdx.x; k < 2 * kExDigits; k += kRedThreads) sh.digit[k / kExDigits][k % kExDigits] = 0;
    if (threadIdx.x < 2) sh.flags[threadIdx.x] = 0;
  }
  const T s = T(s_), t = T(t_);
  const unsigned lg = unsigned(P.lg_group), G = 1u << lg;
  const unsigned lane = threadIdx.x & (G - 1), per_pass = unsigned(kRedThreads) >> lg;
  const unsigned nx = unsigned(P.ext[0]), ey = unsigned(P.ext[1]), rows = ey * unsigned(P.ext[2]);
  const unsigned wl = threadIdx.x & 31u;
  for (unsigned ti = blockIdx.x; ti < P.ntiles; ti += gridDim.x) {
    if (ND) __syncthreads(); // the accumulator is clear
    KryAcc a{{kry_inf(), kry_inf()}, {-kry_inf(), -kry_inf()}, {}, &sh};
    const unsigned r0 = ti * P.rows_per_tile, r1 = min(rows, r0 + P.rows_per_tile);
#pragma unroll 1
    for (unsigned row = r0 + (threadIdx.x >> lg); row < r1; row += per_pass) {
      const long long off = (long long)(row / ey) * P.slice + (long long)(row % ey) * P.pitch;
      char *p[5];
#pragma unroll
      for (int k = 0; k < 5; ++k) p[k] = P.buf[k] + off;
      unsigned head = 0;
      if (WIDE) {
        head = unsigned((16 - (reinterpret_cast<uintptr_t>(p[0]) & 15)) & 15) / unsigned(sizeof(T));
        head = head < nx ? head : nx;
      }
      const unsigned nvec = (nx - head) / unsigned(N);
      if (WIDE) {
#pragma unroll 1
        for (unsigned j = lane; j < head; j += G) {
          KryChunk<T, MODE, 1> c;
          c.load(p, (long long)j * sizeof(T));
          c.apply(s, t, a);
          c.store(p, (long long)j * sizeof(T));
        }
#pragma unroll 1
        for (unsigned j = head + nvec * unsigned(N) + lane; j < nx; j += G) {
          KryChunk<T, MODE, 1> c;
          c.load(p, (long long)j * sizeof(T));
          c.apply(s, t, a);
          c.store(p, (long long)j * sizeof(T));
        }
      }
      const long long body = (long long)head * sizeof(T);
#pragma unroll 1
      for (unsigned c0 = lane; c0 < nvec; c0 += unsigned(IF) * G) {
        KryChunk<T, MODE, N> c[IF];
#pragma unroll
        for (int k = 0; k < IF; ++k)
          if (c0 + unsigned(k) * G < nvec) c[k].load(p, body + (long long)(c0 + unsigned(k) * G) * (N * sizeof(T)));
#pragma unroll
        for (int k = 0; k < IF; ++k) {
          if (c0 + unsigned(k) * G < nvec) {
            c[k].apply(s, t, a);
            c[k].store(p, body + (long long)(c0 + unsigned(k) * G) * (N * sizeof(T)));
          }
        }
      }
    }
    if constexpr (ND > 0) {
#pragma unroll
      for (int d = 0; d < ND; ++d)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a.mn[d] = kry_min(a.mn[d], __shfl_down_sync(0xffffffffu, a.mn[d], o));
          a.mx[d] = kry_max(a.mx[d], __shfl_down_sync(0xffffffffu, a.mx[d], o));
        }
      ex_warp_merge(a.f[0], a.f[1], &sh, wl);
      if (0 == wl) {
#pragma unroll
        for (int d = 0; d < ND; ++d) {
          warp_mn[d][threadIdx.x >> 5] = a.mn[d];
          warp_mx[d][threadIdx.x >> 5] = a.mx[d];
#pragma unroll
          for (int i = 0; i < kExFpe; ++i) ex_add_shared(&sh, d, a.f[d][i]);
        }
      }
      __syncthreads();
      KryPartial &Q = part[ti];
      if (threadIdx.x < ND) {
        const int d = int(threadIdx.x);
        double mn = warp_mn[d][0], mx = warp_mx[d][0];
        for (int i = 1; i < kRedThreads / 32; ++i) {
          mn = kry_min(mn, warp_mn[d][i]);
          mx = kry_max(mx, warp_mx[d][i]);
        }
        Q.min[d] = mn;
        Q.max[d] = mx;
      }
      for (int k = threadIdx.x; k < ND * kExDigits; k += kRedThreads) {
        Q.digit[k / kExDigits][k % kExDigits] = (long long)sh.digit[k / kExDigits][k % kExDigits];
        sh.digit[k / kExDigits][k % kExDigits] = 0;
      }
      if (threadIdx.x < ND) {
        Q.flags[threadIdx.x] = sh.flags[threadIdx.x];
        sh.flags[threadIdx.x] = 0;
      }
    }
  }
}

// The combine, one block per dot d: the digit counters added over the tiles (each split into its low 32 bits and its
// signed high part, so every addend is below 2^32 in magnitude and 2^31 tiles cannot overflow), carried into the
// canonical sum; min / max by the order-independent rule; sumsq an exact zero.
__global__ void __launch_bounds__(kExCombineThreads) krylov_combine_kernel(const KryPartial *__restrict__ part, unsigned n, long long count,
                                                                           sb_reduce_exact_part *__restrict__ out) {
  constexpr int kCols = kExDigits, kGroups = kExCombineThreads / kCols;
  __shared__ long long lo[kGroups][kCols], hi[kGroups][kCols];
  __shared__ unsigned flags;
  __shared__ double wmn[kExCombineThreads / 32], wmx[kExCombineThreads / 32];
  const int d = int(blockIdx.x);
  if (0 == threadIdx.x) flags = 0;
  __syncthreads();
  const int col = int(threadIdx.x) % kCols, grp = int(threadIdx.x) / kCols;
  if (grp < kGroups) {
    long long l = 0, h = 0;
    unsigned f = 0;
    for (unsigned j = unsigned(grp); j < n; j += kGroups) {
      const long long x = part[j].digit[d][col];
      l += x & 0xffffffffll;
      h += x >> 32;
      if (col == 0) f |= part[j].flags[d];
    }
    lo[grp][col] = l;
    hi[grp][col] = h;
    if (col == 0) atomicOr(&flags, f);
  }
  double mn = kry_inf(), mx = -kry_inf();
  for (unsigned j = threadIdx.x; j < n; j += kExCombineThreads) {
    mn = kry_min(mn, part[j].min[d]);
    mx = kry_max(mx, part[j].max[d]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = kry_min(mn, __shfl_down_sync(0xffffffffu, mn, o));
    mx = kry_max(mx, __shfl_down_sync(0xffffffffu, mx, o));
  }
  if (0 == (threadIdx.x & 31u)) {
    wmn[threadIdx.x >> 5] = mn;
    wmx[threadIdx.x >> 5] = mx;
  }
  __syncthreads();
  sb_reduce_exact_part &o = out[d];
  if (threadIdx.x < SB_EXACT_WORDS) o.sumsq.word[threadIdx.x] = 0;
  if (0 == threadIdx.x) {
    ex_carry(lo, hi, 0, o.sum);
    o.sum.flags = flags;
    o.sumsq.flags = 0;
    for (int i = 1; i < kExCombineThreads / 32; ++i) {
      mn = kry_min(mn, wmn[i]);
      mx = kry_max(mx, wmx[i]);
    }
    o.min = n ? kry_min(mn, wmn[0]) : kry_inf();
    o.max = n ? kry_max(mx, wmx[0]) : -kry_inf();
    o.count = count;
  }
}

using KryKernel = void (*)(const KryParams, const double, const double, KryPartial *);
template <typename T, bool WIDE> KryKernel kry_kernel_of(int mode) {
  switch (mode) {
  case kKryDot1: return krylov_kernel<T, kKryDot1, WIDE>;
  case kKryDot2: return krylov_kernel<T, kKryDot2, WIDE>;
  case kKryCopy: return krylov_kernel<T, kKryCopy, WIDE>;
  case kKryXpby: return krylov_kernel<T, kKryXpby, WIDE>;
  case kKryBicgP: return krylov_kernel<T, kKryBicgP, WIDE>;
  case kKryUpdateC: return krylov_kernel<T, kKryUpdateC, WIDE>;
  default: return krylov_kernel<T, kKryUpdate, WIDE>;
  }
}
KryKernel kry_kernel(int dtype, int mode, bool wide) {
  if (dtype == SB_DTYPE_F32) return wide ? kry_kernel_of<float, true>(mode) : kry_kernel_of<float, false>(mode);
  return wide ? kry_kernel_of<double, true>(mode) : kry_kernel_of<double, false>(mode);
}

} // namespace

int krylov_grid(int device, int dtype, int mode, bool wide, unsigned ntiles) {
  return persistent_grid(device, reinterpret_cast<const void *>(kry_kernel(dtype, mode, wide)), ntiles);
}

int launch_krylov(const KryParams &p, int dtype, int mode, bool wide, int grid, double s, double t, KryPartial *scratch, sb_reduce_exact_part *out,
                  cudaStream_t stream) {
  int launches = 0;
  if (p.ntiles > 0) {
    kry_kernel(dtype, mode, wide)<<<grid, kRedThreads, 0, stream>>>(p, s, t, scratch);
    ++launches;
  }
  if (kry_dots(mode) > 0) {
    krylov_combine_kernel<<<kry_dots(mode), kExCombineThreads, 0, stream>>>(scratch, p.ntiles, p.count, out);
    ++launches;
  }
  return launches;
}

} // namespace sb
