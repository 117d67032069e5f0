// The row walk of the reduction tile kernels, shared by reduce.cu (ordered sums) and reduce_exact.cu (exact sums).
// Included inside namespace sb::{anonymous} after the including file has declared its per-thread accumulator A and
// add<KIND>(A &, x, y, z), which takes one cell's widened source values.
#pragma once

template <typename T, int N> struct Vec { using type = T; };
template <> struct Vec<float, 4> { using type = float4; };
template <> struct Vec<double, 2> { using type = double2; };

__device__ __forceinline__ double pos_inf() { return __longlong_as_double(0x7ff0000000000000ll); }

template <int KIND> __host__ __device__ constexpr int num_sources() { return KIND == SB_REDUCE_SCALAR ? 1 : KIND == SB_REDUCE_DIFF ? 2 : 3; }

template <typename T, int KIND, typename A> __device__ __forceinline__ void add_cell(A &a, const char *const *p, unsigned j) {
  constexpr int NS = num_sources<KIND>();
  double x[3] = {0, 0, 0};
#pragma unroll
  for (int s = 0; s < NS; ++s) x[s] = double(__ldg(reinterpret_cast<const T *>(p[s]) + j));
  add<KIND>(a, x[0], x[1], x[2]);
}

// The rows of one tile.  WIDE: cells [0, head) and [tail0, nx) of a row are read one by one (head brings the address to
// a 16-byte boundary), the body in 16-byte vectors; otherwise every access is one element.  Lane l of a row's group
// reads head / tail cells l, l + G, ... and body vectors l, l + G, ..., four per source in flight.  A is the per-thread
// accumulator: Acc (the ordered chains) or ExAcc (exact sums).
template <typename T, int KIND, bool WIDE, typename A> __device__ void reduce_rows(const RedItem &it, const RedTile &t, A &a) {
  constexpr int NS = num_sources<KIND>();
  constexpr int N = WIDE ? 16 / int(sizeof(T)) : 1;
  using V = typename Vec<T, N>::type;
  const unsigned lg = unsigned(it.lg_group), G = 1u << lg;
  const unsigned lane = threadIdx.x & (G - 1), per_pass = unsigned(kRedThreads) >> lg;
  const unsigned nx = unsigned(it.ext[0]), ey = unsigned(it.ext[1]);
#pragma unroll 1
  for (unsigned r = threadIdx.x >> lg; r < t.nrows; r += per_pass) {
    const unsigned row = t.row0 + r;
    const long long off = (long long)(row / ey) * it.slice + (long long)(row % ey) * it.pitch;
    const char *p[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) p[s] = it.src[s] + off;
    unsigned head = 0;
    if (WIDE) {
      head = unsigned((16 - (reinterpret_cast<uintptr_t>(p[0]) & 15)) & 15) / unsigned(sizeof(T));
      head = head < nx ? head : nx;
    }
    const unsigned nvec = (nx - head) / unsigned(N);
    if (WIDE) {
#pragma unroll 1
      for (unsigned j = lane; j < head; j += G) add_cell<T, KIND, A>(a, p, j);
#pragma unroll 1
      for (unsigned j = head + nvec * unsigned(N) + lane; j < nx; j += G) add_cell<T, KIND, A>(a, p, j);
    }
    const V *vp[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) vp[s] = reinterpret_cast<const V *>(p[s] + size_t(head) * sizeof(T));
#pragma unroll 1
    for (unsigned c = lane; c < nvec; c += 4 * G) {
      V w[4][NS];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const unsigned i = c + unsigned(k) * G;
#pragma unroll
        for (int s = 0; s < NS; ++s)
          if (i < nvec) w[k][s] = __ldg(vp[s] + i);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (c + unsigned(k) * G < nvec) {
#pragma unroll
          for (int e = 0; e < N; ++e) {
            double x[3] = {0, 0, 0};
#pragma unroll
            for (int s = 0; s < NS; ++s) x[s] = double(reinterpret_cast<const T *>(&w[k][s])[e]);
            add<KIND>(a, x[0], x[1], x[2]);
          }
        }
      }
    }
  }
}

