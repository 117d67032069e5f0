// Boundary-condition fill kernel (see boundary.cuh and the sb_bc_* entries of include/stencil_b200.h).
#include "boundary.cuh"

#include <cstring>
#include <type_traits>

namespace sb {
namespace {

template <int V> struct Word;
template <> struct Word<1> { using type = unsigned char; };
template <> struct Word<2> { using type = unsigned short; };
template <> struct Word<4> { using type = unsigned; };
template <> struct Word<8> { using type = uint2; };
template <> struct Word<16> { using type = uint4; };

struct Raw {}; // element type of a RAW quantity: bytes are copied, no arithmetic

// the operations of the wall faces on one cell, in the quantity's own type
template <typename T> __device__ __forceinline__ T chain(T v, const BcSeg &g) {
  if (!g.read) v = T(g.value0);
  for (int k = 0; k < g.nops; ++k) v = T(g.twoc[k]) - v;
  return v;
}

template <typename T, int V> __device__ __forceinline__ void apply_word(typename Word<V>::type &w, const BcSeg &g) {
  if constexpr (!std::is_same<T, Raw>::value && V >= int(sizeof(T))) {
    T t[V / sizeof(T)];
    memcpy(t, &w, V);
#pragma unroll
    for (int i = 0; i < V / int(sizeof(T)); ++i) t[i] = chain(t[i], g);
    memcpy(&w, t, V);
  }
}

// Row segments: ghost row (y, z) is source row (y', z') over the same x range.  A group of 2^lg_group lanes shares a row,
// each lane keeps four V-byte accesses in flight.
template <typename T, int V> __device__ void fill_rows(const BcSeg &g, const BcTile &t) {
  using W = typename Word<V>::type;
  const unsigned lg = g.lg_group, G = 1u << lg;
  const unsigned lane = threadIdx.x & (G - 1), per_pass = blockDim.x >> lg;
  const unsigned nvec = unsigned(g.ext[0]) * g.es / unsigned(V);
  const unsigned ey = unsigned(g.ext[1]);
  for (unsigned r = threadIdx.x >> lg; r < t.nrows; r += per_pass) {
    const unsigned row = t.row0 + r;
    const int py = g.pos[1] + int(row % ey), pz = g.pos[2] + int(row / ey);
    const int sy = g.mirror[1] >= 0 ? g.mirror[1] - py : py;
    const int sz = g.mirror[2] >= 0 ? g.mirror[2] - pz : pz;
    const long long x0 = (long long)g.pos[0] * g.es;
    char *d = g.base + pz * g.slice + py * g.pitch + x0;
    const char *s = g.base + sz * g.slice + sy * g.pitch + x0;
    for (unsigned c = lane; c < nvec; c += 4 * G) {
      W w[4] = {};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const unsigned i = c + unsigned(k) * G;
        if (g.read && i < nvec) w[k] = *reinterpret_cast<const W *>(s + size_t(i) * V);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const unsigned i = c + unsigned(k) * G;
        if (i < nvec) {
          apply_word<T, V>(w[k], g);
          *reinterpret_cast<W *>(d + size_t(i) * V) = w[k];
        }
      }
    }
  }
}

template <typename T> __device__ void fill_rows_any(const BcSeg &g, const BcTile &t) {
  switch (g.vec) {
  case 16: fill_rows<T, 16>(g, t); break;
  case 8: fill_rows<T, 8>(g, t); break;
  case 4: fill_rows<T, 4>(g, t); break;
  case 2: fill_rows<T, 2>(g, t); break;
  default: fill_rows<T, 1>(g, t); break;
  }
}

// Mirrored rows (a wall on x): ghost cell x of row (y, z) reads cell mirror.x - x of source row (y', z').  One lane per
// row; the row's (at most a few) loads are issued before its stores.
template <typename T, typename E> __device__ void fill_xrows(const BcSeg &g, const BcTile &t) {
  const unsigned ey = unsigned(g.ext[1]);
  const int nx = g.ext[0];
  for (unsigned r = threadIdx.x; r < t.nrows; r += blockDim.x) {
    const unsigned row = t.row0 + r;
    const int py = g.pos[1] + int(row % ey), pz = g.pos[2] + int(row / ey);
    const int sy = g.mirror[1] >= 0 ? g.mirror[1] - py : py;
    const int sz = g.mirror[2] >= 0 ? g.mirror[2] - pz : pz;
    E *d = reinterpret_cast<E *>(g.base + pz * g.slice + py * g.pitch);
    const E *s = reinterpret_cast<const E *>(g.base + sz * g.slice + sy * g.pitch);
    for (int x = 0; x < nx; x += 4) {
      E v[4] = {};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int px = g.pos[0] + x + k;
        if (g.read && x + k < nx) v[k] = s[g.mirror[0] - px];
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (x + k < nx) {
          if constexpr (!std::is_same<T, Raw>::value) v[k] = chain(v[k], g);
          d[g.pos[0] + x + k] = v[k];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kBcThreads) bc_fill_kernel(const BcSeg *__restrict__ segs, const BcTile *__restrict__ tiles,
                                                             unsigned ntiles) {
  __shared__ BcSeg g;
  __shared__ BcTile t;
  for (unsigned ti = blockIdx.x; ti < ntiles; ti += gridDim.x) {
    __syncthreads(); // everyone is done with the previous tile's descriptor
    if (0 == threadIdx.x) {
      t = tiles[ti];
      g = segs[t.seg];
    }
    __syncthreads();
    if (g.mirror[0] >= 0) {
      if (1 == g.dtype) fill_xrows<float, float>(g, t);
      else if (2 == g.dtype) fill_xrows<double, double>(g, t);
      else if (1 == g.es) fill_xrows<Raw, unsigned char>(g, t);
      else if (2 == g.es) fill_xrows<Raw, unsigned short>(g, t);
      else if (4 == g.es) fill_xrows<Raw, unsigned>(g, t);
      else if (8 == g.es) fill_xrows<Raw, uint2>(g, t);
      else fill_xrows<Raw, uint4>(g, t);
    } else {
      if (1 == g.dtype) fill_rows_any<float>(g, t);
      else if (2 == g.dtype) fill_rows_any<double>(g, t);
      else fill_rows_any<Raw>(g, t);
    }
  }
}

} // namespace

void launch_bc_fill(const BcSeg *segs_dev, const BcTile *tiles_dev, unsigned ntiles, int grid, cudaStream_t stream) {
  bc_fill_kernel<<<grid, kBcThreads, 0, stream>>>(segs_dev, tiles_dev, ntiles);
}

} // namespace sb
