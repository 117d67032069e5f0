// Multigrid transfers for sm_90a (see transfer.cuh and include/stencil_b200.h).  Both kernels are memory-bound by design.
//
// restrict_kernel<T>: one thread per coarse cell, which averages the 2 x 2 x 2 fine cells below it: two fine rows in
// each of two fine planes.  A warp covers 32 coarse cells, so each of its four row reads is 64 contiguous fine
// elements, loaded as 2-element vectors when the pair's address allows it and element by element otherwise (the
// alignment of a pair depends only on its row, so a warp never splits).  No shared memory.
//
// prolong_kernel<T>: a CTA owns a 32 x 8 tile of parent (coarse) cells and a z chunk.  The coarse planes z - 1 .. z + 1
// of the tile and its one-cell ring sit in a 3-slot shared ring, filled one plane ahead through registers, so each
// coarse element is read from HBM about once per tile.  Each thread takes its parent's 3 x 3 x 3 neighbourhood from
// the ring and writes the parent's 2 x 2 x 2 children inside the box: for each of the four child rows, aux is read and
// dst written as one 2-element vector when both children lie in the box and the pair is aligned, element by element
// otherwise.  Only coarse cells the rule reads for a child of the box are loaded.
//
// Numerics: every multiply and add rounded separately (__fmul_rn / __fadd_rn, __dmul_rn / __dadd_rn; no FMA), in the
// order of the rule in include/stencil_b200.h, so a cell's value does not depend on the launch shape or the partition.
#include "transfer.cuh"

namespace sb {
namespace {

template <typename T> struct TNum;
template <> struct TNum<float> {
  using V2 = float2;
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
};
template <> struct TNum<double> {
  using V2 = double2;
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
};

template <typename T> __device__ __forceinline__ bool pair_aligned(const void *a) {
  return (reinterpret_cast<uintptr_t>(a) & (2 * sizeof(T) - 1)) == 0;
}

// the fine elements x and x + 1 of a row
template <typename T> __device__ __forceinline__ void load_pair(const char *a, T &v0, T &v1) {
  if (pair_aligned<T>(a)) {
    const typename TNum<T>::V2 v = __ldg(reinterpret_cast<const typename TNum<T>::V2 *>(a));
    v0 = v.x;
    v1 = v.y;
  } else {
    v0 = __ldg(reinterpret_cast<const T *>(a));
    v1 = __ldg(reinterpret_cast<const T *>(a) + 1);
  }
}

template <typename T> __global__ void __launch_bounds__(kRestrictX * kRestrictY) restrict_kernel(const __grid_constant__ RestrictParams p) {
  using N = TNum<T>;
  constexpr long long ES = sizeof(T);
  const int i = blockIdx.x * kRestrictX + threadIdx.x, j = blockIdx.y * kRestrictY + threadIdx.y;
  if (i >= p.ext[0] || j >= p.ext[1]) return;
  const long long fx = p.flo[0] + 2 * i, fy = p.flo[1] + 2 * j;
  const long long cx = p.lo[0] + i, cy = p.lo[1] + j;
  for (int k = blockIdx.z; k < p.ext[2]; k += gridDim.z) {
    const char *r00 = p.src + (p.flo[2] + 2ll * k) * p.sslice + fy * p.spitch + fx * ES; // fine row y0 of plane z0
    const char *r10 = r00 + p.spitch, *r01 = r00 + p.sslice, *r11 = r01 + p.spitch;
    T a00, b00, a10, b10, a01, b01, a11, b11;
    load_pair<T>(r00, a00, b00);
    load_pair<T>(r10, a10, b10);
    load_pair<T>(r01, a01, b01);
    load_pair<T>(r11, a11, b11);
    T acc = a00;
    acc = N::add(acc, b00); // (1,0,0)
    acc = N::add(acc, a10); // (0,1,0)
    acc = N::add(acc, b10); // (1,1,0)
    acc = N::add(acc, a01); // (0,0,1)
    acc = N::add(acc, b01); // (1,0,1)
    acc = N::add(acc, a11); // (0,1,1)
    acc = N::add(acc, b11); // (1,1,1)
    *reinterpret_cast<T *>(p.dst + (p.lo[2] + (long long)k) * p.dslice + cy * p.dpitch + cx * ES) = N::mul(T(0.125), acc);
  }
}

template <typename T> __global__ void __launch_bounds__(kProlongThreads) prolong_kernel(const __grid_constant__ ProlongParams p) {
  using N = TNum<T>;
  constexpr long long ES = sizeof(T);
  constexpr int PER = (kProlongPlane + kProlongThreads - 1) / kProlongThreads; // ring elements per thread and plane
  __shared__ T ring[3][kProlongPlane];

  const int tid = threadIdx.x, lane = tid & 31, wy = tid >> 5;
  int b = blockIdx.x;
  const int bx = b % p.tiles_x;
  b /= p.tiles_x;
  const int by = b % p.tiles_y, bz = b / p.tiles_y;
  const int X0 = p.plo[0] + bx * kProlongX, Y0 = p.plo[1] + by * kProlongY, Z0 = p.plo[2] + bz * p.zchunk;
  const int Z1 = min(Z0 + p.zchunk, p.plo[2] + p.pext[2]);
  if (Z0 >= Z1) return;

  // plane z of the window [X0 - 1, X0 + kProlongX + 1) x [Y0 - 1, Y0 + kProlongY + 1), only the cells the rule reads
  T buf[PER];
  auto fetch = [&](int z) {
    const bool zin = z >= p.rlo[2] && z < p.rhi[2];
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int q = tid + e * kProlongThreads;
      const int r = q / kProlongSW, c = q - r * kProlongSW;
      const int x = X0 - 1 + c, y = Y0 - 1 + r;
      buf[e] = T(0);
      if (zin && q < kProlongPlane && x >= p.rlo[0] && x < p.rhi[0] && y >= p.rlo[1] && y < p.rhi[1])
        buf[e] = __ldg(reinterpret_cast<const T *>(p.src + z * p.sslice + y * p.spitch + x * ES));
    }
  };
  auto store = [&](int z) {
    T *pl = ring[(z - Z0 + 1) % 3];
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int q = tid + e * kProlongThreads;
      if (q < kProlongPlane) pl[q] = buf[e];
    }
  };
  fetch(Z0 - 1);
  store(Z0 - 1);
  fetch(Z0);
  store(Z0);
  fetch(Z0 + 1);

  const int Px = X0 + lane, Py = Y0 + wy; // this thread's parent (src allocation coordinates)
  const bool mine = Px < p.plo[0] + p.pext[0] && Py < p.plo[1] + p.pext[1];
  const int fx = 2 * Px + p.off[0], fy = 2 * Py + p.off[1]; // its child (0, 0, .) in dst's allocation coordinates
  const bool in_x0 = fx >= p.lo[0] && fx < p.lo[0] + p.ext[0];
  const bool in_x1 = fx + 1 >= p.lo[0] && fx + 1 < p.lo[0] + p.ext[0];
  const T w27 = T(27.0 / 64.0), w9 = T(9.0 / 64.0), w3 = T(3.0 / 64.0), w1 = T(1.0 / 64.0);

  for (int zc = Z0; zc < Z1; ++zc) {
    store(zc + 1);
    __syncthreads();
    if (zc + 1 < Z1) fetch(zc + 2);
    if (mine) {
      // the aux pairs of the four child rows first, so that their loads are in flight together (aux may be dst: every
      // one is read before this thread writes its cells)
      const bool vec_x = in_x0 && in_x1;
      bool row_in[2][2], vec[2][2];
      typename N::V2 a[2][2];
#pragma unroll
      for (int cz = 0; cz < 2; ++cz)
#pragma unroll
        for (int cy = 0; cy < 2; ++cy) {
          const int fz = 2 * zc + cz + p.off[2], fyy = fy + cy;
          row_in[cz][cy] = fz >= p.lo[2] && fz < p.lo[2] + p.ext[2] && fyy >= p.lo[1] && fyy < p.lo[1] + p.ext[1];
          const long long row = (long long)fz * p.dslice + (long long)fyy * p.dpitch + (long long)fx * ES;
          // aux shares dst's pitch but may start at another phase: a vector pair must be aligned in both
          vec[cz][cy] = vec_x && pair_aligned<T>(p.dst + row) && (!p.aux || pair_aligned<T>(p.aux + row));
          a[cz][cy].x = a[cz][cy].y = T(0);
          if (p.aux && row_in[cz][cy]) {
            if (vec[cz][cy]) {
              a[cz][cy] = *reinterpret_cast<const typename N::V2 *>(p.aux + row);
            } else {
              if (in_x0) a[cz][cy].x = *reinterpret_cast<const T *>(p.aux + row);
              if (in_x1) a[cz][cy].y = *reinterpret_cast<const T *>(p.aux + row + ES);
            }
          }
        }
      // E[d] = the parent's neighbour at offset d - 1 on each axis
      T E[3][3][3];
#pragma unroll
      for (int dz = 0; dz < 3; ++dz) {
        const T *pl = ring[(zc - 1 + dz - Z0 + 1) % 3];
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) E[dz][dy][dx] = pl[(wy + dy) * kProlongSW + lane + dx];
      }
#pragma unroll
      for (int cz = 0; cz < 2; ++cz) {
#pragma unroll
        for (int cy = 0; cy < 2; ++cy) {
          if (!row_in[cz][cy]) continue;
          const int sz = cz ? 2 : 0, sy = cy ? 2 : 0; // index of P + s along z / y in E
          T v[2];
#pragma unroll
          for (int cx = 0; cx < 2; ++cx) {
            const int sx = cx ? 2 : 0;
            T acc = N::mul(w27, E[1][1][1]);
            acc = N::add(acc, N::mul(w9, E[1][1][sx]));
            acc = N::add(acc, N::mul(w9, E[1][sy][1]));
            acc = N::add(acc, N::mul(w9, E[sz][1][1]));
            acc = N::add(acc, N::mul(w3, E[1][sy][sx]));
            acc = N::add(acc, N::mul(w3, E[sz][1][sx]));
            acc = N::add(acc, N::mul(w3, E[sz][sy][1]));
            acc = N::add(acc, N::mul(w1, E[sz][sy][sx]));
            v[cx] = p.aux ? N::add(cx ? a[cz][cy].y : a[cz][cy].x, acc) : acc;
          }
          char *d = p.dst + (long long)(2 * zc + cz + p.off[2]) * p.dslice + (long long)(fy + cy) * p.dpitch + (long long)fx * ES;
          if (vec[cz][cy]) {
            typename N::V2 o;
            o.x = v[0];
            o.y = v[1];
            *reinterpret_cast<typename N::V2 *>(d) = o;
          } else {
            if (in_x0) reinterpret_cast<T *>(d)[0] = v[0];
            if (in_x1) reinterpret_cast<T *>(d)[1] = v[1];
          }
        }
      }
    }
    __syncthreads();
  }
}

} // namespace

int launch_restrict(const RestrictParams &p, int es, cudaStream_t stream) {
  if (p.ext[0] <= 0 || p.ext[1] <= 0 || p.ext[2] <= 0) return 0;
  const dim3 grid(unsigned((p.ext[0] + kRestrictX - 1) / kRestrictX), unsigned((p.ext[1] + kRestrictY - 1) / kRestrictY),
                  unsigned(p.ext[2] < 65535 ? p.ext[2] : 65535));
  const dim3 block(kRestrictX, kRestrictY);
  if (es == 4)
    restrict_kernel<float><<<grid, block, 0, stream>>>(p);
  else if (es == 8)
    restrict_kernel<double><<<grid, block, 0, stream>>>(p);
  else
    return 0;
  return 1;
}

int prolong_ctas_per_sm(int es) {
  int ctas = 0;
  const void *fn = es == 4 ? reinterpret_cast<const void *>(&prolong_kernel<float>) : reinterpret_cast<const void *>(&prolong_kernel<double>);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, fn, kProlongThreads, 0) != cudaSuccess) return 0;
  return ctas;
}

int launch_prolong(const ProlongParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0) return 0;
  if (es == 4)
    prolong_kernel<float><<<unsigned(grid), kProlongThreads, 0, stream>>>(p);
  else if (es == 8)
    prolong_kernel<double><<<unsigned(grid), kProlongThreads, 0, stream>>>(p);
  else
    return 0;
  return 1;
}

} // namespace sb
