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
// rop_tile_kernel<T>: the fused residual-restriction (sb_transfer_oplan_create) over a thick box.  A CTA owns 32 x 8
// coarse cells of a z chunk, one per thread, and marches the fine planes of their 64 x 16 footprint: planes z - 1 .. z + 1
// of the footprint and its one-cell ring sit in a 3-slot shared ring, filled one plane ahead through registers (only
// cells inside the checked read box [2 lo - 1, 2 hi + 1) are loaded).  On each fine plane a thread evaluates the op on
// its coarse cell's four fine cells of that plane and adds them to its running sum in the rule's order, so the two
// planes of a coarse cell give the eight values in order and the fine values are never stored.  A chunk starts at an
// even fine plane.  aux is read from global memory as one pair per fine row (a vector where aligned), one plane ahead.
//
// rop_cell_kernel<T>: one thread per coarse cell over up to 16 thin boxes (the exterior slabs, one coarse cell thick),
// every term read through the read-only path.
//
// Coefficient terms (HAS_COEF on both fused kernels, sb_transfer_voplan_create): a term's factor T(w) * C reads its field
// through the read-only path at the term's coefficient offset from each fine cell.
//
// face_restrict_kernel<T, AX>: the face-coefficient restriction (sb_transfer_fplan_create), restrict_kernel's walk over
// the four fine faces normal to AX under each coarse cell.
//
// Numerics: every multiply and add rounded separately (__fmul_rn / __fadd_rn, __dmul_rn / __dadd_rn; no FMA), in the
// order of the rule in include/stencil_b200.h, so a cell's value does not depend on the launch shape or the partition.
#include "transfer.cuh"

#include <type_traits>

namespace sb {
namespace {

template <typename T> struct TNum;
template <> struct TNum<float> {
  using V2 = float2;
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float w(const RopCommon &c, int t) { return c.wf[t]; }
};
template <> struct TNum<double> {
  using V2 = double2;
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double w(const RopCommon &c, int t) { return c.w[t]; }
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

// face_restrict_kernel<T, AX>: restrict_kernel's walk, one thread per coarse cell, reading the four fine faces normal to
// axis AX under it (the fine plane 2I_AX only): on AX = 0 every other element of two rows in two planes, on AX = 1 a
// pair in each of two planes, on AX = 2 a pair in each of two rows
template <typename T, int AX> __global__ void __launch_bounds__(kRestrictX * kRestrictY) face_restrict_kernel(const __grid_constant__ RestrictParams p) {
  using N = TNum<T>;
  constexpr long long ES = sizeof(T);
  const int i = blockIdx.x * kRestrictX + threadIdx.x, j = blockIdx.y * kRestrictY + threadIdx.y;
  if (i >= p.ext[0] || j >= p.ext[1]) return;
  const long long fx = p.flo[0] + 2 * i, fy = p.flo[1] + 2 * j;
  const long long cx = p.lo[0] + i, cy = p.lo[1] + j;
  for (int k = blockIdx.z; k < p.ext[2]; k += gridDim.z) {
    const char *r00 = p.src + (p.flo[2] + 2ll * k) * p.sslice + fy * p.spitch + fx * ES; // fine row y0 of plane z0
    T f0, f1, f2, f3; // F(2I), F(2I + e_b), F(2I + e_c), F(2I + e_b + e_c)
    if constexpr (AX == 0) { // b = y, c = z
      f0 = __ldg(reinterpret_cast<const T *>(r00));
      f1 = __ldg(reinterpret_cast<const T *>(r00 + p.spitch));
      f2 = __ldg(reinterpret_cast<const T *>(r00 + p.sslice));
      f3 = __ldg(reinterpret_cast<const T *>(r00 + p.sslice + p.spitch));
    } else if constexpr (AX == 1) { // b = x, c = z
      load_pair<T>(r00, f0, f1);
      load_pair<T>(r00 + p.sslice, f2, f3);
    } else { // b = x, c = y
      load_pair<T>(r00, f0, f1);
      load_pair<T>(r00 + p.spitch, f2, f3);
    }
    const T acc = N::add(N::add(N::add(f0, f1), f2), f3);
    *reinterpret_cast<T *>(p.dst + (p.lo[2] + (long long)k) * p.dslice + cy * p.dpitch + cx * ES) = N::mul(T(0.25), acc);
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

// HAS_COEF: the coefficient variant (sb_transfer_voplan_create), a compile-time switch, so the plain instantiations are
// the code they were; a coefficient term's factor reads its field through the read-only path
template <typename T, bool HAS_COEF = false>
__global__ void __launch_bounds__(kRestrictX * kRestrictY)
    rop_tile_kernel(const __grid_constant__ typename std::conditional<HAS_COEF, RopVTileParams, RopTileParams>::type p) {
  using N = TNum<T>;
  constexpr long long ES = sizeof(T);
  constexpr int NT = kRestrictX * kRestrictY;
  constexpr int PER = (kRopPlane + NT - 1) / NT; // ring elements per thread and plane
  __shared__ T ring[3][kRopPlane];

  const int tid = threadIdx.x, lane = tid & 31, wy = tid >> 5;
  int b = blockIdx.x;
  const int bx = b % p.tiles_x;
  b /= p.tiles_x;
  const int by = b % p.tiles_y, bz = b / p.tiles_y;
  const int k0 = bz * p.zchunk, k1 = min(k0 + p.zchunk, p.ext[2]); // the chunk's coarse planes, box-relative
  if (k0 >= k1) return;
  const int Z0 = p.flo[2] + 2 * k0, Z1 = p.flo[2] + 2 * k1;        // its fine planes, src allocation coordinates
  const int WX = p.flo[0] + 2 * kRestrictX * bx - 1, WY = p.flo[1] + 2 * kRestrictY * by - 1; // ring window origin

  T buf[PER];
  auto fetch = [&](int z) {
    const char *plane = p.c.src + (long long)z * p.c.sslice;
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int q = tid + e * NT;
      const int r = q / kRopSW, col = q - r * kRopSW;
      const int x = WX + col, y = WY + r;
      buf[e] = T(0);
      if (q < kRopPlane && x >= p.rlo[0] && x < p.rhi[0] && y >= p.rlo[1] && y < p.rhi[1])
        buf[e] = __ldg(reinterpret_cast<const T *>(plane + y * p.c.spitch + x * ES));
    }
  };
  auto store = [&](int z) {
    T *pl = ring[(z - Z0 + 1) % 3];
#pragma unroll
    for (int e = 0; e < PER; ++e) {
      const int q = tid + e * NT;
      if (q < kRopPlane) pl[q] = buf[e];
    }
  };
  fetch(Z0 - 1);
  store(Z0 - 1);
  fetch(Z0);
  store(Z0);
  fetch(Z0 + 1);

  const int i = kRestrictX * bx + lane, j = kRestrictY * by + wy; // this thread's coarse cell, box-relative
  const bool mine = i < p.ext[0] && j < p.ext[1];
  const int fx = p.flo[0] + 2 * i, fy = p.flo[1] + 2 * j;
  const int s00 = (2 * wy + 1) * kRopSW + 2 * lane + 1; // the fine cell (0, 0, .) in a ring slot
  // aux of this thread's two fine rows, one plane ahead like the ring, so its latency hides behind a plane's work
  T ax[2][2] = {{T(0), T(0)}, {T(0), T(0)}};
  auto fetch_aux = [&](int z) {
    if (mine && p.c.aux)
#pragma unroll
      for (int dy = 0; dy < 2; ++dy)
        load_pair<T>(p.c.aux + (long long)z * p.c.sslice + (long long)(fy + dy) * p.c.spitch + fx * ES, ax[dy][0], ax[dy][1]);
  };
  fetch_aux(Z0);
  T acc = T(0);
  for (int zc = Z0; zc < Z1; ++zc) {
    store(zc + 1);
    __syncthreads();
    if (zc + 1 < Z1) fetch(zc + 2);
    const T a[2][2] = {{ax[0][0], ax[0][1]}, {ax[1][0], ax[1][1]}};
    if (zc + 1 < Z1) fetch_aux(zc + 1);
    if (mine) {
      // the op on the four fine cells (dx, dy) of this plane, term by term (each term's table entry read once for all
      // four), each cell's sum in list order; v[2 dy + dx]
      const T *q0 = &ring[0][0] + s00;
      const int *toff = p.toff[(zc - Z0 + 1) % 3];
      T v[4];
      for (int t = 0; t < p.c.n; ++t) {
        const T w = N::w(p.c, t);
        T m[4];
        if constexpr (HAS_COEF) { // (T(w) * C) * S, C at the term's coefficient offset from each fine cell
          T wk[4] = {w, w, w, w};
          const int cf = p.cfield[t];
          if (cf >= 0) {
            const char *c0 = p.coef[cf] + (long long)zc * p.c.sslice + (long long)fy * p.c.spitch + fx * ES + p.cgoff[t];
#pragma unroll
            for (int k = 0; k < 4; ++k) wk[k] = N::mul(w, __ldg(reinterpret_cast<const T *>(c0 + (k >> 1) * p.c.spitch + (k & 1) * ES)));
          }
          if (p.c.source[t] == 0) {
            const T *q = q0 + toff[t];
            m[0] = N::mul(wk[0], q[0]);
            m[1] = N::mul(wk[1], q[1]);
            m[2] = N::mul(wk[2], q[kRopSW]);
            m[3] = N::mul(wk[3], q[kRopSW + 1]);
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) m[k] = N::mul(wk[k], a[k >> 1][k & 1]);
          }
        } else if (p.c.source[t] == 0) {
          const T *q = q0 + toff[t];
          m[0] = N::mul(w, q[0]);
          m[1] = N::mul(w, q[1]);
          m[2] = N::mul(w, q[kRopSW]);
          m[3] = N::mul(w, q[kRopSW + 1]);
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) m[k] = N::mul(w, a[k >> 1][k & 1]);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) v[k] = t == 0 ? m[k] : N::add(v[k], m[k]);
      }
      const bool first = ((zc - Z0) & 1) == 0;
      acc = first ? v[0] : N::add(acc, v[0]);
#pragma unroll
      for (int k = 1; k < 4; ++k) acc = N::add(acc, v[k]);
      if (!first)
        *reinterpret_cast<T *>(p.c.dst + (long long)(p.lo[2] + (zc - p.flo[2]) / 2) * p.c.dslice + (long long)(p.lo[1] + j) * p.c.dpitch +
                               (long long)(p.lo[0] + i) * ES) = N::mul(T(0.125), acc);
    }
    __syncthreads();
  }
}

// HAS_COEF: the coefficient variant (sb_transfer_voplan_create), a compile-time switch, so the plain instantiations are
// the code they were
template <typename T, bool HAS_COEF = false>
__global__ void __launch_bounds__(256) rop_cell_kernel(const __grid_constant__ typename std::conditional<HAS_COEF, RopVCellParams, RopCellParams>::type p) {
  using N = TNum<T>;
  constexpr long long ES = sizeof(T);
  const long long total = p.first[p.n];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int k = 0;
    while (k + 1 < p.n && i >= p.first[k + 1]) ++k;
    const unsigned li = (unsigned)(i - p.first[k]);
    const unsigned ex = p.ext[k][0], ey = p.ext[k][1];
    unsigned xx, yy, zz;
    if (ex >= 32) { // x fastest
      xx = li % ex;
      const unsigned t = li / ex;
      yy = t % ey;
      zz = t / ey;
    } else { // y fastest: an x slab is one column per row
      yy = li % ey;
      const unsigned t = li / ey;
      xx = t % ex;
      zz = t / ex;
    }
    const long long f0 = (long long)(p.flo[k][2] + 2 * (int)zz) * p.c.sslice + (long long)(p.flo[k][1] + 2 * (int)yy) * p.c.spitch +
                         (long long)(p.flo[k][0] + 2 * (int)xx) * ES;
    T acc = T(0);
#pragma unroll
    for (int d = 0; d < 8; ++d) { // the rule's order: x fastest, then y, then z
      const long long f = f0 + (d >> 2) * p.c.sslice + ((d >> 1) & 1) * p.c.spitch + (d & 1) * ES;
      const T a = p.c.aux ? __ldg(reinterpret_cast<const T *>(p.c.aux + f)) : T(0);
      T v = T(0);
      for (int t = 0; t < p.c.n; ++t) {
        const signed char *o = p.c.off[t];
        const T x = p.c.source[t] == 0 ? __ldg(reinterpret_cast<const T *>(p.c.src + f + o[2] * p.c.sslice + o[1] * p.c.spitch + o[0] * ES)) : a;
        T w = N::w(p.c, t);
        if constexpr (HAS_COEF) {
          const int cf = p.cfield[t];
          if (cf >= 0) {
            const signed char *c = p.coff[t];
            w = N::mul(w, __ldg(reinterpret_cast<const T *>(p.coef[cf] + f + c[2] * p.c.sslice + c[1] * p.c.spitch + c[0] * ES)));
          }
        }
        const T m = N::mul(w, x);
        v = t == 0 ? m : N::add(v, m);
      }
      acc = d == 0 ? v : N::add(acc, v);
    }
    *reinterpret_cast<T *>(p.c.dst + (long long)(p.lo[k][2] + (int)zz) * p.c.dslice + (long long)(p.lo[k][1] + (int)yy) * p.c.dpitch +
                           (long long)(p.lo[k][0] + (int)xx) * ES) = N::mul(T(0.125), acc);
  }
}

} // namespace

int rop_tile_ctas_per_sm(int es, bool coef) {
  int ctas = 0;
  const void *fn = coef ? (es == 4 ? reinterpret_cast<const void *>(&rop_tile_kernel<float, true>) : reinterpret_cast<const void *>(&rop_tile_kernel<double, true>))
                        : (es == 4 ? reinterpret_cast<const void *>(&rop_tile_kernel<float>) : reinterpret_cast<const void *>(&rop_tile_kernel<double>));
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, fn, kRestrictX * kRestrictY, 0) != cudaSuccess) return 0;
  return ctas;
}

int launch_rop_tile(const RopTileParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0) return 0;
  if (es == 4)
    rop_tile_kernel<float><<<unsigned(grid), kRestrictX * kRestrictY, 0, stream>>>(p);
  else if (es == 8)
    rop_tile_kernel<double><<<unsigned(grid), kRestrictX * kRestrictY, 0, stream>>>(p);
  else
    return 0;
  return 1;
}

int launch_rop_cells(const RopCellParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0 || p.n <= 0) return 0;
  if (es == 4)
    rop_cell_kernel<float><<<unsigned(grid), 256, 0, stream>>>(p);
  else if (es == 8)
    rop_cell_kernel<double><<<unsigned(grid), 256, 0, stream>>>(p);
  else
    return 0;
  return 1;
}

int launch_rop_vtile(const RopVTileParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0) return 0;
  if (es == 4)
    rop_tile_kernel<float, true><<<unsigned(grid), kRestrictX * kRestrictY, 0, stream>>>(p);
  else if (es == 8)
    rop_tile_kernel<double, true><<<unsigned(grid), kRestrictX * kRestrictY, 0, stream>>>(p);
  else
    return 0;
  return 1;
}

int launch_rop_vcells(const RopVCellParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0 || p.n <= 0) return 0;
  if (es == 4)
    rop_cell_kernel<float, true><<<unsigned(grid), 256, 0, stream>>>(p);
  else if (es == 8)
    rop_cell_kernel<double, true><<<unsigned(grid), 256, 0, stream>>>(p);
  else
    return 0;
  return 1;
}

int launch_face_restrict(const RestrictParams &p, int es, int axis, cudaStream_t stream) {
  if (p.ext[0] <= 0 || p.ext[1] <= 0 || p.ext[2] <= 0 || axis < 0 || axis > 2 || (es != 4 && es != 8)) return 0;
  const dim3 grid(unsigned((p.ext[0] + kRestrictX - 1) / kRestrictX), unsigned((p.ext[1] + kRestrictY - 1) / kRestrictY),
                  unsigned(p.ext[2] < 65535 ? p.ext[2] : 65535));
  const dim3 block(kRestrictX, kRestrictY);
  using K = void (*)(const RestrictParams);
  static const K fn[2][3] = {{face_restrict_kernel<float, 0>, face_restrict_kernel<float, 1>, face_restrict_kernel<float, 2>},
                             {face_restrict_kernel<double, 0>, face_restrict_kernel<double, 1>, face_restrict_kernel<double, 2>}};
  fn[es == 8][axis]<<<grid, block, 0, stream>>>(p);
  return 1;
}

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
