// Constant-coefficient linear stencil operators for sm_90a (see stencil_op.cuh and include/stencil_b200.h).
//
// op_tile_kernel<T, R>: z-march over thick boxes.  A CTA owns a 64 x 8 tile of cells and a z chunk; the halo'd planes
// z - R .. z + R of the tile sit in a shared-memory ring of 2R + 1 slots, so each input plane of the tile is read from
// HBM once (16-byte loads wherever the whole 16 bytes lie inside the allocation; element loads at the ends of a row that
// would otherwise leave it), and every neighbour a term reads comes from shared memory.  The next plane's loads are
// issued into registers before the current plane is computed, so their latency hides behind the arithmetic.  The term
// table is a __grid_constant__ parameter: weights already rounded to T and, for each position of the ring, each term's
// shared-memory offset, precomputed by the plan.
//
// op_cell_kernel<T>: one thread per cell over up to 16 thin boxes (the exterior slabs of a subdomain) in ONE launch,
// neighbours through the read-only path.
//
// Numerics (both kernels): acc = T(w_0) * S_0; acc = acc + T(w_k) * S_k in list order, every multiply and add rounded
// separately (__fmul_rn / __fadd_rn, __dmul_rn / __dadd_rn: no FMA contraction), so the result is a function of the
// inputs only, whatever the launch shape.
#include "stencil_op.cuh"

#include <cstring>

namespace sb {
namespace {

template <typename T> struct OpNum;
template <> struct OpNum<float> {
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float w(const OpCommon &c, int t) { return c.wf[t]; }
};
template <> struct OpNum<double> {
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double w(const OpCommon &c, int t) { return c.w[t]; }
};

template <typename T, int R>
__global__ void __launch_bounds__(kOpThreads, 2) op_tile_kernel(const __grid_constant__ OpTileParams p) {
  extern __shared__ __align__(16) unsigned char op_smem[];
  T *ring = reinterpret_cast<T *>(op_smem);
  constexpr int SW = op_tile_sw(R), P = op_tile_plane(R), NS = 2 * R + 1;
  constexpr int V = 16 / int(sizeof(T));
  constexpr int NCH = (SW + V - 1) / V + 1;                         // 16-byte chunks a row of the window can touch
  constexpr int PER = ((kOpTileY + 2 * R) * NCH + kOpThreads - 1) / kOpThreads; // chunks per thread and plane
  constexpr long long ES = sizeof(T);

  const int tid = threadIdx.x, lane = tid & 31, wy = tid >> 5;
  int b = blockIdx.x;
  const int bx = b % p.tiles_x;
  b /= p.tiles_x;
  const int by = b % p.tiles_y, bz = b / p.tiles_y;
  const int x0 = p.lo[0] + bx * kOpTileX, y0 = p.lo[1] + by * kOpTileY, z0 = p.lo[2] + bz * p.zchunk;
  const int xe = min(x0 + kOpTileX, p.lo[0] + p.ext[0]), ye = min(y0 + kOpTileY, p.lo[1] + p.ext[1]);
  const int z1 = min(z0 + p.zchunk, p.lo[2] + p.ext[2]);
  // the window a plane needs: only as far as the op reaches (cells beyond its reach are never loaded into the ring)
  const int xa = x0 - p.rm[0], xb = xe + p.rp[0], ya = y0 - p.rm[1], nrows = ye + p.rp[1] - ya;
  const int srow0 = R - p.rm[1], scol0 = R - x0; // shared row of window row 0; shared column of x = scol0 + x

  uint4 buf[PER];
  int xc[PER]; // x of the chunk's first element (INT32_MIN: nothing to store)
  auto fetch = [&](int z) {
    const char *plane = p.c.src + (long long)z * p.c.slice;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int q = tid + i * kOpThreads;
      const int j = q / NCH, k = q - j * NCH;
      xc[i] = INT32_MIN;
      if (j < nrows) {
        const char *row = plane + (long long)(ya + j) * p.c.pitch;
        const char *wa = row + xa * ES, *wb = row + xb * ES;
        const char *ca = reinterpret_cast<const char *>((reinterpret_cast<uintptr_t>(wa) & ~uintptr_t(15)) + 16 * uintptr_t(k));
        if (ca < wb) {
          xc[i] = int((ca - row) / ES);
          if (ca >= p.c.src && ca + 16 <= p.src_end) {
            buf[i] = __ldg(reinterpret_cast<const uint4 *>(ca));
          } else { // a chunk that would leave the allocation: its wanted elements one by one
            T e[V];
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const char *a = ca + v * ES;
              e[v] = (a >= wa && a < wb) ? __ldg(reinterpret_cast<const T *>(a)) : T(0);
            }
            memcpy(&buf[i], e, 16);
          }
        }
      }
    }
  };
  auto store = [&](int slot) {
    T *pl = ring + slot * P;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      if (xc[i] == INT32_MIN) continue;
      const int q = tid + i * kOpThreads;
      const int j = q / NCH;
      T e[V];
      memcpy(e, &buf[i], 16);
      T *srow = pl + (srow0 + j) * SW + scol0;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int x = xc[i] + v;
        if (x >= xa && x < xb) srow[x] = e[v];
      }
    }
  };
  auto slot_of = [&](int z) { return (z - z0 + R) % NS; };

  for (int z = z0 - p.rm[2]; z < z0 + p.rp[2]; ++z) {
    fetch(z);
    store(slot_of(z));
  }
  if (z0 < z1) fetch(z0 + p.rp[2]);

  const int y = y0 + wy, xA = x0 + lane, xB = xA + 32;
  const bool okA = y < ye && xA < xe, okB = y < ye && xB < xe;
  const T *own = ring + (wy + R) * SW + lane + R;
  for (int zc = z0; zc < z1; ++zc) {
    store(slot_of(zc + p.rp[2])); // the slot of plane zc + rp - (2R + 1), which no cell of plane zc reads
    __syncthreads();
    if (zc + 1 < z1) fetch(zc + 1 + p.rp[2]);
    const long long cell = (long long)zc * p.c.slice + (long long)y * p.c.pitch;
    T auxA = T(0), auxB = T(0);
    if (p.c.has_aux) { // read before the cell is written: dst may be aux
      if (okA) auxA = *reinterpret_cast<const T *>(p.c.aux + cell + xA * ES);
      if (okB) auxB = *reinterpret_cast<const T *>(p.c.aux + cell + xB * ES);
    }
    const int c = slot_of(zc);
    T accA = T(0), accB = T(0);
    for (int t = 0; t < p.c.n; ++t) {
      T vA, vB;
      if (p.c.source[t] == 0) {
        const int o = p.toff[c][t];
        vA = own[o];
        vB = own[o + 32];
      } else {
        vA = auxA;
        vB = auxB;
      }
      const T w = OpNum<T>::w(p.c, t);
      const T mA = OpNum<T>::mul(w, vA), mB = OpNum<T>::mul(w, vB);
      accA = t == 0 ? mA : OpNum<T>::add(accA, mA);
      accB = t == 0 ? mB : OpNum<T>::add(accB, mB);
    }
    if (okA) *reinterpret_cast<T *>(p.c.dst + cell + xA * ES) = accA;
    if (okB) *reinterpret_cast<T *>(p.c.dst + cell + xB * ES) = accB;
    __syncthreads();
  }
}

template <typename T> __global__ void __launch_bounds__(256) op_cell_kernel(const __grid_constant__ OpCellParams p) {
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
    const long long off = (long long)(p.lo[k][2] + (int)zz) * p.c.slice + (long long)(p.lo[k][1] + (int)yy) * p.c.pitch +
                          (long long)(p.lo[k][0] + (int)xx) * (long long)sizeof(T);
    const char *s = p.c.src + off;
    const T a = p.c.has_aux ? *reinterpret_cast<const T *>(p.c.aux + off) : T(0); // before the write: dst may be aux
    T acc = T(0);
    for (int t = 0; t < p.c.n; ++t) {
      const T v = p.c.source[t] == 0 ? __ldg(reinterpret_cast<const T *>(s + p.goff[t])) : a;
      const T m = OpNum<T>::mul(OpNum<T>::w(p.c, t), v);
      acc = t == 0 ? m : OpNum<T>::add(acc, m);
    }
    *reinterpret_cast<T *>(p.c.dst + off) = acc;
  }
}

template <typename T, int R> const void *tile_fn() { return reinterpret_cast<const void *>(&op_tile_kernel<T, R>); }

const void *tile_kernel(int R, int es) {
  switch (R * 10 + es) {
  case 14: return tile_fn<float, 1>();
  case 24: return tile_fn<float, 2>();
  case 34: return tile_fn<float, 3>();
  case 44: return tile_fn<float, 4>();
  case 18: return tile_fn<double, 1>();
  case 28: return tile_fn<double, 2>();
  case 38: return tile_fn<double, 3>();
  case 48: return tile_fn<double, 4>();
  default: return nullptr;
  }
}

} // namespace

size_t op_tile_smem(int R, int es) { return size_t(2 * R + 1) * size_t(op_tile_plane(R)) * size_t(es); }

int op_tile_prepare(int R, int es, int device) {
  const void *fn = tile_kernel(R, es);
  if (!fn) return 0;
  const int smem = int(op_tile_smem(R, es));
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 0;
  int ctas = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, fn, kOpThreads, smem) != cudaSuccess) return 0;
  (void)device;
  return ctas;
}

int launch_op_tile(const OpTileParams &p, int R, int es, int grid, cudaStream_t stream) {
  if (grid <= 0) return 0;
  const void *fn = tile_kernel(R, es);
  if (!fn) return 0;
  void *args[] = {const_cast<OpTileParams *>(&p)};
  cudaLaunchKernel(fn, dim3(unsigned(grid)), dim3(kOpThreads), args, op_tile_smem(R, es), stream);
  return 1;
}

int launch_op_cells(const OpCellParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0 || p.n <= 0) return 0;
  if (es == 4)
    op_cell_kernel<float><<<unsigned(grid), 256, 0, stream>>>(p);
  else
    op_cell_kernel<double><<<unsigned(grid), 256, 0, stream>>>(p);
  return 1;
}

} // namespace sb
