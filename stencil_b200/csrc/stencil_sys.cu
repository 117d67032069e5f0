// Linear stencil systems for sm_90a: up to 8 inputs and 4 outputs per launch (see stencil_sys.cuh and
// include/stencil_b200.h).
//
// sys_tile_kernel<T>: z-march over thick boxes.  A CTA owns a 64 x 8 tile of cells and a z chunk.  Each input the system
// reads has its own ring of halo'd planes in shared memory, cut to that input's reach, so an input read only at offset 0
// holds the tile's own cells and nothing more.  Planes go global -> shared through cp.async one plane ahead (no
// register staging, so the register count does not grow with the number of inputs), each input plane of a tile is read
// from HBM once, and every read a term makes comes from shared memory.  At the top of each plane the threads turn the
// term table (a __grid_constant__ parameter of at most 4 KB) into this plane's shared offsets, one term per thread.
//
// sys_cell_kernel<T>: one thread per cell over up to 16 thin boxes (the exterior slabs of a subdomain) in ONE launch.
//
// Numerics (both kernels): for each output j, over its terms in list order, acc = m_first; acc = acc + m; with
// m = T(w) * I_in(p + o) or (T(w) * I_coef(p + c)) * I_in(p + o), every multiply and add rounded separately (no FMA
// contraction).  Every output of a cell is computed before any is written, so an output may be an input read only at
// offset 0 (an in-place update).
#include "stencil_sys.cuh"

namespace sb {
namespace {

template <typename T> struct SysNum;
template <> struct SysNum<float> {
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float w(const SysTerms &c, int t) { return c.wf[t]; }
};
template <> struct SysNum<double> {
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double w(const SysTerms &c, int t) { return c.w[t]; }
};

template <int BYTES> __device__ __forceinline__ void cp_async(void *dst, const void *src) {
  const unsigned s = unsigned(__cvta_generic_to_shared(dst));
  if constexpr (BYTES == 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(src) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2;\n" ::"r"(s), "l"(src), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

template <typename T>
__global__ void __launch_bounds__(kOpThreads, 1) sys_tile_kernel(const __grid_constant__ SysTileParams p) {
  extern __shared__ __align__(16) unsigned char sys_smem[];
  int *const tbl = reinterpret_cast<int *>(sys_smem); // [2 planes][2 (source, coefficient)][kSysMaxTerms]
  T *const ring = reinterpret_cast<T *>(sys_smem + kSysTableBytes);
  constexpr int V = 16 / int(sizeof(T));
  constexpr long long ES = sizeof(T);

  const int tid = threadIdx.x, lane = tid & 31, wy = tid >> 5;
  int b = blockIdx.x;
  const int bx = b % p.tiles_x;
  b /= p.tiles_x;
  const int by = b % p.tiles_y, bz = b / p.tiles_y;
  const int x0 = p.lo[0] + bx * kOpTileX, y0 = p.lo[1] + by * kOpTileY, z0 = p.lo[2] + bz * p.zchunk;
  const int xe = min(x0 + kOpTileX, p.lo[0] + p.ext[0]), ye = min(y0 + kOpTileY, p.lo[1] + p.ext[1]);
  const int z1 = min(z0 + p.zchunk, p.lo[2] + p.ext[2]);
  const int sw = p.sw;

  // plane z of input r into its slot: warps own rows, lanes 16-byte chunks (or elements)
  auto load = [&](int r, int z) {
    const int xa = x0 - p.rm[r][0], xb = xe + p.rp[r][0], ya = y0 - p.rm[r][1], rows = ye + p.rp[r][1] - ya;
    const int rows_all = kOpTileY + p.rm[r][1] + p.rp[r][1];
    T *const pl = ring + p.base[r] + ((z - z0 + p.rm[r][2]) % p.ns[r]) * rows_all * sw;
    const char *const plane = p.in[r] + (long long)z * p.c.slice;
    for (int j = wy; j < rows; j += kOpThreads / 32) {
      const char *const row = plane + (long long)(ya + j) * p.c.pitch;
      T *const srow = pl + j * sw;
      const char *const wa = row + xa * ES, *const wb = row + xb * ES;
      if (p.vec[r]) {
        const char *const c0 = reinterpret_cast<const char *>(reinterpret_cast<uintptr_t>(wa) & ~uintptr_t(15));
        const int nch = int((wb - c0 + 15) >> 4);
        for (int k = lane; k < nch; k += 32) {
          const char *const ca = c0 + 16 * k;
          if (ca >= wa && ca + 16 <= wb) {
            cp_async<16>(srow + k * V, ca);
          } else { // a chunk that reaches past the window: its wanted elements one by one, so no cell outside the window
                   // is read (those may be written meanwhile: by this launch where an output is this input, by
                   // exchange() in ghost cells, by the exterior launch)
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const char *const a = ca + v * ES;
              if (a >= wa && a < wb) cp_async<int(sizeof(T))>(srow + k * V + v, a);
            }
          }
        }
      } else {
        for (int i = lane; i < xb - xa; i += 32) cp_async<int(sizeof(T))>(srow + i, wa + i * ES);
      }
    }
  };

  if (z0 < z1)
    for (int r = 0; r < p.nr; ++r)
      for (int z = z0 - p.rm[r][2]; z <= z0 + p.rp[r][2]; ++z) load(r, z);

  const int y = y0 + wy, xA = x0 + lane, xB = xA + 32;
  const bool okA = y < ye && xA < xe, okB = y < ye && xB < xe;
  const T *const own = ring + wy * sw + lane;
  for (int zc = z0; zc < z1; ++zc) {
    int *const to = tbl + ((zc - z0) & 1) * 2 * kSysMaxTerms, *const tc = to + kSysMaxTerms;
    for (int t = tid; t < p.c.n; t += kOpThreads) { // this plane's shared offsets (the table of plane zc - 2 is free)
      const int r = p.c.in[t];
      const int rows_r = kOpTileY + p.rm[r][1] + p.rp[r][1];
      to[t] = p.base[r] + ((zc - z0 + p.rm[r][2] + p.oz[t]) % p.ns[r]) * rows_r * sw + p.inpl[t];
      const int k = p.c.cin[t];
      if (k >= 0) {
        const int rows_k = kOpTileY + p.rm[k][1] + p.rp[k][1];
        tc[t] = p.base[k] + ((zc - z0 + p.rm[k][2] + p.coz[t]) % p.ns[k]) * rows_k * sw + p.cinpl[t];
      }
    }
    cp_async_wait_all(); // this thread's planes up to zc + rp have landed
    __syncthreads();     // everyone's have, and every read of plane zc - 1 is done
    if (zc + 1 < z1)     // into the slots of planes zc - rm - 1, which no cell of plane zc reads
      for (int r = 0; r < p.nr; ++r) load(r, zc + 1 + p.rp[r][2]);

    T acc[kSysMaxOutputs][2];
#pragma unroll
    for (int j = 0; j < kSysMaxOutputs; ++j) {
      acc[j][0] = acc[j][1] = T(0);
      if (j >= p.c.nout) continue;
      for (int t = p.c.first[j]; t < p.c.first[j + 1]; ++t) {
        const int o = to[t];
        const T vA = own[o], vB = own[o + 32];
        const T w = SysNum<T>::w(p.c, t);
        T wA = w, wB = w;
        if (p.c.cin[t] >= 0) {
          const int co = tc[t];
          wA = SysNum<T>::mul(w, own[co]);
          wB = SysNum<T>::mul(w, own[co + 32]);
        }
        const T mA = SysNum<T>::mul(wA, vA), mB = SysNum<T>::mul(wB, vB);
        const bool first = t == p.c.first[j];
        acc[j][0] = first ? mA : SysNum<T>::add(acc[j][0], mA);
        acc[j][1] = first ? mB : SysNum<T>::add(acc[j][1], mB);
      }
    }
    const long long cell = (long long)zc * p.c.slice + (long long)y * p.c.pitch;
#pragma unroll
    for (int j = 0; j < kSysMaxOutputs; ++j) {
      if (j >= p.c.nout) continue;
      if (okA) *reinterpret_cast<T *>(p.c.out[j] + cell + xA * ES) = acc[j][0];
      if (okB) *reinterpret_cast<T *>(p.c.out[j] + cell + xB * ES) = acc[j][1];
    }
  }
}

template <typename T> __global__ void __launch_bounds__(256) sys_cell_kernel(const __grid_constant__ SysCellParams p) {
  constexpr long long ES = sizeof(T);
  const long long total = p.first[p.nb];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int k = 0;
    while (k + 1 < p.nb && i >= p.first[k + 1]) ++k;
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
                          (long long)(p.lo[k][0] + (int)xx) * ES;
    auto at = [&](int r, const signed char o[3]) { // plain loads: an input may be an output of this launch
      return *reinterpret_cast<const T *>(p.in[r] + off + o[2] * p.c.slice + o[1] * p.c.pitch + o[0] * ES);
    };
    T acc[kSysMaxOutputs];
#pragma unroll
    for (int j = 0; j < kSysMaxOutputs; ++j) {
      acc[j] = T(0);
      if (j >= p.c.nout) continue;
      for (int t = p.c.first[j]; t < p.c.first[j + 1]; ++t) {
        T w = SysNum<T>::w(p.c, t);
        if (p.c.cin[t] >= 0) w = SysNum<T>::mul(w, at(p.c.cin[t], p.co[t]));
        const T m = SysNum<T>::mul(w, at(p.c.in[t], p.o[t]));
        acc[j] = t == p.c.first[j] ? m : SysNum<T>::add(acc[j], m);
      }
    }
#pragma unroll
    for (int j = 0; j < kSysMaxOutputs; ++j)
      if (j < p.c.nout) *reinterpret_cast<T *>(p.c.out[j] + off) = acc[j];
  }
}

const void *tile_fn(int es) {
  return es == 4 ? reinterpret_cast<const void *>(&sys_tile_kernel<float>) : reinterpret_cast<const void *>(&sys_tile_kernel<double>);
}

} // namespace

int sys_tile_prepare(int es, int device, size_t smem) {
  const void *fn = tile_fn(es);
  int optin = 0;
  if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) return 0;
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, optin) != cudaSuccess) return 0;
  int ctas = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, fn, kOpThreads, smem) != cudaSuccess) return 0;
  return ctas;
}

int launch_sys_tile(const SysTileParams &p, int es, size_t smem, int grid, cudaStream_t stream) {
  if (grid <= 0) return 0;
  if (es == 4)
    sys_tile_kernel<float><<<unsigned(grid), kOpThreads, smem, stream>>>(p);
  else
    sys_tile_kernel<double><<<unsigned(grid), kOpThreads, smem, stream>>>(p);
  return 1;
}

int launch_sys_cells(const SysCellParams &p, int es, int grid, cudaStream_t stream) {
  if (grid <= 0 || p.nb <= 0) return 0;
  if (es == 4)
    sys_cell_kernel<float><<<unsigned(grid), 256, 0, stream>>>(p);
  else
    sys_cell_kernel<double><<<unsigned(grid), 256, 0, stream>>>(p);
  return 1;
}

} // namespace sb
