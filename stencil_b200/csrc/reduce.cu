// Reduction kernels (see reduce.cuh and the sb_reduce_* entries of include/stencil_b200.h).
#include "reduce.cuh"

namespace sb {
namespace {

struct Acc {
  double mn, mx, s, q;
};

// One cell: v and q (the operations of cell_terms, written out so that the SASS stays as it is), then one step of each
// chain.  `v < mn || v != v` keeps a NaN once it is in and lets a NaN in.
template <int KIND> __device__ __forceinline__ void add(Acc &a, double x, double y, double z) {
  double v, q;
  if (KIND == SB_REDUCE_SCALAR) {
    v = x;
    q = __dmul_rn(v, v);
  } else if (KIND == SB_REDUCE_DIFF) {
    v = __dadd_rn(x, -y);
    q = __dmul_rn(v, v);
  } else {
    q = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
    v = __dsqrt_rn(q);
  }
  a.mn = (v < a.mn || v != v) ? v : a.mn;
  a.mx = (v > a.mx || v != v) ? v : a.mx;
  a.s = __dadd_rn(a.s, v);
  a.q = __dadd_rn(a.q, q);
}

#include "reduce_rows.cuh"

__device__ __forceinline__ sb_reduce_result as_result(const Acc &a) { return sb_reduce_result{a.mn, a.mx, a.s, a.q, 0}; }
__device__ __forceinline__ Acc as_acc(const sb_reduce_result &r) { return Acc{r.min, r.max, r.sum, r.sumsq}; }

// Launch 1, one instance per class (element type, kind, access width): the tiles [begin, end) of the table.  (One
// kernel that branches over all twelve classes per tile needs 255 registers and spills; each class alone needs 44-102.)
template <typename T, int KIND, bool WIDE>
__global__ void __launch_bounds__(kRedThreads) reduce_tiles_kernel(const RedItem *__restrict__ items, const RedTile *__restrict__ tiles,
                                                                   unsigned begin, unsigned end, RedPartial *__restrict__ part) {
  __shared__ RedItem it;
  __shared__ RedTile t;
  __shared__ Acc warp_acc[kRedThreads / 32];
  for (unsigned ti = begin + blockIdx.x; ti < end; ti += gridDim.x) {
    __syncthreads(); // everyone is done with the previous tile's descriptor and warp_acc
    if (0 == threadIdx.x) {
      t = tiles[ti];
      it = items[t.item];
    }
    __syncthreads();
    Acc a{pos_inf(), -pos_inf(), 0.0, 0.0};
    reduce_rows<T, KIND, WIDE, Acc>(it, t, a);
    // the block's 256 chains: a fixed tree, lane l + o into lane l for o = 16, 8, 4, 2, 1, then warps 2i + 1 into 2i,
    // 4i + 2 into 4i, 4 into 0
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const Acc b{__shfl_down_sync(0xffffffffu, a.mn, o), __shfl_down_sync(0xffffffffu, a.mx, o), __shfl_down_sync(0xffffffffu, a.s, o),
                  __shfl_down_sync(0xffffffffu, a.q, o)};
      a = as_acc(red_merge(as_result(a), as_result(b)));
    }
    if (0 == (threadIdx.x & 31)) warp_acc[threadIdx.x >> 5] = a;
    __syncthreads();
    if (0 == threadIdx.x) {
      for (int s = 1; s < kRedThreads / 32; s <<= 1)
        for (int i = 0; i + s < kRedThreads / 32; i += 2 * s) warp_acc[i] = as_acc(red_merge(as_result(warp_acc[i]), as_result(warp_acc[i + s])));
      const Acc &r = warp_acc[0];
      part[ti] = RedPartial{r.mn, r.mx, r.s, r.q};
    }
  }
}

// One block per item: its tile partials, in tile order, by the pairwise tree "i += i + s for i % 2s == 0" for s = 1, 2,
// 4, ... in place (the scratch is rewritten by every launch).
__global__ void __launch_bounds__(kRedThreads) reduce_items_kernel(const RedItem *__restrict__ items, RedPartial *part,
                                                                   sb_reduce_result *__restrict__ out) {
  const unsigned n = items[blockIdx.x].ntiles;
  RedPartial *p = part + items[blockIdx.x].tile0;
  for (unsigned long long s = 1; s < n; s <<= 1) {
    for (unsigned long long i = threadIdx.x * 2 * s; i + s < n; i += 2 * s * kRedThreads) {
      const RedPartial a = p[i], b = p[i + s];
      const sb_reduce_result m = red_merge(sb_reduce_result{a.min, a.max, a.sum, a.sumsq, 0}, sb_reduce_result{b.min, b.max, b.sum, b.sumsq, 0});
      p[i] = RedPartial{m.min, m.max, m.sum, m.sumsq};
    }
    __syncthreads();
  }
  if (0 == threadIdx.x) {
    sb_reduce_result r{pos_inf(), -pos_inf(), 0.0, 0.0, items[blockIdx.x].count};
    if (n) {
      r.min = p[0].min;
      r.max = p[0].max;
      r.sum = p[0].sum;
      r.sumsq = p[0].sumsq;
    }
    out[blockIdx.x] = r;
  }
}

// the instance of class c = 6 * (dtype == F64) + 2 * kind + (vec == 16)
using ClassKernel = void (*)(const RedItem *, const RedTile *, unsigned, unsigned, RedPartial *);
ClassKernel class_kernel(int c) {
  static const ClassKernel k[kRedClasses] = {
      reduce_tiles_kernel<float, SB_REDUCE_SCALAR, false>,  reduce_tiles_kernel<float, SB_REDUCE_SCALAR, true>,
      reduce_tiles_kernel<float, SB_REDUCE_DIFF, false>,    reduce_tiles_kernel<float, SB_REDUCE_DIFF, true>,
      reduce_tiles_kernel<float, SB_REDUCE_NORM3, false>,   reduce_tiles_kernel<float, SB_REDUCE_NORM3, true>,
      reduce_tiles_kernel<double, SB_REDUCE_SCALAR, false>, reduce_tiles_kernel<double, SB_REDUCE_SCALAR, true>,
      reduce_tiles_kernel<double, SB_REDUCE_DIFF, false>,   reduce_tiles_kernel<double, SB_REDUCE_DIFF, true>,
      reduce_tiles_kernel<double, SB_REDUCE_NORM3, false>,  reduce_tiles_kernel<double, SB_REDUCE_NORM3, true>};
  return k[c];
}

} // namespace

int reduce_class(const RedItem &it) { return 6 * (it.dtype == SB_DTYPE_F64) + 2 * it.kind + (it.vec == 16); }

int persistent_grid(int device, const void *kernel, unsigned ntiles) {
  int sms = 132, per_sm = 1;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kRedThreads, 0) != cudaSuccess || per_sm < 1) {
    cudaGetLastError();
    per_sm = 1;
  }
  const long long cap = (long long)sms * per_sm;
  return int(ntiles < cap ? ntiles : cap);
}

int reduce_grid(int device, int cls, unsigned ntiles) { return persistent_grid(device, reinterpret_cast<const void *>(class_kernel(cls)), ntiles); }

int launch_reduce(const RedItem *items_dev, unsigned nitems, const RedTile *tiles_dev, const unsigned (*class_tiles)[2], const int *grids,
                  RedPartial *scratch, sb_reduce_result *out, cudaStream_t stream) {
  int launches = 0;
  for (int c = 0; c < kRedClasses; ++c) {
    if (class_tiles[c][1] > class_tiles[c][0]) {
      class_kernel(c)<<<grids[c], kRedThreads, 0, stream>>>(items_dev, tiles_dev, class_tiles[c][0], class_tiles[c][1], scratch);
      ++launches;
    }
  }
  reduce_items_kernel<<<nitems, kRedThreads, 0, stream>>>(items_dev, scratch, out);
  return launches + 1;
}

} // namespace sb
