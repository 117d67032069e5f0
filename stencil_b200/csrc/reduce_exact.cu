// Exact reduction kernels (see reduce.cuh and the sb_reduce_exact_* entries of include/stencil_b200.h).
#include "exact_acc.cuh"
#include "reduce.cuh"

namespace sb {
namespace {

struct ExAcc {
  double mn, mx;
  double fv[kExFpe], fq[kExFpe];
  ExShared *sh;
};

template <int KIND> __device__ __forceinline__ void add(ExAcc &a, double x, double y, double z) {
  double v, q;
  cell_terms<KIND>(x, y, z, v, q);
  a.mn = (v < a.mn || v != v) ? v : a.mn;
  a.mx = (v > a.mx || v != v) ? v : a.mx;
  ex_add(a.fv, v, a.sh, 0);
  ex_add(a.fq, q, a.sh, 1);
}

#include "reduce_rows.cuh"

// Exact launch 1: the tiles [begin, end) of one class, any CTA any tile.  Per tile: min / max by the plain kernel's
// tree, the expansions merged per warp by shuffles and added to the CTA's accumulator, which goes to the tile's partial
// and is cleared for the next tile.
template <typename T, int KIND, bool WIDE>
__global__ void __launch_bounds__(kRedThreads, 1) reduce_exact_tiles_kernel(const RedItem *__restrict__ items, const RedTile *__restrict__ tiles,
                                                                         unsigned begin, unsigned end, RedExactPartial *__restrict__ part) {
  __shared__ RedItem it;
  __shared__ RedTile t;
  __shared__ double warp_mn[kRedThreads / 32], warp_mx[kRedThreads / 32];
  __shared__ ExShared sh;
  for (int k = threadIdx.x; k < 2 * kExDigits; k += kRedThreads) sh.digit[k / kExDigits][k % kExDigits] = 0;
  if (threadIdx.x < 2) sh.flags[threadIdx.x] = 0;
  const unsigned lane = threadIdx.x & 31u;
  for (unsigned ti = begin + blockIdx.x; ti < end; ti += gridDim.x) {
    __syncthreads(); // the accumulator is clear, everyone is done with the previous tile's descriptor
    if (0 == threadIdx.x) {
      t = tiles[ti];
      it = items[t.item];
    }
    __syncthreads();
    ExAcc a{pos_inf(), -pos_inf(), {}, {}, &sh};
    reduce_rows<T, KIND, WIDE, ExAcc>(it, t, a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a.mn = red_min(a.mn, __shfl_down_sync(0xffffffffu, a.mn, o));
      a.mx = red_max(a.mx, __shfl_down_sync(0xffffffffu, a.mx, o));
    }
    ex_warp_merge(a.fv, a.fq, &sh, lane); // lane 0 ends with the warp's expansions
    if (0 == lane) {
      warp_mn[threadIdx.x >> 5] = a.mn;
      warp_mx[threadIdx.x >> 5] = a.mx;
#pragma unroll
      for (int i = 0; i < kExFpe; ++i) {
        ex_add_shared(&sh, 0, a.fv[i]);
        ex_add_shared(&sh, 1, a.fq[i]);
      }
    }
    __syncthreads();
    RedExactPartial &P = part[ti];
    if (0 == threadIdx.x) {
      for (int s = 1; s < kRedThreads / 32; s <<= 1)
        for (int i = 0; i + s < kRedThreads / 32; i += 2 * s) {
          warp_mn[i] = red_min(warp_mn[i], warp_mn[i + s]);
          warp_mx[i] = red_max(warp_mx[i], warp_mx[i + s]);
        }
      P.min = warp_mn[0];
      P.max = warp_mx[0];
    }
    for (int k = threadIdx.x; k < 2 * kExDigits; k += kRedThreads) {
      P.digit[k / kExDigits][k % kExDigits] = (long long)sh.digit[k / kExDigits][k % kExDigits];
      sh.digit[k / kExDigits][k % kExDigits] = 0;
    }
    if (threadIdx.x < 2) {
      P.flags[threadIdx.x] = sh.flags[threadIdx.x];
      sh.flags[threadIdx.x] = 0;
    }
  }
}

// Exact launch 2, one block per item: min / max of its tile partials by reduce_items_kernel's tree in tile order; the
// digit counters added over the tiles (each split into its low 32 bits and its signed high part, so every addend is
// below 2^32 in magnitude and 2^31 tiles cannot overflow), then carried into the canonical two's complement words.
__global__ void __launch_bounds__(kExCombineThreads) reduce_exact_items_kernel(const RedItem *__restrict__ items, RedExactPartial *part,
                                                                               sb_reduce_exact_part *__restrict__ out) {
  constexpr int kCols = 2 * kExDigits, kGroups = kExCombineThreads / kCols;
  __shared__ long long lo[kGroups][kCols], hi[kGroups][kCols];
  __shared__ unsigned flags[2];
  const unsigned n = items[blockIdx.x].ntiles;
  RedExactPartial *p = part + items[blockIdx.x].tile0;
  if (threadIdx.x < 2) flags[threadIdx.x] = 0;
  __syncthreads();
  const int col = int(threadIdx.x) % kCols, grp = int(threadIdx.x) / kCols;
  if (grp < kGroups) {
    long long l = 0, h = 0;
    unsigned f = 0;
    const int w = col / kExDigits, k = col % kExDigits;
    for (unsigned j = unsigned(grp); j < n; j += kGroups) {
      const long long x = p[j].digit[w][k];
      l += x & 0xffffffffll;
      h += x >> 32;
      if (k == 0) f |= p[j].flags[w];
    }
    lo[grp][col] = l;
    hi[grp][col] = h;
    if (k == 0) atomicOr(&flags[w], f);
  }
  __syncthreads(); // every counter is read before the min / max tree rewrites the partials
  for (unsigned long long s = 1; s < n; s <<= 1) {
    for (unsigned long long i = threadIdx.x * 2 * s; i + s < n; i += 2 * s * kExCombineThreads) {
      p[i].min = red_min(p[i].min, p[i + s].min);
      p[i].max = red_max(p[i].max, p[i + s].max);
    }
    __syncthreads();
  }
  sb_reduce_exact_part &o = out[blockIdx.x];
  if (threadIdx.x < 2) {
    const int w = int(threadIdx.x);
    sb_exact_sum &e = w ? o.sumsq : o.sum;
    ex_carry(lo, hi, w, e);
    e.flags = flags[w];
  }
  if (0 == threadIdx.x) {
    o.count = items[blockIdx.x].count;
    o.min = n ? p[0].min : pos_inf();
    o.max = n ? p[0].max : -pos_inf();
  }
}

using ExactClassKernel = void (*)(const RedItem *, const RedTile *, unsigned, unsigned, RedExactPartial *);
ExactClassKernel exact_class_kernel(int c) {
  static const ExactClassKernel k[kRedClasses] = {
      reduce_exact_tiles_kernel<float, SB_REDUCE_SCALAR, false>,  reduce_exact_tiles_kernel<float, SB_REDUCE_SCALAR, true>,
      reduce_exact_tiles_kernel<float, SB_REDUCE_DIFF, false>,    reduce_exact_tiles_kernel<float, SB_REDUCE_DIFF, true>,
      reduce_exact_tiles_kernel<float, SB_REDUCE_NORM3, false>,   reduce_exact_tiles_kernel<float, SB_REDUCE_NORM3, true>,
      reduce_exact_tiles_kernel<double, SB_REDUCE_SCALAR, false>, reduce_exact_tiles_kernel<double, SB_REDUCE_SCALAR, true>,
      reduce_exact_tiles_kernel<double, SB_REDUCE_DIFF, false>,   reduce_exact_tiles_kernel<double, SB_REDUCE_DIFF, true>,
      reduce_exact_tiles_kernel<double, SB_REDUCE_NORM3, false>,  reduce_exact_tiles_kernel<double, SB_REDUCE_NORM3, true>};
  return k[c];
}

} // namespace

int reduce_exact_grid(int device, int cls, unsigned ntiles) {
  return persistent_grid(device, reinterpret_cast<const void *>(exact_class_kernel(cls)), ntiles);
}

int launch_reduce_exact(const RedItem *items_dev, unsigned nitems, const RedTile *tiles_dev, const unsigned (*class_tiles)[2], const int *grids,
                        RedExactPartial *scratch, sb_reduce_exact_part *out, cudaStream_t stream) {
  int launches = 0;
  for (int c = 0; c < kRedClasses; ++c) {
    if (class_tiles[c][1] > class_tiles[c][0]) {
      exact_class_kernel(c)<<<grids[c], kRedThreads, 0, stream>>>(items_dev, tiles_dev, class_tiles[c][0], class_tiles[c][1], scratch);
      ++launches;
    }
  }
  reduce_exact_items_kernel<<<nitems, kExCombineThreads, 0, stream>>>(items_dev, scratch, out);
  return launches + 1;
}

} // namespace sb
