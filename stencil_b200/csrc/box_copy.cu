// Box-copy kernels (see box_copy.cuh for the design).  sm_90a only.
#include "box_copy.cuh"

namespace sb {

namespace {

// Halo source cells are read exactly once and never written by the same launch (sources are compute
// cells, destinations ghost cells or dense buffers).  Wide rows go through the read-only path
// (ld.global.nc), thin strided rows through plain loads rather than evict-first .cs loads
// (scripts/time_pack.py times both).
template <typename V> __device__ __forceinline__ V ld_wide(const V *p) { return __ldg(p); }
template <> __device__ __forceinline__ unsigned char ld_wide(const unsigned char *p) { return *p; }
template <> __device__ __forceinline__ unsigned short ld_wide(const unsigned short *p) { return *p; }
template <typename V> __device__ __forceinline__ V ld_thin(const V *p) { return *p; }

// Row index -> (plane, row-in-plane) without an integer divide.
__device__ __forceinline__ void split_row(const Seg &s, unsigned R, unsigned &z, unsigned &y) {
  z = (unsigned)(((unsigned long long)R * s.ny_magic) >> s.ny_shift);
  y = R - z * s.ny;
}

template <typename V> __device__ __forceinline__ void copy_tile(const Seg &s, unsigned row0, unsigned nrows) {
  const unsigned lg = s.lg_group;
  const unsigned g = 1u << lg;
  const unsigned lane = threadIdx.x & (g - 1);
  const unsigned rsub = threadIdx.x >> lg;
  const unsigned rows_per_pass = kCopyThreads >> lg;
  const unsigned nvec = s.row_bytes / (unsigned)sizeof(V);

  if (nvec <= g) {
    // Thin rows (x-faces, edges, corners): one access per row; keep 4 rows in flight per thread.
    if (lane >= nvec) return;
    for (unsigned r = rsub; r < nrows; r += 4 * rows_per_pass) {
      V v[4];
      char *d[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const unsigned rr = r + k * rows_per_pass;
        d[k] = nullptr;
        if (rr < nrows) {
          unsigned z, y;
          split_row(s, row0 + rr, z, y);
          const V *sp = reinterpret_cast<const V *>(s.src + z * s.src_slice + y * s.src_pitch) + lane;
          d[k] = s.dst + z * s.dst_slice + y * s.dst_pitch;
          v[k] = ld_thin(sp);
        }
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (d[k]) reinterpret_cast<V *>(d[k])[lane] = v[k];
      }
    }
  } else {
    // Wide rows (y/z faces, yz edges, dense buffers): a lane group streams each row.
    for (unsigned r = rsub; r < nrows; r += rows_per_pass) {
      unsigned z, y;
      split_row(s, row0 + r, z, y);
      const V *sp = reinterpret_cast<const V *>(s.src + z * s.src_slice + y * s.src_pitch);
      V *dp = reinterpret_cast<V *>(s.dst + z * s.dst_slice + y * s.dst_pitch);
      for (unsigned c = lane; c < nvec; c += 4 * g) {
        V v[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned cc = c + k * g;
          if (cc < nvec) v[k] = ld_wide(sp + cc);
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned cc = c + k * g;
          if (cc < nvec) dp[cc] = v[k];
        }
      }
    }
  }
}

__device__ __forceinline__ void copy_tile_dispatch(const Seg &s, unsigned row0, unsigned nrows) {
  switch (s.vec) {
  case 16:
    copy_tile<uint4>(s, row0, nrows);
    break;
  case 8:
    copy_tile<uint2>(s, row0, nrows);
    break;
  case 4:
    copy_tile<unsigned>(s, row0, nrows);
    break;
  case 2:
    copy_tile<unsigned short>(s, row0, nrows);
    break;
  default:
    copy_tile<unsigned char>(s, row0, nrows);
    break;
  }
}

// ------------------------------------------------------------------------------------------- TMA tiles
constexpr int kTmaStages = 4;
constexpr unsigned kTmaStageBytes = 8192;

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "SB_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra SB_DONE_%=;\n"
      "bra SB_WAIT_%=;\n"
      "SB_DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *smem, const void *map, unsigned long long *bar, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   smem_u32(smem)),
               "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void *map, const void *smem, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(map), "r"(smem_u32(smem)),
               "r"(x), "r"(y), "r"(z)
               : "memory");
}

// executed by ONE thread of the CTA
__device__ void tma_tile(const TmaSeg &t, const void *smap, const void *dmap, unsigned row0, unsigned nrows, unsigned char *ring,
                         unsigned long long *bars, unsigned &phases) {
  const unsigned per_group = kTmaStageBytes / t.cstride; // chunks per ring stage (>= 4: chunks are <= 2 KiB)
  const unsigned total = nrows * t.chunks_per_row;
  const unsigned ngroups = (total + per_group - 1) / per_group;

  auto coords = [&](unsigned c, int &cx, int &y, int &z) {
    const unsigned r = row0 + c / t.chunks_per_row;
    const unsigned zz = (unsigned)(((unsigned long long)r * t.ny_magic) >> t.ny_shift);
    cx = (int)((c % t.chunks_per_row) * t.bx);
    y = (int)(r - zz * t.ny);
    z = (int)zz;
  };
  auto issue_loads = [&](unsigned g) {
    const unsigned s = g % kTmaStages;
    const unsigned first = g * per_group;
    const unsigned n = (total - first < per_group) ? total - first : per_group;
    mbar_expect_tx(&bars[s], n * t.chunk_bytes);
    for (unsigned k = 0; k < n; ++k) {
      int cx, y, z;
      coords(first + k, cx, y, z);
      tma_load_3d(ring + s * kTmaStageBytes + k * t.cstride, smap, &bars[s], t.sx0 + cx, t.sy0 + y, t.sz0 + z);
    }
  };

  for (unsigned g = 0; g < ngroups && g < kTmaStages - 1; ++g) issue_loads(g);
  for (unsigned g = 0; g < ngroups; ++g) {
    const unsigned s = g % kTmaStages;
    mbar_wait(&bars[s], (phases >> s) & 1u);
    phases ^= 1u << s;
    const unsigned first = g * per_group;
    const unsigned n = (total - first < per_group) ? total - first : per_group;
    for (unsigned k = 0; k < n; ++k) {
      int cx, y, z;
      coords(first + k, cx, y, z);
      tma_store_3d(dmap, ring + s * kTmaStageBytes + k * t.cstride, t.dx0 + cx, t.dy0 + y, t.dz0 + z);
    }
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    const unsigned gn = g + kTmaStages - 1;
    if (gn < ngroups) {
      // the ring slot of group gn was last used by group g-1: its stores must have finished READING it
      asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      issue_loads(gn);
    }
  }
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// Persistent walk over the tile table: grid is a multiple of the SM count, tiles are taken
// round-robin so consecutive CTAs stream consecutive rows of the same segment.
// kind 2: one thread feeds the ring with TMA loads, all threads drain it with vector stores
__device__ void tma_ld_tile(const TmaSeg &t, const void *smap, unsigned row0, unsigned nrows, unsigned char *ring, unsigned long long *bars,
                            unsigned &phases) {
  const unsigned per_group = kTmaStageBytes / t.cstride;
  const unsigned total = nrows * t.chunks_per_row;
  const unsigned ngroups = (total + per_group - 1) / per_group;
  const unsigned box_bytes = t.bxa * t.es;
  const unsigned po = t.pre * t.es;        // payload offset inside a chunk image
  const unsigned pay = t.chunk_bytes;      // payload bytes per chunk

  auto coords = [&](unsigned c, unsigned &cxe, unsigned &y, unsigned &z) {
    const unsigned r = row0 + c / t.chunks_per_row;
    z = (unsigned)(((unsigned long long)r * t.ny_magic) >> t.ny_shift);
    y = r - z * t.ny;
    cxe = (c % t.chunks_per_row) * t.bx; // payload element offset of this chunk inside its row
  };
  auto issue_loads = [&](unsigned g) { // thread 0 only
    const unsigned s = g % kTmaStages;
    const unsigned first = g * per_group;
    const unsigned n = (total - first < per_group) ? total - first : per_group;
    mbar_expect_tx(&bars[s], n * box_bytes);
    for (unsigned k = 0; k < n; ++k) {
      unsigned cxe, y, z;
      coords(first + k, cxe, y, z);
      tma_load_3d(ring + s * kTmaStageBytes + k * t.cstride, smap, &bars[s], t.sx0 - (int)t.pre + (int)cxe, t.sy0 + (int)y, t.sz0 + (int)z);
    }
  };

  if (threadIdx.x == 0)
    for (unsigned g = 0; g < ngroups && g < kTmaStages - 1; ++g) issue_loads(g);

  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (unsigned g = 0; g < ngroups; ++g) {
    // everybody has finished reading the slot that is refilled next (group g-1's)
    __syncthreads();
    if (threadIdx.x == 0 && g + kTmaStages - 1 < ngroups) issue_loads(g + kTmaStages - 1);
    const unsigned s = g % kTmaStages;
    mbar_wait(&bars[s], (phases >> s) & 1u);
    phases ^= 1u << s;
    const unsigned first = g * per_group;
    const unsigned n = (total - first < per_group) ? total - first : per_group;
    // one warp per chunk
    for (unsigned k = warp; k < n; k += kCopyThreads / 32) {
      unsigned cxe, y, z;
      coords(first + k, cxe, y, z);
      const unsigned char *img = ring + s * kTmaStageBytes + k * t.cstride;
      char *d = t.dst + (long long)z * t.dst_slice + (long long)y * t.dst_pitch + (long long)cxe * t.es;
      if (t.same_phase) {
        // 16-byte vectors of the aligned image; the first and last may hold ghost / trailing bytes
        char *dal = d - po;
        const unsigned nv = box_bytes / 16;
        for (unsigned j = lane; j < nv; j += 32) {
          const uint4 v = *reinterpret_cast<const uint4 *>(img + 16 * j);
          const unsigned lo = (16 * j < po) ? po : 16 * j;
          const unsigned hi = (16 * j + 16 > po + pay) ? po + pay : 16 * j + 16;
          if (hi - lo == 16) {
            *reinterpret_cast<uint4 *>(dal + 16 * j) = v;
          } else if (hi > lo) {
            const unsigned char *vb = reinterpret_cast<const unsigned char *>(&v);
            if (t.es == 8) {
              for (unsigned b = lo; b < hi; b += 8)
                *reinterpret_cast<unsigned long long *>(dal + b) = *reinterpret_cast<const unsigned long long *>(vb + (b - 16 * j));
            } else {
              for (unsigned b = lo; b < hi; b += 4)
                *reinterpret_cast<unsigned *>(dal + b) = *reinterpret_cast<const unsigned *>(vb + (b - 16 * j));
            }
          }
        }
      } else if (t.vec == 8) {
        for (unsigned j = lane; j < pay / 8; j += 32)
          reinterpret_cast<unsigned long long *>(d)[j] = *reinterpret_cast<const unsigned long long *>(img + po + 8 * j);
      } else {
        for (unsigned j = lane; j < pay / 4; j += 32) reinterpret_cast<unsigned *>(d)[j] = *reinterpret_cast<const unsigned *>(img + po + 4 * j);
      }
    }
  }
}

template <bool TMA> struct CopyShared {
  Seg seg;
  Tile tile;
};
template <> struct CopyShared<true> {
  alignas(128) unsigned char ring[kTmaStages * kTmaStageBytes];
  alignas(8) unsigned long long bars[kTmaStages];
  Seg seg;
  Tile tile;
};

template <bool TMA>
__device__ __forceinline__ void box_copy_body(CopyShared<TMA> &sh, const Seg *__restrict__ segs, const TmaSeg *__restrict__ tsegs,
                                              const TmaMaps *maps, const Tile *__restrict__ tiles, unsigned ntiles) {
  Seg &seg = sh.seg;
  Tile &tile = sh.tile;
  unsigned cached = 0xFFFFFFFFu;
  unsigned phases = 0; // parity of each ring barrier (thread 0)
  if constexpr (TMA) {
    if (threadIdx.x == 0) {
      for (int i = 0; i < kTmaStages; ++i) mbar_init(&sh.bars[i], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
  }
  for (unsigned t = blockIdx.x; t < ntiles; t += gridDim.x) {
    __syncthreads(); // previous tile done before the descriptors are replaced
    if (threadIdx.x == 0) tile = tiles[t];
    __syncthreads();
    if constexpr (TMA) {
      if (tile.kind == 1) { // TMA tile: one elected thread drives the copy engine
        __shared__ TmaSeg ts1;
        if (threadIdx.x == 0) ts1 = tsegs[tile.seg];
        __syncthreads();
        unsigned mine = phases;
        if (threadIdx.x == 0) tma_tile(ts1, &maps->m[ts1.smap][0], &maps->m[ts1.dmap][0], tile.row0, tile.nrows, sh.ring, sh.bars, mine);
        // every thread keeps the ring-barrier parities in step (kind-2 tiles wait on them with all threads)
        const unsigned per_group = kTmaStageBytes / ts1.cstride;
        const unsigned ngroups = (tile.nrows * ts1.chunks_per_row + per_group - 1) / per_group;
#pragma unroll
        for (unsigned st = 0; st < kTmaStages; ++st)
          if (((ngroups + kTmaStages - 1 - st) / kTmaStages) & 1u) phases ^= 1u << st;
        continue;
      }
      if (tile.kind == 2) { // TMA loads by one thread, vector stores by all
        __shared__ TmaSeg ts2;
        if (threadIdx.x == 0) ts2 = tsegs[tile.seg];
        __syncthreads();
        tma_ld_tile(ts2, &maps->m[ts2.smap][0], tile.row0, tile.nrows, sh.ring, sh.bars, phases);
        continue;
      }
    }
    if (tile.seg != cached) {
      // cooperative 80-byte descriptor fetch
      if (threadIdx.x < sizeof(Seg) / 4)
        reinterpret_cast<unsigned *>(&seg)[threadIdx.x] = reinterpret_cast<const unsigned *>(&segs[tile.seg])[threadIdx.x];
      cached = tile.seg;
      __syncthreads();
    }
    copy_tile_dispatch(seg, tile.row0, tile.nrows);
  }
}

__global__ void __launch_bounds__(kCopyThreads, 3)
    box_copy_kernel(const Seg *__restrict__ segs, const Tile *__restrict__ tiles, unsigned ntiles) {
  __shared__ CopyShared<false> sh;
  box_copy_body<false>(sh, segs, nullptr, nullptr, tiles, ntiles);
}

// Same walk, plus TMA tiles; the tensor maps are a __grid_constant__ parameter.
__global__ void __launch_bounds__(kCopyThreads, 3)
    box_copy_tma_kernel(const Seg *__restrict__ segs, const TmaSeg *__restrict__ tsegs, const __grid_constant__ TmaMaps maps,
                        const Tile *__restrict__ tiles, unsigned ntiles) {
  __shared__ CopyShared<true> sh;
  box_copy_body<true>(sh, segs, tsegs, &maps, tiles, ntiles);
}

// One segment passed by value: the pack_kernel / unpack_kernel / translate one-shots.
__global__ void __launch_bounds__(kCopyThreads, 3) box_copy_single_kernel(const __grid_constant__ Seg seg, unsigned rows_per_tile) {
  const unsigned total = seg.ny * seg.nz;
  for (unsigned long long row0 = (unsigned long long)blockIdx.x * rows_per_tile; row0 < total;
       row0 += (unsigned long long)gridDim.x * rows_per_tile) {
    // NOTE: written as end = min(row0 + rpt, total); nrows = end - row0.  The natural
    // min(total - row0, rpt) is miscompiled by ptxas 12.9 for sm_100a (Blackwell): the subtract and the minimum
    // are fused into VIADDMNMX.U32 with the negation dropped (it computes min(row0 + total, rpt)),
    // which turned every partial last tile into a full one (caught by tests/test_gpu_copy.py cases 7, 11).
    const unsigned long long stop = row0 + rows_per_tile;
    const unsigned end = stop < total ? (unsigned)stop : total;
    copy_tile_dispatch(seg, (unsigned)row0, end - (unsigned)row0);
  }
}

} // namespace

void launch_box_copy(const Seg *segs_dev, const TmaSeg *tsegs_dev, const TmaMaps *maps_host, const Tile *tiles_dev, unsigned ntiles, int grid,
                     cudaStream_t stream) {
  if (tsegs_dev != nullptr && maps_host != nullptr)
    box_copy_tma_kernel<<<grid, kCopyThreads, 0, stream>>>(segs_dev, tsegs_dev, *maps_host, tiles_dev, ntiles);
  else
    box_copy_kernel<<<grid, kCopyThreads, 0, stream>>>(segs_dev, tiles_dev, ntiles);
}

unsigned rows_per_tile_for(unsigned row_bytes) {
  // a thin row costs at least one 32-byte sector on each side however few bytes it carries
  const unsigned cost = row_bytes < 32u ? 32u : row_bytes;
  const unsigned rows = kTileBytes / cost;
  return rows < 1 ? 1 : rows;
}

void preload_box_copy_kernels() {
  // CUDA loads kernels lazily: resolve them at plan-creation time so the first exchange does not pay
  // the module load (bench_pack of the reference has no warm-up iteration)
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, box_copy_kernel);
  cudaFuncGetAttributes(&a, box_copy_tma_kernel);
  cudaFuncGetAttributes(&a, box_copy_single_kernel);
}

void launch_box_copy_single(const Seg &seg, cudaStream_t stream) {
  const unsigned total = seg.ny * seg.nz;
  const unsigned rows_per_tile = rows_per_tile_for(seg.row_bytes);
  unsigned ntiles = (total + rows_per_tile - 1) / rows_per_tile;
  if (ntiles == 0) return;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const unsigned cap = unsigned(sms > 0 ? sms : 1) * 8u;
  box_copy_single_kernel<<<ntiles < cap ? ntiles : cap, kCopyThreads, 0, stream>>>(seg, rows_per_tile);
}

} // namespace sb
