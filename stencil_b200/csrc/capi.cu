// C ABI of stencil_b200 (include/stencil_b200.h): geometry wrappers over the C++ host mirror
// (include/stencil/*.hpp), copy plans over box_copy.cu, jacobi launches, device/peer/IPC plumbing.
#include "stencil_b200.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include <cuda_runtime.h>

#include "box_copy.cuh"
#include "boundary.cuh"
#include "reduce.cuh"
#include "astaroth.cuh"
#include "jacobi.cuh"
#include "krylov.cuh"
#include "stencil_op.cuh"
#include "stencil_sys.cuh"
#include "transfer.cuh"

#include "stencil/exchange_plan.hpp"
#include "stencil/geometry.hpp"
#include "stencil/partition_core.hpp"

namespace {

thread_local std::string g_err;
std::atomic<uint64_t> g_launches{0};

int fail(sb_status code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return int(code);
}

#define SB_CUDA(expr)                                                                                                  \
  do {                                                                                                                 \
    cudaError_t e_ = (expr);                                                                                           \
    if (e_ != cudaSuccess) return fail(SB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) {
      ok = false;
      return;
    }
    if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// A cudaMalloc block of a plan (a table uploaded at creation, or scratch), freed on its device with the plan.
template <class T> struct DeviceTable {
  int device = 0;
  T *ptr = nullptr;
  DeviceTable() = default;
  DeviceTable(const DeviceTable &) = delete;
  DeviceTable &operator=(const DeviceTable &) = delete;
  ~DeviceTable() {
    if (!ptr) return;
    DeviceGuard guard(device);
    cudaFree(ptr);
  }
  // n elements on dev, the current device, the first host.size() of them copied from host
  cudaError_t upload(int dev, const std::vector<T> &host, size_t n) {
    device = dev;
    cudaError_t e = cudaMalloc(&ptr, n * sizeof(T));
    if (e == cudaSuccess && !host.empty()) e = cudaMemcpy(ptr, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice);
    return e;
  }
};

// The kernel launches of a stencil or transfer plan, in order: each holds its parameters by value and returns the
// number of launches it issued (the launch_* functions of the kernel headers).
struct LaunchList {
  int device = 0;
  int64_t bytes = 0;
  std::vector<std::function<int(cudaStream_t)>> launches;
};

int run_launches(const LaunchList *p, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (p->launches.empty()) return SB_OK;
  DeviceGuard guard(p->device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", p->device);
  for (const auto &launch : p->launches) g_launches += uint64_t(launch(static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// The compute entry points take pointers and a stream but no device: the launch must happen on the device that owns the
// memory (and the stream), whatever the calling thread's current device is -- a caller that drives several GPUs (or a test
// that ran on another GPU before) would otherwise get "invalid resource handle" from the launch.
int device_of(const void *ptr) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
}
struct PtrDeviceGuard {
  int prev = -1;
  explicit PtrDeviceGuard(const void *ptr) {
    const int dev = device_of(ptr);
    int cur = -1;
    if (dev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != dev && cudaSetDevice(dev) == cudaSuccess) prev = cur;
  }
  ~PtrDeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

Dim3 d3(const int64_t v[3]) { return Dim3(v[0], v[1], v[2]); }
void put(const Dim3 &d, int64_t out[3]) {
  out[0] = d.x;
  out[1] = d.y;
  out[2] = d.z;
}
Radius radius_of(const int64_t r27[27]) {
  Radius r = Radius::constant(0);
  int i = 0;
  for (int z = -1; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) r.dir(x, y, z) = size_t(r27[i++]);
  return r;
}
bool dir_ok(const int64_t d[3]) {
  for (int a = 0; a < 3; ++a)
    if (d[a] < -1 || d[a] > 1) return false;
  return true;
}

unsigned ceil_log2(unsigned v) {
  unsigned b = 0;
  while ((1ull << b) < v) ++b;
  return b;
}

// Turn one sb_box_copy into >= 1 kernel segments (see box_copy.cuh).
int build_segments(const sb_box_copy &c, std::vector<sb::Seg> &out) {
  const int64_t es = c.elem_size;
  if (es <= 0 || (es & (es - 1)) != 0 || es > 16) return fail(SB_ERR_INVALID, "elem_size %lld must be 1,2,4,8 or 16", (long long)es);
  for (int a = 0; a < 3; ++a) {
    if (c.extent[a] < 0 || c.src_pos[a] < 0 || c.dst_pos[a] < 0) return fail(SB_ERR_INVALID, "negative extent/position");
  }
  if (c.extent[0] == 0 || c.extent[1] == 0 || c.extent[2] == 0) return SB_OK; // empty box: nothing to do
  if (!c.src.ptr || !c.dst.ptr) return fail(SB_ERR_INVALID, "null pointer in box copy");
  if (c.src.pitch <= 0 || c.dst.pitch <= 0 || c.src.ysize <= 0 || c.dst.ysize <= 0)
    return fail(SB_ERR_INVALID, "pitch/ysize must be positive");

  long long row_bytes = c.extent[0] * es;
  long long ny = c.extent[1], nz = c.extent[2];
  long long sp = c.src.pitch, ss = c.src.pitch * c.src.ysize;
  long long dp = c.dst.pitch, ds = c.dst.pitch * c.dst.ysize;
  const char *src = static_cast<const char *>(c.src.ptr) + (c.src_pos[2] * c.src.ysize + c.src_pos[1]) * c.src.pitch + c.src_pos[0] * es;
  char *dst = static_cast<char *>(c.dst.ptr) + (c.dst_pos[2] * c.dst.ysize + c.dst_pos[1]) * c.dst.pitch + c.dst_pos[0] * es;

  // merge dimensions that are contiguous on BOTH sides (full-width rows / full planes)
  const long long kMaxRow = 1ll << 30;
  if (ny > 1 && sp == row_bytes && dp == row_bytes && row_bytes * ny < kMaxRow) {
    row_bytes *= ny;
    ny = 1;
  }
  if (ny == 1 && nz > 1 && ss == row_bytes && ds == row_bytes && row_bytes * nz < kMaxRow) {
    row_bytes *= nz;
    nz = 1;
  }
  if (ny == 1 && nz > 1) { // a single row per plane: planes become the rows
    ny = nz;
    nz = 1;
    sp = ss;
    dp = ds;
  }
  if (row_bytes >= (1ll << 31)) return fail(SB_ERR_INVALID, "row of %lld bytes too long", row_bytes);

  auto emit = [&](const char *s, char *d, long long rb, long long rows_y, long long rows_z, long long spitch, long long sslice,
                  long long dpitch, long long dslice) -> int {
    // keep rows per segment below 2^24 (range of the divide-free row split)
    const long long kMaxRows = (1ll << 24) - 1;
    if (rows_y > kMaxRows) return fail(SB_ERR_INVALID, "more than 2^24 rows per plane");
    long long zmax = kMaxRows / rows_y;
    for (long long z0 = 0; z0 < rows_z; z0 += zmax) {
      const long long zn = (rows_z - z0 < zmax) ? rows_z - z0 : zmax;
      sb::Seg g{};
      g.src = s + z0 * sslice;
      g.dst = d + z0 * dslice;
      g.src_pitch = spitch;
      g.src_slice = sslice;
      g.dst_pitch = dpitch;
      g.dst_slice = dslice;
      g.row_bytes = unsigned(rb);
      g.ny = unsigned(rows_y);
      g.nz = unsigned(zn);
      unsigned long long align = (unsigned long long)(uintptr_t)g.src | (unsigned long long)(uintptr_t)g.dst | (unsigned long long)rb;
      if (rows_y > 1) align |= (unsigned long long)spitch | (unsigned long long)dpitch;
      if (zn > 1) align |= (unsigned long long)sslice | (unsigned long long)dslice;
      unsigned vec = 16;
      while (vec > 1 && (align & (vec - 1))) vec >>= 1;
      g.vec = vec;
      const unsigned nvec = unsigned(rb) / vec;
      unsigned lg = ceil_log2(nvec);
      if (lg > 5) lg = 5;
      g.lg_group = lg;
      const unsigned bits = ceil_log2(unsigned(rows_y));
      g.ny_shift = 24 + bits;
      g.ny_magic = ((1ull << g.ny_shift) + unsigned(rows_y) - 1) / unsigned(rows_y);
      out.push_back(g);
    }
    return SB_OK;
  };

  if (ny == 1 && nz == 1 && row_bytes > 2 * (long long)sb::kTileBytes) {
    // one long contiguous run: cut it into tile-sized "rows"
    const long long chunk = sb::kTileBytes;
    const long long q = row_bytes / chunk, rem = row_bytes % chunk;
    int rc = emit(src, dst, chunk, q, 1, chunk, chunk * q, chunk, chunk * q);
    if (rc != SB_OK) return rc;
    if (rem) rc = emit(src + q * chunk, dst + q * chunk, rem, 1, 1, rem, rem, rem, rem);
    return rc;
  }
  return emit(src, dst, row_bytes, ny, nz, sp, ss, dp, ds);
}

void build_tiles(const std::vector<sb::Seg> &segs, std::vector<sb::Tile> &tiles) {
  for (size_t si = 0; si < segs.size(); ++si) {
    const sb::Seg &g = segs[si];
    const unsigned rows_per_tile = sb::rows_per_tile_for(g.row_bytes);
    const unsigned total = g.ny * g.nz;
    for (unsigned r = 0; r < total; r += rows_per_tile) {
      sb::Tile t{};
      t.seg = unsigned(si);
      t.row0 = r;
      t.nrows = (total - r < rows_per_tile) ? total - r : rows_per_tile;
      tiles.push_back(t);
    }
  }
}

struct SlotTable {
  uint32_t *p[64];
};

__global__ void signal_kernel(const __grid_constant__ SlotTable slots, int n, uint32_t value) {
  // all earlier work of this stream is complete (stream order); publish it system-wide
  __threadfence_system();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(slots.p[i]), "r"(value) : "memory");
  }
}

__global__ void wait_kernel(const uint32_t *slots, int n, uint32_t value) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(slots + i) : "memory");
      if ((int32_t)(v - value) >= 0) break; // wrap-safe "v >= value"
      __nanosleep(64);
    } while (true);
  }
  __threadfence_system();
}

// ------------------------------------------------------------------------------------------- boundary conditions
const char *const kFaceName[6] = {"-x", "+x", "-y", "+y", "-z", "+z"};

// The BC regions of one subdomain (the geometry behind sb_bc_regions and sb_bc_plan_create).
int bc_regions(const int64_t size[3], const int64_t r27[27], const int32_t kinds[6], std::vector<sb_bc_region> &out) {
  if (!size || !r27 || !kinds) return fail(SB_ERR_INVALID, "null argument");
  for (int f = 0; f < 6; ++f) {
    if (kinds[f] < SB_BC_NONE || kinds[f] > SB_BC_ODD) return fail(SB_ERR_INVALID, "face %s: unknown BC kind %d", kFaceName[f], int(kinds[f]));
    const int a = f / 2, s = (f % 2) ? 1 : -1;
    const int64_t g = r27[(a == 2 ? s + 1 : 1) * 9 + (a == 1 ? s + 1 : 1) * 3 + (a == 0 ? s + 1 : 1)];
    if ((kinds[f] == SB_BC_EVEN || kinds[f] == SB_BC_ODD) && g > size[a])
      return fail(SB_ERR_INVALID, "face %s: EVEN and ODD mirror the compute cells, the ghost width %lld exceeds the subdomain's %lld cells",
                  kFaceName[f], (long long)g, (long long)size[a]);
  }
  const Radius r = radius_of(r27);
  const Dim3 sz = d3(size);
  for (int z = -1; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) {
        const int d[3] = {x, y, z};
        if ((0 == x && 0 == y && 0 == z) || 0 == r27[(z + 1) * 9 + (y + 1) * 3 + (x + 1)]) continue;
        int32_t faces = 0;
        for (int a = 0; a < 3; ++a)
          if (d[a] && kinds[2 * a + (d[a] > 0)] != SB_BC_NONE) faces |= 1 << (2 * a + (d[a] > 0));
        if (!faces) continue;
        const Dim3 dir(x, y, z);
        const Dim3 pos = stencil::geom::halo_pos(dir, sz, r, true), ext = stencil::geom::halo_extent(dir, sz, r);
        if (0 == ext.flatten()) continue;
        sb_bc_region reg{};
        put(dir, reg.dir);
        put(pos, reg.pos);
        put(ext, reg.extent);
        for (int a = 0; a < 3; ++a) {
          reg.mirror[a] = -1;
          if (!(faces & (3 << (2 * a)))) continue;
          const int64_t gm = a == 0 ? r.x(-1) : a == 1 ? r.y(-1) : r.z(-1);
          reg.mirror[a] = d[a] < 0 ? 2 * gm - 1 : 2 * (gm + size[a]) - 1;
        }
        reg.faces = faces;
        out.push_back(reg);
      }
  return SB_OK;
}

// ------------------------------------------------------------------------------------------- exchange plan
bool in_grid(const int64_t idx[3], const int64_t dim[3]) {
  for (int a = 0; a < 3; ++a)
    if (idx[a] < 0 || idx[a] >= dim[a]) return false;
  return true;
}

// The messages of src_idx (the arithmetic behind sb_exchange_messages and sb_staging_layout), after checking the grid.
int exchange_messages(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                      const int64_t r27[27], const int64_t src_idx[3], std::vector<stencil::Message> &out) {
  if (!dim || !base || !rem || !boundary || !r27 || !src_idx) return fail(SB_ERR_INVALID, "null argument");
  Topology::Boundary kind[3];
  for (int a = 0; a < 3; ++a) {
    if (dim[a] < 1) return fail(SB_ERR_INVALID, "the grid needs at least one subdomain per axis (dim[%d] = %lld)", a, (long long)dim[a]);
    if (boundary[a] != int32_t(Topology::Boundary::PERIODIC) && boundary[a] != int32_t(Topology::Boundary::FIXED))
      return fail(SB_ERR_INVALID, "boundary[%d] = %d: must be 1 (PERIODIC) or 2 (FIXED)", a, int(boundary[a]));
    kind[a] = Topology::Boundary(boundary[a]);
  }
  if (!in_grid(src_idx, dim)) return fail(SB_ERR_INVALID, "source subdomain index outside the grid");
  const stencil::detail::CutGrid grid{d3(base), d3(rem)};
  out = stencil::messages_from(d3(src_idx), Topology(d3(dim), kind[0], kind[1], kind[2]), radius_of(r27),
                               [&](const Dim3 &idx) { return grid.size_of(idx); });
  return SB_OK;
}

// ------------------------------------------------------------------------------------------- boxes of a plan
// The non-empty boxes of an operator, system or fused-restriction plan: lo in the destination's allocation coordinates,
// and the extent.  Thick boxes go to the tile kernel, one launch each; thin ones to the cell kernel in groups.
struct PlanBox {
  int lo[3], ext[3];
};
struct PlanBoxes {
  std::vector<PlanBox> thick, thin; // in box order
  int64_t cells = 0;
};

// Whether a non-empty box of extent e has 2^32 cells or more, without overflowing: the kernels count cells in 32 bits.
bool over_2_32_cells(const int64_t e[3]) {
  const int64_t cap = 1ll << 32;
  if (e[0] >= cap || e[1] >= cap || e[2] >= cap) return true;
  return uint64_t(e[0]) * uint64_t(e[1]) >= uint64_t((cap + e[2] - 1) / e[2]);
}

// Checks and sorts the nbox boxes [lo, hi) (global coordinates, 3 per box) of a destination whose allocation starts at
// acc_origin: a box is thick when its extent is at least `thick` on every axis.  reads(b, l, e) checks what box b reads
// (allocation-relative lo l, extent e) and returns SB_OK or its error; it checks a window that holds the box with
// stencil_box_reads_ok, so l and l + e fit an int.
template <class Reads>
int plan_boxes(int nbox, const int64_t *lo, const int64_t *hi, const int64_t acc_origin[3], int thick, Reads reads, PlanBoxes &out) {
  for (int b = 0; b < nbox; ++b) {
    int64_t l[3], e[3];
    bool empty = false;
    for (int a = 0; a < 3; ++a) {
      if (lo[3 * b + a] > hi[3 * b + a]) return fail(SB_ERR_INVALID, "box %d: lo > hi on axis %c", b, "xyz"[a]);
      l[a] = lo[3 * b + a] - acc_origin[a];
      e[a] = hi[3 * b + a] - lo[3 * b + a];
      empty = empty || e[a] == 0;
    }
    if (empty) continue;
    const int rc = reads(b, l, e);
    if (rc != SB_OK) return rc;
    if (over_2_32_cells(e)) return fail(SB_ERR_INVALID, "box %d: more than 2^32 cells", b);
    const PlanBox box = {{int(l[0]), int(l[1]), int(l[2])}, {int(e[0]), int(e[1]), int(e[2])}};
    (e[0] >= thick && e[1] >= thick && e[2] >= thick ? out.thick : out.thin).push_back(box);
    out.cells += e[0] * e[1] * e[2];
  }
  return SB_OK;
}

// The tile grid of a z-marching kernel (kernel: its name in the message) over a box of extent ext, in columns of tx x ty
// cells: z chunks for at least two waves of per_sm resident CTAs per SM, no shorter than min_chunk planes (each chunk
// reloads the planes around it).  Sets p.tiles_x, p.tiles_y and p.zchunk.
template <class P> int tile_grid(P &p, const int ext[3], int tx, int ty, int sms, int per_sm, int min_chunk, const char *kernel, int &grid) {
  p.tiles_x = (ext[0] + tx - 1) / tx;
  p.tiles_y = (ext[1] + ty - 1) / ty;
  const long long cols = (long long)p.tiles_x * p.tiles_y;
  const long long want = (2ll * sms * per_sm + cols - 1) / cols;
  p.zchunk = std::max(int((ext[2] + want - 1) / want), std::min(min_chunk, ext[2]));
  const long long g = cols * ((ext[2] + p.zchunk - 1) / p.zchunk);
  if (g >= (1ll << 31)) return fail(SB_ERR_INVALID, "box too large for the %s", kernel);
  grid = int(g);
  return SB_OK;
}

// The thin boxes in groups of as many as a cell kernel's parameters hold: each group is p with its boxes in lo / ext, its
// box count in p.*count and the prefix sums of their cells in first.  add(group, grid) takes each group in order; the
// grid has one thread per cell, at most 32 CTAs of 256 per SM.
template <class P, class Q, class Add> void cell_groups(const std::vector<PlanBox> &thin, const P &p, int Q::*count, int sms, Add add) {
  constexpr size_t kMax = std::extent<decltype(P::first)>::value - 1;
  for (size_t b0 = 0; b0 < thin.size(); b0 += kMax) {
    P g = p;
    g.first[0] = 0;
    for (size_t b = b0; b < thin.size() && b < b0 + kMax; ++b) {
      const int m = (g.*count)++;
      for (int a = 0; a < 3; ++a) {
        g.lo[m][a] = thin[b].lo[a];
        g.ext[m][a] = thin[b].ext[a];
      }
      g.first[m + 1] = g.first[m] + (long long)thin[b].ext[0] * thin[b].ext[1] * thin[b].ext[2];
    }
    add(g, int(std::min<long long>((g.first[g.*count] + 255) / 256, 32ll * sms)));
  }
}

} // namespace

struct sb_bc_plan {
  int device = 0;
  DeviceTable<sb::BcSeg> segs;
  DeviceTable<sb::BcTile> tiles;
  unsigned ntiles = 0;
  int grid = 0;
  int64_t bytes = 0;
};

// An ordered or exact reduction plan: Partial is the kernel's per-tile partial.
template <class Partial> struct ReducePlan {
  int device = 0;
  DeviceTable<sb::RedItem> items;
  DeviceTable<sb::RedTile> tiles;
  DeviceTable<Partial> scratch; // one partial per tile, rewritten by every launch
  unsigned nitems = 0;
  unsigned class_tiles[sb::kRedClasses][2] = {}; // tiles [begin, end) of each class
  int grids[sb::kRedClasses] = {};
  int64_t bytes = 0;
};
struct sb_reduce_plan : ReducePlan<sb::RedPartial> {};
struct sb_reduce_exact_plan : ReducePlan<sb::RedExactPartial> {};

struct sb_krylov_plan {
  int device = 0;
  int dtype = SB_DTYPE_F64, mode = 0; // mode: the kernel mode (krylov.cuh)
  bool wide = false;
  sb::KryParams params{};
  DeviceTable<sb::KryPartial> scratch; // one partial per tile, rewritten by every launch (modes with dots)
  int grid = 0, copy_grid = 0;
  int64_t bytes = 0;
};

struct sb_stencil_plan : LaunchList {};  // an operator or a system: tile launches in box order, then the cell groups
struct sb_transfer_plan : LaunchList {}; // no launch for an empty box

struct sb_copy_plan {
  int device = 0;
  DeviceTable<sb::Seg> segs;
  DeviceTable<sb::Tile> tiles;
  unsigned ntiles = 0;
  int grid = 0;
  int64_t bytes = 0;
};

extern "C" {

const char *sb_last_error(void) { return g_err.c_str(); }
int sb_version(void) { return SB_VERSION; }
uint64_t sb_launch_count(void) { return g_launches.load(); }

// ----------------------------------------------------------------------------------------- geometry
int sb_halo_pos(const int64_t dir[3], const int64_t size[3], const int64_t radius27[27], int halo, int64_t out[3]) {
  if (!dir_ok(dir)) return fail(SB_ERR_INVALID, "direction components must be in -1..1");
  put(stencil::geom::halo_pos(d3(dir), d3(size), radius_of(radius27), halo != 0), out);
  return SB_OK;
}
int sb_halo_extent(const int64_t dir[3], const int64_t size[3], const int64_t radius27[27], int64_t out[3]) {
  if (!dir_ok(dir)) return fail(SB_ERR_INVALID, "direction components must be in -1..1");
  put(stencil::geom::halo_extent(d3(dir), d3(size), radius_of(radius27)), out);
  return SB_OK;
}
int sb_raw_size(const int64_t size[3], const int64_t radius27[27], int64_t out[3]) {
  put(stencil::geom::raw_size(d3(size), radius_of(radius27)), out);
  return SB_OK;
}
int sb_prime_factors(int64_t n, int64_t *out, int cap) {
  if (n < 0) return fail(SB_ERR_INVALID, "n must be >= 0");
  const std::vector<int64_t> f = prime_factors<int64_t>(n);
  if (int(f.size()) > cap) return fail(SB_ERR_INVALID, "output capacity %d too small for %zu factors", cap, f.size());
  for (size_t i = 0; i < f.size(); ++i) out[i] = f[i];
  return int(f.size());
}
int sb_rank_partition(const int64_t size[3], int64_t n, int64_t dim[3], int64_t base[3], int64_t rem[3]) {
  if (n < 1) return fail(SB_ERR_INVALID, "n must be >= 1");
  RankPartition p(d3(size), n);
  const Dim3 d = p.dim();
  put(d, dim);
  put(p.subdomain_size(Dim3(0, 0, 0)), base);
  put(d3(size) % d, rem);
  return SB_OK;
}
int sb_node_partition(const int64_t size[3], const int64_t radius27[27], int64_t nodes, int64_t gpus, int64_t sys_dim[3],
                      int64_t node_dim[3], int64_t base[3], int64_t rem[3]) {
  if (nodes < 1 || gpus < 1) return fail(SB_ERR_INVALID, "nodes and gpus must be >= 1");
  NodePartition p(d3(size), radius_of(radius27), nodes, gpus);
  put(p.sys_dim(), sys_dim);
  put(p.node_dim(), node_dim);
  put(p.subdomain_size(Dim3(0, 0, 0)), base);
  put(d3(size) % p.dim(), rem);
  return SB_OK;
}
int sb_subdomain_size(const int64_t base[3], const int64_t rem[3], const int64_t idx[3], int64_t out[3]) {
  stencil::detail::CutGrid g{d3(base), d3(rem)};
  put(g.size_of(d3(idx)), out);
  return SB_OK;
}
int sb_subdomain_origin(const int64_t base[3], const int64_t rem[3], const int64_t idx[3], int64_t out[3]) {
  stencil::detail::CutGrid g{d3(base), d3(rem)};
  put(g.origin_of(d3(idx)), out);
  return SB_OK;
}
int sb_interior(const int64_t lo[3], const int64_t hi[3], const int64_t radius27[27], int64_t int_lo[3], int64_t int_hi[3]) {
  const Rect3 in = stencil::geom::interior(Rect3(d3(lo), d3(hi)), radius_of(radius27));
  put(in.lo, int_lo);
  put(in.hi, int_hi);
  return SB_OK;
}
int sb_exterior(const int64_t lo[3], const int64_t hi[3], const int64_t radius27[27], int64_t *ext_lo, int64_t *ext_hi) {
  const std::vector<Rect3> slabs = stencil::geom::exterior(Rect3(d3(lo), d3(hi)), radius_of(radius27));
  for (size_t i = 0; i < slabs.size(); ++i) {
    put(slabs[i].lo, ext_lo + 3 * i);
    put(slabs[i].hi, ext_hi + 3 * i);
  }
  return int(slabs.size());
}

// ----------------------------------------------------------------------------------------- box copies
static int one_shot(const sb_box_copy &c, void *stream) {
  PtrDeviceGuard guard(c.src.ptr); // launch where the source lives
  std::vector<sb::Seg> segs;
  int rc = build_segments(c, segs);
  if (rc != SB_OK) return rc;
  for (const sb::Seg &g : segs) {
    sb::launch_box_copy_single(g, static_cast<cudaStream_t>(stream));
    ++g_launches;
  }
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_pack(void *dst, sb_pitched src, const int64_t pos[3], const int64_t extent[3], int64_t elem_size, void *stream) {
  sb_box_copy c{};
  c.dst = sb_pitched{dst, extent[0] * elem_size, extent[1]};
  c.src = src;
  for (int a = 0; a < 3; ++a) {
    c.src_pos[a] = pos[a];
    c.extent[a] = extent[a];
  }
  c.elem_size = elem_size;
  return one_shot(c, stream);
}

int sb_unpack(sb_pitched dst, const void *src, const int64_t pos[3], const int64_t extent[3], int64_t elem_size, void *stream) {
  sb_box_copy c{};
  c.dst = dst;
  c.src = sb_pitched{const_cast<void *>(src), extent[0] * elem_size, extent[1]};
  for (int a = 0; a < 3; ++a) {
    c.dst_pos[a] = pos[a];
    c.extent[a] = extent[a];
  }
  c.elem_size = elem_size;
  return one_shot(c, stream);
}

int sb_translate(sb_pitched dst, const int64_t dst_pos[3], sb_pitched src, const int64_t src_pos[3], const int64_t extent[3],
                 int64_t elem_size, void *stream) {
  sb_box_copy c{};
  c.dst = dst;
  c.src = src;
  for (int a = 0; a < 3; ++a) {
    c.dst_pos[a] = dst_pos[a];
    c.src_pos[a] = src_pos[a];
    c.extent[a] = extent[a];
  }
  c.elem_size = elem_size;
  return one_shot(c, stream);
}

int sb_copy_plan_create(sb_copy_plan **out, int device, const sb_box_copy *copies, int64_t n) {
  if (!out || (n > 0 && !copies) || n < 0) return fail(SB_ERR_INVALID, "bad arguments to sb_copy_plan_create");
  std::vector<sb::Seg> segs;
  int64_t bytes = 0;
  for (int64_t i = 0; i < n; ++i) {
    bytes += copies[i].extent[0] * copies[i].extent[1] * copies[i].extent[2] * copies[i].elem_size;
    int rc = build_segments(copies[i], segs);
    if (rc != SB_OK) return rc;
  }
  std::vector<sb::Tile> tiles;
  build_tiles(segs, tiles);

  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  sb::preload_box_copy_kernels();
  std::unique_ptr<sb_copy_plan> p(new sb_copy_plan());
  p->device = device;
  p->bytes = bytes;
  p->ntiles = unsigned(tiles.size());
  if (p->ntiles) {
    SB_CUDA(p->segs.upload(device, segs, segs.size() + 1));
    SB_CUDA(p->tiles.upload(device, tiles, tiles.size()));
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    const long long cap = (long long)sms * sb::kCopyCtasPerSm;
    p->grid = int(p->ntiles < cap ? p->ntiles : cap);
  }
  *out = p.release();
  return SB_OK;
}

int sb_copy_plan_launch(sb_copy_plan *p, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (0 == p->ntiles) return SB_OK;
  DeviceGuard guard(p->device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", p->device);
  sb::launch_box_copy(p->segs.ptr, p->tiles.ptr, p->ntiles, p->grid, static_cast<cudaStream_t>(stream));
  ++g_launches;
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int64_t sb_copy_plan_bytes(const sb_copy_plan *p) { return p ? p->bytes : 0; }
int64_t sb_copy_plan_num_tiles(const sb_copy_plan *p) { return p ? p->ntiles : 0; }

int sb_copy_plan_destroy(sb_copy_plan *p) {
  delete p;
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- boundary conditions
int sb_bc_regions(const int64_t size[3], const int64_t radius27[27], const int32_t kinds[6], sb_bc_region *out, int cap) {
  if (cap < 0 || (cap > 0 && !out)) return fail(SB_ERR_INVALID, "bad output buffer");
  std::vector<sb_bc_region> regs;
  const int rc = bc_regions(size, radius27, kinds, regs);
  if (rc != SB_OK) return rc;
  for (size_t i = 0; i < regs.size() && int(i) < cap; ++i) out[i] = regs[i];
  return int(regs.size());
}

// ----------------------------------------------------------------------------------------- exchange plan
int sb_exchange_messages(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                         const int64_t radius27[27], const int64_t src_idx[3], sb_message *out, int cap) {
  std::vector<stencil::Message> msgs;
  const int rc = exchange_messages(dim, base, rem, boundary, radius27, src_idx, msgs);
  if (rc != SB_OK) return rc;
  if (cap < int(msgs.size()) || (!msgs.empty() && !out))
    return fail(SB_ERR_INVALID, "output capacity %d too small for %zu messages", cap, msgs.size());
  for (size_t i = 0; i < msgs.size(); ++i) {
    put(msgs[i].dir, out[i].dir);
    put(msgs[i].dstIdx, out[i].dst_idx);
    put(msgs[i].srcPos, out[i].src_pos);
    put(msgs[i].dstPos, out[i].dst_pos);
    put(msgs[i].ext, out[i].extent);
  }
  return int(msgs.size());
}

int sb_staging_layout(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                      const int64_t radius27[27], const int64_t src_idx[3], const int64_t dst_idx[3],
                      const int64_t *elem_sizes, int nq, sb_staged *out, int cap, int64_t *total) {
  return sb_staging_layout_subset(dim, base, rem, boundary, radius27, src_idx, dst_idx, elem_sizes, nq, stencil::kAllQuantities, out, cap, total);
}

int sb_staging_layout_subset(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                             const int64_t radius27[27], const int64_t src_idx[3], const int64_t dst_idx[3],
                             const int64_t *elem_sizes, int nq, uint64_t quantities, sb_staged *out, int cap, int64_t *total) {
  static_assert(SB_STAGE_MAX_ROW_BYTES == stencil::kStageMaxRowBytes, "one staging threshold");
  if (!dst_idx || !total || nq < 0 || (nq > 0 && !elem_sizes)) return fail(SB_ERR_INVALID, "bad arguments to sb_staging_layout");
  if (0 == quantities) return fail(SB_ERR_INVALID, "the quantity subset is empty");
  if (quantities != stencil::kAllQuantities)
    for (int q = 0; q < 64; ++q)
      if (((quantities >> q) & 1u) && q >= nq) return fail(SB_ERR_INVALID, "quantity %d is not one of the %d quantities", q, nq);
  std::vector<stencil::Message> msgs;
  const int rc = exchange_messages(dim, base, rem, boundary, radius27, src_idx, msgs);
  if (rc != SB_OK) return rc;
  if (!in_grid(dst_idx, dim)) return fail(SB_ERR_INVALID, "destination subdomain index outside the grid");
  for (int q = 0; q < nq; ++q)
    if (elem_sizes[q] <= 0) return fail(SB_ERR_INVALID, "quantity %d: elem_size %lld must be > 0", q, (long long)elem_sizes[q]);
  const std::vector<stencil::Staged> staged =
      stencil::staging_layout(msgs, d3(dst_idx), std::vector<int64_t>(elem_sizes, elem_sizes + nq), total, quantities);
  if (cap < int(staged.size()) || (!staged.empty() && !out))
    return fail(SB_ERR_INVALID, "output capacity %d too small for %zu staged entries", cap, staged.size());
  for (size_t i = 0; i < staged.size(); ++i) out[i] = sb_staged{int64_t(staged[i].msg), staged[i].q, staged[i].offset};
  return int(staged.size());
}

int sb_bc_plan_create(sb_bc_plan **out, int device, const sb_bc_quantity *quantities, int64_t n, const int64_t size[3],
                      const int64_t radius27[27]) {
  if (!out || n < 0 || (n > 0 && !quantities) || !size || !radius27) return fail(SB_ERR_INVALID, "bad arguments to sb_bc_plan_create");
  for (int a = 0; a < 3; ++a)
    if (size[a] < 1 || size[a] >= (1ll << 30)) return fail(SB_ERR_INVALID, "subdomain size must be in [1, 2^30) on every axis");
  std::vector<sb::BcSeg> segs;
  std::vector<sb::BcTile> tiles;
  int64_t bytes = 0;
  for (int64_t q = 0; q < n; ++q) {
    const sb_bc_quantity &Q = quantities[q];
    const int64_t es = Q.elem_size;
    if (Q.dtype == SB_DTYPE_RAW) {
      if (es <= 0 || (es & (es - 1)) || es > 16) return fail(SB_ERR_INVALID, "quantity %lld: elem_size %lld must be 1, 2, 4, 8 or 16", (long long)q, (long long)es);
    } else if (Q.dtype == SB_DTYPE_F32 || Q.dtype == SB_DTYPE_F64) {
      if (es != (Q.dtype == SB_DTYPE_F32 ? 4 : 8)) return fail(SB_ERR_INVALID, "quantity %lld: elem_size %lld does not match its dtype", (long long)q, (long long)es);
    } else {
      return fail(SB_ERR_INVALID, "quantity %lld: unknown dtype %d", (long long)q, int(Q.dtype));
    }
    for (int f = 0; f < 6; ++f)
      if (Q.dtype == SB_DTYPE_RAW && (Q.kind[f] == SB_BC_VALUE || Q.kind[f] == SB_BC_ODD))
        return fail(SB_ERR_INVALID, "quantity %lld, face %s: VALUE and ODD need a floating-point quantity (EVEN copies any type)", (long long)q, kFaceName[f]);
    std::vector<sb_bc_region> regs;
    int rc = bc_regions(size, radius27, Q.kind, regs);
    if (rc != SB_OK) return rc;
    if (regs.empty()) continue;
    if (!Q.data.ptr || Q.data.pitch <= 0 || Q.data.ysize <= 0) return fail(SB_ERR_INVALID, "quantity %lld: bad pitched pointer", (long long)q);
    if ((uintptr_t(Q.data.ptr) % uintptr_t(es)) || (Q.data.pitch % es))
      return fail(SB_ERR_INVALID, "quantity %lld: pointer and pitch must be multiples of the %lld-byte element", (long long)q, (long long)es);
    // a value in the quantity's type, carried as an (exact) double
    auto in_type = [&](double c) { return Q.dtype == SB_DTYPE_F32 ? double(float(c)) : c; };
    auto twice = [&](double c) { return Q.dtype == SB_DTYPE_F32 ? double(2.0f * float(c)) : 2.0 * c; };
    for (const sb_bc_region &reg : regs) {
      sb::BcSeg g{};
      g.base = static_cast<char *>(Q.data.ptr);
      g.pitch = Q.data.pitch;
      g.slice = Q.data.pitch * Q.data.ysize;
      for (int a = 0; a < 3; ++a) {
        g.pos[a] = int(reg.pos[a]);
        g.ext[a] = int(reg.extent[a]);
        g.mirror[a] = int(reg.mirror[a]);
      }
      g.read = 1;
      for (int a = 0; a < 3; ++a) { // wall faces in order x, y, z: a VALUE face restarts the chain, ODD appends a step
        if (reg.mirror[a] < 0) continue;
        const int f = 2 * a + (reg.dir[a] > 0);
        if (Q.kind[f] == SB_BC_VALUE) {
          g.read = 0;
          g.nops = 0;
          g.value0 = in_type(Q.value[f]);
        } else if (Q.kind[f] == SB_BC_ODD) {
          g.twoc[g.nops++] = twice(Q.value[f]);
        }
      }
      g.es = unsigned(es);
      g.dtype = unsigned(Q.dtype);
      const long long row_bytes = reg.extent[0] * es;
      const unsigned rows = unsigned(reg.extent[1] * reg.extent[2]);
      unsigned rows_per_tile = unsigned(sb::kBcThreads);
      if (reg.mirror[0] < 0) { // row segment: widest access that divides every row start and the row length
        const unsigned long long align =
            (unsigned long long)(uintptr_t)(g.base + reg.pos[0] * es) | (unsigned long long)g.pitch | (unsigned long long)g.slice | (unsigned long long)row_bytes;
        unsigned vec = 16;
        while (vec > 1 && (align & (vec - 1))) vec >>= 1;
        g.vec = vec;
        g.lg_group = std::min(5u, ceil_log2(unsigned(row_bytes / vec)));
        // ~16 KiB of payload, and at least one pass of the whole block (kBcThreads >> lg_group rows)
        rows_per_tile = unsigned(std::max<long long>(sb::kBcThreads >> g.lg_group, sb::kTileBytes / row_bytes));
      }
      const unsigned si = unsigned(segs.size());
      segs.push_back(g);
      for (unsigned r0 = 0; r0 < rows; r0 += rows_per_tile) tiles.push_back(sb::BcTile{si, r0, std::min(rows_per_tile, rows - r0)});
      bytes += row_bytes * reg.extent[1] * reg.extent[2];
    }
  }
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  std::unique_ptr<sb_bc_plan> p(new sb_bc_plan());
  p->device = device;
  p->bytes = bytes;
  p->ntiles = unsigned(tiles.size());
  if (p->ntiles) {
    cudaError_t e = p->segs.upload(device, segs, segs.size());
    if (e == cudaSuccess) e = p->tiles.upload(device, tiles, tiles.size());
    if (e != cudaSuccess) return fail(SB_ERR_CUDA, "BC plan upload: %s", cudaGetErrorString(e));
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    const long long cap = (long long)sms * 8;
    p->grid = int(p->ntiles < cap ? p->ntiles : cap);
  }
  *out = p.release();
  return SB_OK;
}

int sb_bc_plan_launch(sb_bc_plan *p, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (0 == p->ntiles) return SB_OK;
  DeviceGuard guard(p->device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", p->device);
  sb::launch_bc_fill(p->segs.ptr, p->tiles.ptr, p->ntiles, p->grid, static_cast<cudaStream_t>(stream));
  ++g_launches;
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int64_t sb_bc_plan_bytes(const sb_bc_plan *p) { return p ? p->bytes : 0; }

int sb_bc_plan_destroy(sb_bc_plan *p) {
  delete p;
  return SB_OK;
}

int sb_signal(uint32_t *const *remote_slots, int n, uint32_t value, int device, void *stream) {
  if (n <= 0) return SB_OK;
  if (n > 64) return fail(SB_ERR_INVALID, "at most 64 slots per signal");
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SlotTable tab{};
  for (int i = 0; i < n; ++i) tab.p[i] = remote_slots[i];
  signal_kernel<<<1, 64, 0, static_cast<cudaStream_t>(stream)>>>(tab, n, value);
  ++g_launches;
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_wait(const uint32_t *local_slots, int n, uint32_t value, int device, void *stream) {
  if (n <= 0) return SB_OK;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  wait_kernel<<<1, 64, 0, static_cast<cudaStream_t>(stream)>>>(local_slots, n, value);
  ++g_launches;
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- jacobi
static int to_alloc_box(const sb_pitched &a, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3],
                        const int64_t hi[3], int alo[3], int ahi[3]) {
  if (dtype_size != 4 && dtype_size != 8) return fail(SB_ERR_INVALID, "dtype_size must be 4 (float) or 8 (double)");
  if (!a.ptr || a.pitch <= 0 || a.ysize <= 0) return fail(SB_ERR_INVALID, "bad pitched pointer");
  for (int k = 0; k < 3; ++k) {
    const int64_t l = lo[k] - acc_origin[k], h = hi[k] - acc_origin[k];
    if (l < 0 || h > (1ll << 30)) return fail(SB_ERR_INVALID, "region outside the allocation on axis %d", k);
    alo[k] = int(l);
    ahi[k] = int(h);
  }
  return SB_OK;
}

static int jacobi_common(sb::JacobiParams &p, const sb_pitched &dst, const sb_pitched &src, int dtype_size,
                         const int64_t acc_origin[3], const int64_t clo[3], const int64_t chi[3]) {
  if (!dst.ptr || dst.pitch != src.pitch || dst.ysize != src.ysize)
    return fail(SB_ERR_INVALID, "dst and src must have the same pitch and ysize");
  p.dst = static_cast<char *>(dst.ptr);
  p.src = static_cast<const char *>(src.ptr);
  p.pitch = src.pitch;
  p.slice = src.pitch * src.ysize;
  p.raw[0] = int(src.pitch / dtype_size);
  p.raw[1] = int(src.ysize);
  for (int k = 0; k < 3; ++k) p.org[k] = int(acc_origin[k]);
  // sphere placement, bin/jacobi3d.cu:46-51
  const int64_t ex = chi[0] - clo[0];
  p.hot_x = int(clo[0] + ex / 3);
  p.cold_x = int(clo[0] + ex * 2 / 3);
  p.cy = int((clo[1] + chi[1]) / 2);
  p.cz = int((clo[2] + chi[2]) / 2);
  p.rad = int(ex / 10);
  p.zchunk = 0;
  return SB_OK;
}

int sb_jacobi3d_regions(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], int n, const int64_t *lo,
                        const int64_t *hi, const int64_t clo[3], const int64_t chi[3], void *stream) {
  if (n < 0 || n > 8) return fail(SB_ERR_INVALID, "between 0 and 8 regions per launch");
  PtrDeviceGuard guard(dst.ptr);
  sb::JacobiParams p{};
  sb::JacobiRegions r{};
  int zmax = 0;
  r.first[0] = 0;
  int m = 0;
  for (int i = 0; i < n; ++i) {
    int alo[3], ahi[3];
    int rc = to_alloc_box(src, dtype_size, acc_origin, lo + 3 * i, hi + 3 * i, alo, ahi);
    if (rc != SB_OK) return rc;
    long long cells = 1;
    for (int k = 0; k < 3; ++k) {
      if (ahi[k] > alo[k] && alo[k] < 1) return fail(SB_ERR_INVALID, "region needs one ghost cell below it on axis %d", k);
      cells *= (ahi[k] > alo[k]) ? (ahi[k] - alo[k]) : 0;
    }
    if (cells == 0) continue;
    if (cells >= (1ll << 32)) return fail(SB_ERR_INVALID, "region too large for sb_jacobi3d_regions");
    for (int k = 0; k < 3; ++k) {
      r.lo[m][k] = alo[k];
      r.ext[m][k] = ahi[k] - alo[k];
    }
    if (ahi[2] > zmax) zmax = ahi[2];
    r.first[m + 1] = r.first[m] + cells;
    ++m;
  }
  r.n = m;
  if (m == 0) return SB_OK;
  int rc = jacobi_common(p, dst, src, dtype_size, acc_origin, clo, chi);
  if (rc != SB_OK) return rc;
  p.raw[2] = zmax + 1;
  g_launches += uint64_t(sb::launch_jacobi_regions(p, r, dtype_size, static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_jacobi3d(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3],
                const int64_t hi[3], const int64_t clo[3], const int64_t chi[3], void *stream) {
  PtrDeviceGuard guard(dst.ptr);
  sb::JacobiParams p{};
  int rc = to_alloc_box(src, dtype_size, acc_origin, lo, hi, p.lo, p.hi);
  if (rc != SB_OK) return rc;
  for (int k = 0; k < 3; ++k) {
    if (p.lo[k] < 1 && p.hi[k] > p.lo[k]) return fail(SB_ERR_INVALID, "region needs one ghost cell below it on axis %d", k);
  }
  rc = jacobi_common(p, dst, src, dtype_size, acc_origin, clo, chi);
  if (rc != SB_OK) return rc;
  p.dst = static_cast<char *>(dst.ptr);
  p.src = static_cast<const char *>(src.ptr);
  p.pitch = src.pitch;
  p.slice = src.pitch * src.ysize;
  p.raw[0] = int(src.pitch / dtype_size);
  p.raw[1] = int(src.ysize);
  p.raw[2] = p.hi[2] + 1; // planes: the caller guarantees plane hi.z (one ghost plane above) exists
  const int n = sb::launch_jacobi(p, dtype_size, static_cast<cudaStream_t>(stream));
  g_launches += uint64_t(n);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_jacobi3d_fused(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3], const int64_t hi[3],
                      const int64_t clo[3], const int64_t chi[3], const sb_halo_push *push, void *stream) {
  return sb_jacobi3d_fused_sync(dst, src, dtype_size, acc_origin, lo, hi, clo, chi, push, nullptr, stream);
}

int sb_jacobi3d_fused_sync(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3], const int64_t hi[3],
                           const int64_t clo[3], const int64_t chi[3], const sb_halo_push *push, const sb_step_sync *sync, void *stream) {
  if (!push) return fail(SB_ERR_INVALID, "null push table");
  PtrDeviceGuard guard(dst.ptr);
  sb::FusedSync fs{};
  if (sync) {
    for (int f = 0; f < 6; ++f) {
      fs.wait_row[f] = sync->wait_rows[f];
      fs.signal_row[f] = sync->signal_rows[f];
    }
    fs.wait_value = sync->wait_value;
    fs.signal_value = sync->signal_value;
  }
  sb::JacobiParams p{};
  int rc = to_alloc_box(src, dtype_size, acc_origin, lo, hi, p.lo, p.hi);
  if (rc != SB_OK) return rc;
  for (int k = 0; k < 3; ++k) {
    if (p.hi[k] <= p.lo[k]) return SB_OK;
    if (p.lo[k] < 1) return fail(SB_ERR_INVALID, "region needs one ghost cell below it on axis %d", k);
  }
  if (p.hi[0] - p.lo[0] < 16) return fail(SB_ERR_INVALID, "fused step needs at least 16 cells along x");
  rc = jacobi_common(p, dst, src, dtype_size, acc_origin, clo, chi);
  if (rc != SB_OK) return rc;
  p.raw[2] = p.hi[2] + 1;
  for (int d = 0; d < 6; ++d) {
    const sb_pitched &n = push->nbr[d];
    p.push_ptr[d] = nullptr;
    if (!n.ptr) continue;
    const long long npitch = n.pitch, nslice = n.pitch * n.ysize;
    const long long nraw[3] = {npitch / dtype_size, (long long)n.ysize, (long long)push->nbr_zsize[d]};
    const int axis = d / 2;
    if (axis == 0 && push->x_dense[d]) { // dense [y][z] array in the neighbour's memory, my allocation coordinates
      if (n.ysize < p.hi[1] || push->nbr_zsize[d] < p.hi[2]) return fail(SB_ERR_INVALID, "dense x array %d too small", d);
      p.push_ptr[d] = static_cast<char *>(n.ptr);
      p.push_pitch[d] = (long long)push->nbr_zsize[d] * dtype_size;
      p.push_slice[d] = dtype_size;
      p.xdense[d] = 1;
      continue;
    }
    // -axis neighbour: my first cells are its HIGH ghost (index raw-1); +axis neighbour: my last cells are its ghost 0
    const long long fixed = (d % 2 == 0) ? nraw[axis] - 1 : 0;
    if (nraw[axis] < 3) return fail(SB_ERR_INVALID, "neighbour %d allocation too small", d);
    const long long stride[3] = {(long long)dtype_size, npitch, nslice};
    p.push_ptr[d] = static_cast<char *>(n.ptr) + fixed * stride[axis];
    p.push_pitch[d] = npitch;
    p.push_slice[d] = nslice;
    // the two varying coordinates are MY allocation coordinates: they must exist in the neighbour's allocation
    for (int k = 0; k < 3; ++k) {
      if (k != axis && p.hi[k] > nraw[k]) return fail(SB_ERR_INVALID, "neighbour %d is smaller than this subdomain on axis %d", d, k);
    }
  }
  for (int sd = 0; sd < 2; ++sd) {
    p.xghost_ptr[sd] = static_cast<const char *>(push->x_recv[sd]);
    p.xghost_pitch[sd] = (long long)(p.hi[2] + 1) * dtype_size; // [y][z] over this subdomain's planes (raw z = hi.z + 1)
  }
  // A periodic self-neighbour on both sides of an axis needs neither ghost cells nor a push: the kernel reads the
  // opposite face of src in place (x: the edge lane's scalar, y: the row above / below a strip).  With alternating row
  // phases (FP32 rows not a multiple of 16 bytes) the wrapped row must have the parity of the ghost row it replaces.
  auto self = [&](int d) { return push->nbr[d].ptr == dst.ptr && push->nbr[d].pitch == dst.pitch && push->nbr[d].ysize == dst.ysize; };
  if (self(0) && self(1)) p.xwrap = 1; // a request: launch_jacobi_fused keeps the x pushes when the vector layout rules it out
  if (self(2) && self(3) && (src.pitch % 16 == 0 || (p.hi[1] - p.lo[1]) % 2 == 0)) p.ywrap = 1, p.push_ptr[2] = p.push_ptr[3] = nullptr;
  if (self(4) && self(5)) p.zwrap = 1, p.push_ptr[4] = p.push_ptr[5] = nullptr; // planes have one phase: nothing else to check
  const int n = sb::launch_jacobi_fused(p, fs, dtype_size, static_cast<cudaStream_t>(stream));
  if (n == -1) return fail(SB_ERR_INVALID, "a dense received x array needs a 16-byte aligned first compute cell and whole warp strips along x");
  if (n == -2) return fail(SB_ERR_INVALID, "more than %d z chunks or tile rows: too tall for the fused kernel's face groups", SB_FUSED_MAX_GROUPS);
  if (n < 0) return fail(SB_ERR_CUDA, "cannot allocate the face-group counters");
  g_launches += uint64_t(n);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_astaroth_substep(int step, const void *const in[8], void *const out[8], int dtype_size, const int64_t raw[3], const int64_t lo[3],
                        const int64_t hi[3], const sb_astaroth_params *params, int variant, void *stream) {
  if (!in || !out || !raw || !lo || !hi || !params) return fail(SB_ERR_INVALID, "null argument");
  if (step < 0 || step > 2) return fail(SB_ERR_INVALID, "substep %d (Williamson RK3 has substeps 0, 1, 2)", step);
  if (dtype_size != 4 && dtype_size != 8) return fail(SB_ERR_INVALID, "dtype_size %d (4 = float, 8 = double)", dtype_size);
  PtrDeviceGuard guard(out[0]);
  if (variant < 0 || variant > 5) return fail(SB_ERR_INVALID, "variant %d", variant);
  sb::AcFields f;
  for (int i = 0; i < sb::kAcFields; ++i) {
    if (!in[i] || !out[i]) return fail(SB_ERR_INVALID, "field %d is null", i);
    f.in[i] = in[i];
    f.out[i] = out[i];
  }
  int ilo[3], ihi[3];
  for (int k = 0; k < 3; ++k) {
    if (raw[k] <= 0 || raw[k] >= (1ll << 31)) return fail(SB_ERR_INVALID, "raw size");
    if (hi[k] > lo[k] && (lo[k] < 3 || hi[k] > raw[k] - 3))
      return fail(SB_ERR_INVALID, "box [%lld,%lld) on axis %d needs 3 allocated cells on each side (raw %lld)", (long long)lo[k], (long long)hi[k], k,
                  (long long)raw[k]);
    ilo[k] = int(lo[k]);
    ihi[k] = int(hi[k] > lo[k] ? hi[k] : lo[k]);
  }
  sb::AcParams p;
  static_assert(sizeof(sb::AcParams) == sizeof(sb_astaroth_params), "same layout");
  memcpy(&p, params, sizeof(p));
  const int n = sb::launch_astaroth_substep(step, f, dtype_size, raw[0], raw[1], raw[2], ilo, ihi, p, variant, static_cast<cudaStream_t>(stream));
  if (n < 0) return fail(SB_ERR_INVALID, "astaroth substep rejected (code %d)", n);
  g_launches += uint64_t(n);
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_fill(sb_pitched dst, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3], const int64_t hi[3], double value,
            void *stream) {
  PtrDeviceGuard guard(dst.ptr);
  int alo[3], ahi[3];
  int rc = to_alloc_box(dst, dtype_size, acc_origin, lo, hi, alo, ahi);
  if (rc != SB_OK) return rc;
  g_launches += uint64_t(sb::launch_fill(static_cast<char *>(dst.ptr), dst.pitch, dst.pitch * dst.ysize, alo, ahi, dtype_size, value,
                                         static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int sb_sqdiff(sb_pitched a, sb_pitched b, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3], const int64_t hi[3],
              double *out_dev, void *stream) {
  PtrDeviceGuard guard(a.ptr);
  int alo[3], ahi[3];
  int rc = to_alloc_box(a, dtype_size, acc_origin, lo, hi, alo, ahi);
  if (rc != SB_OK) return rc;
  if (b.pitch != a.pitch || b.ysize != a.ysize || !b.ptr || !out_dev) return fail(SB_ERR_INVALID, "mismatched operands");
  g_launches += uint64_t(sb::launch_sqdiff(static_cast<const char *>(a.ptr), static_cast<const char *>(b.ptr), a.pitch,
                                           a.pitch * a.ysize, alo, ahi, dtype_size, out_dev, static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- reductions
namespace {
// Lanes per row (log2) and rows per tile of a reduction or Krylov pass over rows of nx es-byte cells, read 16 bytes at
// a time where wide: functions of the box and the access width only.
struct RowTiles {
  int lg_group;
  long long rows_per_tile;
};
RowTiles row_tiles(long long nx, int es, bool wide) {
  const int lg = int(std::min(5u, ceil_log2(unsigned(std::max(1ll, (nx * es + 15) / 16)))));
  const long long N = wide ? 16 / es : 1, G = 1ll << lg;
  // longest chain of one lane over one row: its body vectors, one head and one tail cell
  const long long per_row = N * (((nx / N) + G - 1) / G) + 2 * ((std::min(nx, N - 1) + G - 1) / G);
  return {lg, std::max(1ll, sb::kRedChain / std::max(1ll, per_row)) * (sb::kRedThreads >> lg)};
}

// The checks, items and tile table of a reduction plan, ordered or exact (`fn` names the entry point in the messages).
struct RedTables {
  std::vector<sb::RedItem> its;
  std::vector<sb::RedTile> tiles;
  unsigned class_tiles[sb::kRedClasses][2];
  int64_t bytes = 0;
};
int reduce_tables(const char *fn, bool out_ok, const sb_reduce_item *items, int64_t n, RedTables &T) {
  if (!out_ok || !items || n < 1) return fail(SB_ERR_INVALID, "%s needs an output handle and n >= 1 items", fn);
  if (n > (1 << 20)) return fail(SB_ERR_INVALID, "at most 2^20 items per plan");
  std::vector<sb::RedItem> &its = T.its;
  std::vector<sb::RedTile> &tiles = T.tiles;
  int64_t &bytes = T.bytes;
  for (int64_t i = 0; i < n; ++i) {
    const sb_reduce_item &I = items[i];
    const long long li = (long long)i;
    if (I.kind < SB_REDUCE_SCALAR || I.kind > SB_REDUCE_NORM3) return fail(SB_ERR_INVALID, "item %lld: unknown kind %d", li, int(I.kind));
    if (I.dtype != SB_DTYPE_F32 && I.dtype != SB_DTYPE_F64)
      return fail(SB_ERR_INVALID, "item %lld: dtype %d must be SB_DTYPE_F32 or SB_DTYPE_F64", li, int(I.dtype));
    const int es = I.dtype == SB_DTYPE_F32 ? 4 : 8;
    const int ns = I.kind == SB_REDUCE_SCALAR ? 1 : I.kind == SB_REDUCE_DIFF ? 2 : 3;
    for (int a = 0; a < 3; ++a)
      if (I.lo[a] > I.hi[a]) return fail(SB_ERR_INVALID, "item %lld: lo > hi on axis %d", li, a);
    int alo[3] = {0, 0, 0}, ahi[3] = {0, 0, 0};
    for (int s = 0; s < ns; ++s) {
      const sb_pitched &P = I.src[s];
      const int rc = to_alloc_box(P, es, I.acc_origin, I.lo, I.hi, alo, ahi);
      if (rc != SB_OK) return fail(SB_ERR_INVALID, "item %lld, source %d: %s", li, s, g_err.c_str());
      if (P.pitch != I.src[0].pitch || P.ysize != I.src[0].ysize)
        return fail(SB_ERR_INVALID, "item %lld: its sources have different pitches or row counts", li);
      if ((uintptr_t(P.ptr) % uintptr_t(es)) || (P.pitch % es))
        return fail(SB_ERR_INVALID, "item %lld, source %d: pointer and pitch must be multiples of the %d-byte element", li, s, es);
    }
    const sb_pitched &P0 = I.src[0];
    if ((long long)ahi[0] * es > P0.pitch || ahi[1] > P0.ysize) return fail(SB_ERR_INVALID, "item %lld: box outside the allocation", li);
    sb::RedItem r{};
    r.pitch = P0.pitch;
    r.slice = P0.pitch * P0.ysize;
    for (int a = 0; a < 3; ++a) r.ext[a] = ahi[a] - alo[a];
    const long long off = (long long)alo[2] * r.slice + (long long)alo[1] * r.pitch + (long long)alo[0] * es;
    bool wide = true;
    for (int s = 0; s < 3; ++s) {
      r.src[s] = static_cast<const char *>(I.src[s < ns ? s : 0].ptr) + off;
      wide = wide && ((uintptr_t(r.src[s]) - uintptr_t(r.src[0])) % 16 == 0);
    }
    r.kind = I.kind;
    r.dtype = I.dtype;
    r.vec = wide ? 16 : es;
    const long long nx = r.ext[0], rows = (long long)r.ext[1] * r.ext[2];
    r.lg_group = row_tiles(nx, es, wide).lg_group;
    r.count = nx * rows;
    if (rows >= (1ll << 31)) return fail(SB_ERR_INVALID, "item %lld: more than 2^31 rows", li);
    its.push_back(r);
    bytes += r.count * es * ns;
  }
  // the tile table, class by class; inside a class item by item
  unsigned(&class_tiles)[sb::kRedClasses][2] = T.class_tiles;
  for (int c = 0; c < sb::kRedClasses; ++c) {
    class_tiles[c][0] = unsigned(tiles.size());
    for (size_t i = 0; i < its.size(); ++i) {
      sb::RedItem &r = its[i];
      if (sb::reduce_class(r) != c) continue;
      r.tile0 = unsigned(tiles.size());
      if (r.count > 0) {
        const long long rows = (long long)r.ext[1] * r.ext[2];
        const long long rows_per_tile = row_tiles(r.ext[0], r.dtype == SB_DTYPE_F32 ? 4 : 8, r.vec == 16).rows_per_tile;
        for (long long r0 = 0; r0 < rows; r0 += rows_per_tile)
          tiles.push_back(sb::RedTile{unsigned(i), unsigned(r0), unsigned(std::min(rows_per_tile, rows - r0))});
        if (tiles.size() >= (1ull << 31)) return fail(SB_ERR_INVALID, "too many tiles");
      }
      r.ntiles = unsigned(tiles.size()) - r.tile0;
    }
    class_tiles[c][1] = unsigned(tiles.size());
  }
  return SB_OK;
}

// An ordered or exact reduction plan over the tables T, its per-class grids from grid (reduce_grid or
// reduce_exact_grid).  The tile table and the scratch hold at least one element.
extern "C++" template <class Plan> int reduce_plan_upload(Plan **out, int device, const RedTables &T, int (*grid)(int, int, unsigned)) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  std::unique_ptr<Plan> p(new Plan());
  p->device = device;
  p->bytes = T.bytes;
  p->nitems = unsigned(T.its.size());
  const size_t ntiles = std::max<size_t>(1, T.tiles.size());
  cudaError_t e = p->items.upload(device, T.its, T.its.size());
  if (e == cudaSuccess) e = p->tiles.upload(device, T.tiles, ntiles);
  if (e == cudaSuccess) e = p->scratch.upload(device, {}, ntiles);
  if (e != cudaSuccess) return fail(SB_ERR_CUDA, "reduction plan upload: %s", cudaGetErrorString(e));
  for (int c = 0; c < sb::kRedClasses; ++c) {
    p->class_tiles[c][0] = T.class_tiles[c][0];
    p->class_tiles[c][1] = T.class_tiles[c][1];
    p->grids[c] = grid(device, c, T.class_tiles[c][1] - T.class_tiles[c][0]);
  }
  *out = p.release();
  return SB_OK;
}
} // namespace

int sb_reduce_plan_create(sb_reduce_plan **out, int device, const sb_reduce_item *items, int64_t n) {
  RedTables T;
  const int rc = reduce_tables("sb_reduce_plan_create", out != nullptr, items, n, T);
  if (rc != SB_OK) return rc;
  return reduce_plan_upload(out, device, T, sb::reduce_grid);
}

int sb_reduce_plan_launch(sb_reduce_plan *p, sb_reduce_result *out_dev, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (!out_dev) return fail(SB_ERR_INVALID, "null output buffer");
  DeviceGuard guard(p->device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", p->device);
  g_launches += uint64_t(sb::launch_reduce(p->items.ptr, p->nitems, p->tiles.ptr, p->class_tiles, p->grids, p->scratch.ptr, out_dev,
                                           static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int64_t sb_reduce_plan_bytes(const sb_reduce_plan *p) { return p ? p->bytes : 0; }

int sb_reduce_plan_destroy(sb_reduce_plan *p) {
  delete p;
  return SB_OK;
}

int sb_reduce_combine(const sb_reduce_result *parts, int64_t n, sb_reduce_result *out) {
  if (!parts || !out || n < 1) return fail(SB_ERR_INVALID, "sb_reduce_combine needs n >= 1 results and an output");
  std::vector<sb_reduce_result> a(parts, parts + n);
  for (int64_t s = 1; s < n; s *= 2)
    for (int64_t i = 0; i + s < n; i += 2 * s) a[size_t(i)] = sb::red_merge(a[size_t(i)], a[size_t(i + s)]);
  *out = a[0];
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- exact reductions
int sb_reduce_exact_plan_create(sb_reduce_exact_plan **out, int device, const sb_reduce_item *items, int64_t n) {
  RedTables T;
  const int rc = reduce_tables("sb_reduce_exact_plan_create", out != nullptr, items, n, T);
  if (rc != SB_OK) return rc;
  // a tile then holds at most 2^30 cells, and the kernel's per-tile digit counters cannot overflow (reduce.cuh)
  for (size_t i = 0; i < T.its.size(); ++i)
    if (T.its[i].ext[0] > (1 << 27)) return fail(SB_ERR_INVALID, "item %lld: rows of more than 2^27 cells", (long long)i);
  return reduce_plan_upload(out, device, T, sb::reduce_exact_grid);
}

int sb_reduce_exact_plan_launch(sb_reduce_exact_plan *p, sb_reduce_exact_part *out_dev, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (!out_dev) return fail(SB_ERR_INVALID, "null output buffer");
  DeviceGuard guard(p->device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", p->device);
  g_launches += uint64_t(sb::launch_reduce_exact(p->items.ptr, p->nitems, p->tiles.ptr, p->class_tiles, p->grids, p->scratch.ptr, out_dev,
                                                 static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int64_t sb_reduce_exact_plan_bytes(const sb_reduce_exact_plan *p) { return p ? p->bytes : 0; }

int sb_reduce_exact_plan_destroy(sb_reduce_exact_plan *p) {
  delete p;
  return SB_OK;
}

namespace {
uint64_t bits_of(double x) {
  uint64_t b;
  std::memcpy(&b, &x, sizeof b);
  return b;
}
// min / max whose result does not depend on the operand order: a NaN wins (of two, the larger bit pattern); of +0 and
// -0 min takes -0, max +0
double exact_min(double a, double b) {
  if (a != a || b != b) return (a != a && b != b) ? (bits_of(a) > bits_of(b) ? a : b) : (a != a ? a : b);
  if (a != b) return a < b ? a : b;
  return std::signbit(a) ? a : b;
}
double exact_max(double a, double b) {
  if (a != a || b != b) return (a != a && b != b) ? (bits_of(a) > bits_of(b) ? a : b) : (a != a ? a : b);
  if (a != b) return a > b ? a : b;
  return std::signbit(a) ? b : a;
}
void exact_add(sb_exact_sum &a, const sb_exact_sum &b) {
  unsigned carry = 0;
  for (int k = 0; k < SB_EXACT_WORDS; ++k) {
    const uint64_t s = a.word[k] + b.word[k];
    const unsigned c1 = s < a.word[k];
    a.word[k] = s + carry;
    carry = c1 | (a.word[k] < s);
  }
  a.flags |= b.flags;
}
// the exact sum rounded to nearest, ties to even, with the special-value rule of include/stencil_b200.h
double exact_round(const sb_exact_sum &e) {
  if ((e.flags & SB_EXACT_NAN) || ((e.flags & SB_EXACT_POS_INF) && (e.flags & SB_EXACT_NEG_INF))) return std::nan("");
  if (e.flags & SB_EXACT_POS_INF) return HUGE_VAL;
  if (e.flags & SB_EXACT_NEG_INF) return -HUGE_VAL;
  uint64_t m[SB_EXACT_WORDS];
  const bool neg = e.word[SB_EXACT_WORDS - 1] >> 63;
  unsigned carry = 1;
  for (int k = 0; k < SB_EXACT_WORDS; ++k) { // magnitude: two's complement negation for a negative sum
    m[k] = neg ? ~e.word[k] + carry : e.word[k];
    if (neg) carry = carry && m[k] == 0;
  }
  int top = -1; // highest set bit, in units of 2^-1074
  for (int k = SB_EXACT_WORDS - 1; k >= 0 && top < 0; --k)
    if (m[k]) top = 64 * k + 63 - __builtin_clzll(m[k]);
  if (top < 0) return 0.0;
  auto bit = [&](int i) { return i >= 0 ? int((m[i / 64] >> (i % 64)) & 1u) : 0; };
  double r;
  if (top < 53) {
    r = std::ldexp(double(m[0]), -1074); // below 2^53 units: exact (subnormal or the smallest normal binade)
  } else {
    const int lsb = top - 52; // the 53 kept bits are [lsb, top]
    uint64_t mant = 0;
    for (int i = top; i >= lsb; --i) mant = (mant << 1) | uint64_t(bit(i));
    bool sticky = false;
    for (int i = 0; i < lsb - 1 && !sticky; ++i) sticky = bit(i);
    if (bit(lsb - 1) && (sticky || (mant & 1u))) ++mant; // 2^53 stays exact: ldexp scales it
    r = std::ldexp(double(mant), lsb - 1074);            // beyond the double range: inf
  }
  return neg ? -r : r;
}
} // namespace

int sb_reduce_exact_combine(const sb_reduce_exact_part *parts, int64_t n, sb_reduce_exact_part *out) {
  if (!parts || !out || n < 1) return fail(SB_ERR_INVALID, "sb_reduce_exact_combine needs n >= 1 parts and an output");
  sb_reduce_exact_part r = parts[0];
  for (int64_t i = 1; i < n; ++i) {
    const sb_reduce_exact_part &b = parts[i];
    r.min = exact_min(r.min, b.min);
    r.max = exact_max(r.max, b.max);
    r.count += b.count;
    exact_add(r.sum, b.sum);
    exact_add(r.sumsq, b.sumsq);
  }
  *out = r;
  return SB_OK;
}

int sb_reduce_exact_round(const sb_reduce_exact_part *part, sb_reduce_result *out) {
  if (!part || !out) return fail(SB_ERR_INVALID, "sb_reduce_exact_round needs a part and an output");
  *out = sb_reduce_result{part->min, part->max, exact_round(part->sum), exact_round(part->sumsq), part->count};
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- krylov vector kernels
int sb_krylov_plan_create(sb_krylov_plan **out, int device, int mode, int dtype, const sb_pitched *bufs, int nbuf, const int64_t acc_origin[3],
                          const int64_t lo[3], const int64_t hi[3]) {
  if (!out || !acc_origin || !lo || !hi) return fail(SB_ERR_INVALID, "sb_krylov_plan_create needs an output handle, acc_origin, lo and hi");
  if (mode < SB_KRYLOV_DOT || mode > SB_KRYLOV_BICG_P || mode == 3) return fail(SB_ERR_INVALID, "unknown krylov mode %d", mode);
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) return fail(SB_ERR_INVALID, "dtype %d must be SB_DTYPE_F32 or SB_DTYPE_F64", dtype);
  static const char *const names[5][5] = {{"a", "b", "c", "", ""}, {"p", "z", "", "", ""}, {"x", "p", "r", "q", "c"}, {}, {"p", "r", "v", "", ""}};
  static const char *const mode_name[5] = {"SB_KRYLOV_DOT", "SB_KRYLOV_XPBY", "SB_KRYLOV_UPDATE", "", "SB_KRYLOV_BICG_P"};
  const bool count_ok = mode == SB_KRYLOV_DOT      ? (nbuf == 2 || nbuf == 3)
                        : mode == SB_KRYLOV_XPBY   ? nbuf == 2
                        : mode == SB_KRYLOV_BICG_P ? nbuf == 3
                                                   : (nbuf == 4 || nbuf == 5);
  if (!bufs || !count_ok)
    return fail(SB_ERR_INVALID, "%s takes %s buffers, not %d%s", mode_name[mode],
                mode == SB_KRYLOV_DOT ? "2 or 3" : mode == SB_KRYLOV_XPBY ? "2" : mode == SB_KRYLOV_BICG_P ? "3" : "4", nbuf,
                mode == SB_KRYLOV_UPDATE ? " (5 with c)" : "");
  const int es = dtype == SB_DTYPE_F32 ? 4 : 8;
  for (int a = 0; a < 3; ++a)
    if (lo[a] > hi[a]) return fail(SB_ERR_INVALID, "lo > hi on axis %d", a);
  int alo[3] = {0, 0, 0}, ahi[3] = {0, 0, 0};
  for (int k = 0; k < nbuf; ++k) {
    const sb_pitched &P = bufs[k];
    if (!P.ptr) return fail(SB_ERR_INVALID, "buffer %s is NULL", names[mode][k]);
    const int rc = to_alloc_box(P, es, acc_origin, lo, hi, alo, ahi);
    if (rc != SB_OK) return fail(SB_ERR_INVALID, "buffer %s: %s", names[mode][k], g_err.c_str());
    if (P.pitch != bufs[0].pitch || P.ysize != bufs[0].ysize) return fail(SB_ERR_INVALID, "the buffers have different pitches or row counts");
    if ((uintptr_t(P.ptr) % uintptr_t(es)) || (P.pitch % es))
      return fail(SB_ERR_INVALID, "buffer %s: pointer and pitch must be multiples of the %d-byte element", names[mode][k], es);
  }
  if ((long long)ahi[0] * es > bufs[0].pitch || ahi[1] > bufs[0].ysize) return fail(SB_ERR_INVALID, "box outside the allocation");
  if (ahi[0] - alo[0] > (1 << 27)) return fail(SB_ERR_INVALID, "rows of more than 2^27 cells");
  if ((long long)(ahi[1] - alo[1]) * (ahi[2] - alo[2]) >= (1ll << 31)) return fail(SB_ERR_INVALID, "more than 2^31 rows");
  if (mode == SB_KRYLOV_XPBY && bufs[0].ptr == bufs[1].ptr) return fail(SB_ERR_INVALID, "SB_KRYLOV_XPBY: p must not be z");
  if (mode == SB_KRYLOV_UPDATE)
    for (int i = 0; i < 4; ++i)
      for (int j = i + 1; j < 4; ++j)
        if (bufs[i].ptr == bufs[j].ptr) return fail(SB_ERR_INVALID, "SB_KRYLOV_UPDATE: x, p, r and q must be four distinct buffers (%s is %s)", names[2][j], names[2][i]);
  if (mode == SB_KRYLOV_UPDATE && nbuf == 5 && (bufs[4].ptr == bufs[0].ptr || bufs[4].ptr == bufs[2].ptr))
    return fail(SB_ERR_INVALID, "SB_KRYLOV_UPDATE: c must not be x or r (c is %s)", bufs[4].ptr == bufs[0].ptr ? "x" : "r");
  if (mode == SB_KRYLOV_BICG_P && (bufs[0].ptr == bufs[1].ptr || bufs[0].ptr == bufs[2].ptr))
    return fail(SB_ERR_INVALID, "SB_KRYLOV_BICG_P: p must not be r or v (%s is p)", bufs[0].ptr == bufs[1].ptr ? "r" : "v");
  // a written buffer must not overlap another buffer of the pass: the bytes from the box's first cell to its last.  Of
  // two read-only buffers, only UPDATE's p and q are checked (UPDATE's c and BICG_P's r and v may alias).
  const unsigned written = mode == SB_KRYLOV_UPDATE ? 5u : 1u;
  if (mode != SB_KRYLOV_DOT && ahi[0] > alo[0] && ahi[1] > alo[1] && ahi[2] > alo[2]) {
    const long long slice = bufs[0].pitch * bufs[0].ysize;
    const long long first = (long long)alo[2] * slice + (long long)alo[1] * bufs[0].pitch + (long long)alo[0] * es;
    const long long last = (long long)(ahi[2] - 1) * slice + (long long)(ahi[1] - 1) * bufs[0].pitch + (long long)ahi[0] * es;
    for (int i = 0; i < nbuf; ++i)
      for (int j = i + 1; j < nbuf; ++j) {
        const bool read_only = !((written >> i) & 1u) && !((written >> j) & 1u);
        if (read_only && (mode == SB_KRYLOV_BICG_P || j == 4)) continue;
        const uintptr_t a = uintptr_t(bufs[i].ptr), b = uintptr_t(bufs[j].ptr);
        if (a + uintptr_t(first) < b + uintptr_t(last) && b + uintptr_t(first) < a + uintptr_t(last))
          return fail(SB_ERR_INVALID, "%s: buffers %s and %s overlap over the box", mode_name[mode], names[mode][i], names[mode][j]);
      }
  }
  sb::KryParams kp{};
  kp.pitch = bufs[0].pitch;
  kp.slice = bufs[0].pitch * bufs[0].ysize;
  for (int a = 0; a < 3; ++a) kp.ext[a] = ahi[a] - alo[a];
  const long long off = (long long)alo[2] * kp.slice + (long long)alo[1] * kp.pitch + (long long)alo[0] * es;
  bool wide = true;
  for (int k = 0; k < 5; ++k) {
    kp.buf[k] = static_cast<char *>(bufs[k < nbuf ? k : 0].ptr) + off;
    wide = wide && ((uintptr_t(kp.buf[k]) - uintptr_t(kp.buf[0])) % 16 == 0);
  }
  const long long nx = kp.ext[0], rows = (long long)kp.ext[1] * kp.ext[2];
  const RowTiles rt = row_tiles(nx, es, wide);
  kp.lg_group = rt.lg_group;
  kp.count = nx * rows;
  kp.rows_per_tile = unsigned(rt.rows_per_tile);
  kp.ntiles = kp.count > 0 ? unsigned((rows + rt.rows_per_tile - 1) / rt.rows_per_tile) : 0u;
  int kmode = nbuf == 5 ? sb::kKryUpdateC : sb::kKryUpdate;
  if (mode == SB_KRYLOV_DOT) kmode = nbuf == 3 ? sb::kKryDot2 : sb::kKryDot1;
  if (mode == SB_KRYLOV_XPBY) kmode = sb::kKryXpby;
  if (mode == SB_KRYLOV_BICG_P) kmode = sb::kKryBicgP;
  // per cell: one element per distinct buffer read, one per buffer written
  int nread = 0;
  for (int k = 0; k < nbuf; ++k) {
    bool dup = false;
    for (int j = 0; j < k; ++j) dup = dup || bufs[j].ptr == bufs[k].ptr;
    nread += !dup;
  }
  const int nwrite = mode == SB_KRYLOV_XPBY || mode == SB_KRYLOV_BICG_P ? 1 : mode == SB_KRYLOV_UPDATE ? 2 : 0;
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  std::unique_ptr<sb_krylov_plan> p(new sb_krylov_plan());
  p->device = device;
  p->dtype = dtype;
  p->mode = kmode;
  p->wide = wide;
  p->params = kp;
  p->bytes = kp.count * es * (nread + nwrite);
  if (sb::kry_dots(kmode) > 0) {
    const cudaError_t e = p->scratch.upload(device, {}, std::max<size_t>(1, kp.ntiles));
    if (e != cudaSuccess) return fail(SB_ERR_CUDA, "krylov plan scratch: %s", cudaGetErrorString(e));
  }
  p->grid = sb::krylov_grid(device, dtype, kmode, wide, kp.ntiles);
  p->copy_grid = mode == SB_KRYLOV_XPBY ? sb::krylov_grid(device, dtype, sb::kKryCopy, wide, kp.ntiles) : 0;
  *out = p.release();
  return SB_OK;
}

int sb_krylov_plan_launch(sb_krylov_plan *p, double s, sb_reduce_exact_part *parts_dev, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (p->mode == sb::kKryBicgP) return fail(SB_ERR_INVALID, "sb_krylov_plan_launch: SB_KRYLOV_BICG_P takes two scalars; use sb_krylov_plan_launch2");
  return sb_krylov_plan_launch2(p, s, 0.0, parts_dev, stream);
}

int sb_krylov_plan_launch2(sb_krylov_plan *p, double s, double t, sb_reduce_exact_part *parts_dev, void *stream) {
  if (!p) return fail(SB_ERR_INVALID, "null plan");
  if (!parts_dev && sb::kry_dots(p->mode) > 0) return fail(SB_ERR_INVALID, "null output buffer");
  DeviceGuard guard(p->device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", p->device);
  int mode = p->mode, grid = p->grid;
  // T(s) = +-0: p = z, never reading p (a NaN in p stays out)
  if (mode == sb::kKryXpby && (p->dtype == SB_DTYPE_F32 ? float(s) == 0.0f : s == 0.0)) {
    mode = sb::kKryCopy;
    grid = p->copy_grid;
  }
  g_launches += uint64_t(sb::launch_krylov(p->params, p->dtype, mode, p->wide, grid, s, t, p->scratch.ptr, parts_dev, static_cast<cudaStream_t>(stream)));
  SB_CUDA(cudaGetLastError());
  return SB_OK;
}

int64_t sb_krylov_plan_bytes(const sb_krylov_plan *p) { return p ? p->bytes : 0; }

int sb_krylov_plan_destroy(sb_krylov_plan *p) {
  delete p;
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- linear stencil operators
// The limits every term list obeys, whatever the domain: n, sources, |o_a| <= 4, aux terms without offset, coefficient
// fields 0 .. 3 (or -1) read within reach 1, plain terms without a coefficient offset.
// |o_a| <= 4 for the source offset of term t (operators and systems alike)
static int stencil_offset_ok(int t, const int32_t o[3]) {
  for (int a = 0; a < 3; ++a)
    if (o[a] < -SB_STENCIL_MAX_REACH || o[a] > SB_STENCIL_MAX_REACH)
      return fail(SB_ERR_INVALID, "term %d: offset (%d, %d, %d) reaches beyond %d cells", t, int(o[0]), int(o[1]), int(o[2]),
                  SB_STENCIL_MAX_REACH);
  return SB_OK;
}

// The coefficient of term t (operators and systems alike): -1 or 0 .. ncoef - 1 (what: "field" or "input"), read within
// reach 1, and no coefficient offset without a coefficient.
static int stencil_coef_ok(int t, int32_t coef, const int32_t c[3], int ncoef, const char *what) {
  if (coef < -1 || coef >= ncoef) return fail(SB_ERR_INVALID, "term %d: coefficient %s %d must be -1 (none) or 0 .. %d", t, what, int(coef), ncoef - 1);
  if (coef == -1 && (c[0] || c[1] || c[2]))
    return fail(SB_ERR_INVALID, "term %d: a term without a coefficient field has coefficient offset (0, 0, 0), not (%d, %d, %d)", t,
                int(c[0]), int(c[1]), int(c[2]));
  for (int a = 0; a < 3; ++a)
    if (c[a] < -SB_STENCIL_COEF_REACH || c[a] > SB_STENCIL_COEF_REACH)
      return fail(SB_ERR_INVALID, "term %d: coefficient offset (%d, %d, %d) reaches beyond %d cell", t, int(c[0]), int(c[1]), int(c[2]),
                  SB_STENCIL_COEF_REACH);
  return SB_OK;
}

static int stencil_terms_ok(const sb_stencil_vterm *terms, int n) {
  if (!terms || n < 1 || n > SB_STENCIL_MAX_TERMS) return fail(SB_ERR_INVALID, "an op has 1 to %d terms, not %d", SB_STENCIL_MAX_TERMS, terms ? n : 0);
  for (int t = 0; t < n; ++t) {
    const sb_stencil_vterm &T = terms[t];
    if (T.source != 0 && T.source != 1) return fail(SB_ERR_INVALID, "term %d: source %d must be 0 (src) or 1 (aux)", t, int(T.source));
    int rc = stencil_offset_ok(t, T.offset);
    if (rc != SB_OK) return rc;
    if (T.source == 1 && (T.offset[0] || T.offset[1] || T.offset[2]))
      return fail(SB_ERR_INVALID, "term %d: an aux term has offset (0, 0, 0), not (%d, %d, %d)", t, int(T.offset[0]), int(T.offset[1]),
                  int(T.offset[2]));
    if ((rc = stencil_coef_ok(t, T.coef, T.coef_offset, SB_STENCIL_MAX_COEFS, "field")) != SB_OK) return rc;
  }
  return SB_OK;
}

// Whether box b (allocation-relative lo l, extent e), read rm cells below and rp above on each axis, stays inside an
// allocation of size[3], with the window's end below 2^31: the kernels take these coordinates as int.  who: what reads
// ("the op reads", "input 2 is read at", ...).
static int stencil_box_reads_ok(int b, const int64_t l[3], const int64_t e[3], const int rm[3], const int rp[3], const int64_t size[3],
                                const std::string &who) {
  for (int a = 0; a < 3; ++a) {
    if (l[a] - rm[a] < 0 || l[a] + e[a] + rp[a] > size[a])
      return fail(SB_ERR_INVALID, "box %d: %s cells %lld .. %lld on axis %c, outside the allocation's 0 .. %lld", b, who.c_str(),
                  (long long)(l[a] - rm[a]), (long long)(l[a] + e[a] + rp[a] - 1), "xyz"[a], (long long)(size[a] - 1));
    if (l[a] + e[a] + rp[a] >= (1ll << 31))
      return fail(SB_ERR_INVALID, "box %d: %s cells %lld .. %lld on axis %c, beyond the kernels' 32-bit coordinates (at most 2^31 - 2)", b,
                  who.c_str(), (long long)(l[a] - rm[a]), (long long)(l[a] + e[a] + rp[a] - 1), "xyz"[a]);
  }
  return SB_OK;
}

// Whether a subdomain with ghost widths radius27 holds the cell at offset o of term t (what: "offset" or "coefficient
// offset"): the ghost box of sign(o) is exchanged and each non-zero component fits the face radius on its side.
static int stencil_offset_in_reach(int t, const char *what, const int32_t o[3], const int64_t radius27[27]) {
  if (!o[0] && !o[1] && !o[2]) return SB_OK;
  int s[3];
  for (int a = 0; a < 3; ++a) s[a] = (o[a] > 0) - (o[a] < 0);
  if (radius27[(s[2] + 1) * 9 + (s[1] + 1) * 3 + (s[0] + 1)] <= 0)
    return fail(SB_ERR_INVALID, "term %d: %s (%d, %d, %d) reads the ghost box in direction (%d, %d, %d), whose radius is 0", t, what,
                int(o[0]), int(o[1]), int(o[2]), s[0], s[1], s[2]);
  for (int a = 0; a < 3; ++a) {
    if (!o[a]) continue;
    int d[3] = {0, 0, 0};
    d[a] = s[a];
    const int64_t face = radius27[(d[2] + 1) * 9 + (d[1] + 1) * 3 + (d[0] + 1)];
    if (int64_t(o[a] < 0 ? -o[a] : o[a]) > face)
      return fail(SB_ERR_INVALID, "term %d: %s (%d, %d, %d) reaches %d cells on side %c%c, whose face radius is %lld", t, what,
                  int(o[0]), int(o[1]), int(o[2]), int(o[a] < 0 ? -o[a] : o[a]), s[a] < 0 ? '-' : '+', "xyz"[a], (long long)face);
  }
  return SB_OK;
}

// Every buffer shares ref's pitch and row count (ref_name: what ref is called), and its pointer and pitch are positive
// multiples of the es-byte element.
static int stencil_buffers_ok(const std::vector<const sb_pitched *> &bufs, const std::vector<std::string> &names, const sb_pitched &ref,
                              const char *ref_name, int es) {
  for (size_t b = 0; b < bufs.size(); ++b) {
    const sb_pitched &P = *bufs[b];
    if (P.pitch != ref.pitch || P.ysize != ref.ysize)
      return fail(SB_ERR_INVALID, "%s has another pitch or row count than %s", names[b].c_str(), ref_name);
    if ((uintptr_t(P.ptr) % uintptr_t(es)) || P.pitch <= 0 || (P.pitch % es) || P.ysize <= 0)
      return fail(SB_ERR_INVALID, "%s: pointer and pitch must be positive multiples of the %d-byte element", names[b].c_str(), es);
  }
  return SB_OK;
}

// A plain term list as coefficient terms without a field (at most SB_STENCIL_MAX_TERMS are converted: a longer list is
// rejected by stencil_terms_ok on its count; the result holds at least one element so that its data() is not NULL).
static std::vector<sb_stencil_vterm> stencil_vterms_of(const sb_stencil_term *terms, int n) {
  std::vector<sb_stencil_vterm> v(size_t(std::max(1, std::min(n, SB_STENCIL_MAX_TERMS))), sb_stencil_vterm{0, {0, 0, 0}, -1, {0, 0, 0}, 0.0});
  for (int t = 0; terms && t < std::min(n, SB_STENCIL_MAX_TERMS); ++t) {
    sb_stencil_vterm &V = v[size_t(t)];
    V.source = terms[t].source;
    for (int a = 0; a < 3; ++a) V.offset[a] = terms[t].offset[a];
    V.weight = terms[t].weight;
  }
  return v;
}

int sb_stencil_vcheck(const sb_stencil_vterm *terms, int n, const int64_t radius27[27]) {
  if (!radius27) return fail(SB_ERR_INVALID, "sb_stencil_check needs radius27");
  int rc = stencil_terms_ok(terms, n);
  if (rc != SB_OK) return rc;
  for (int t = 0; t < n; ++t) {
    if ((rc = stencil_offset_in_reach(t, "offset", terms[t].offset, radius27)) != SB_OK) return rc;
    if (terms[t].coef >= 0 && (rc = stencil_offset_in_reach(t, "coefficient offset", terms[t].coef_offset, radius27)) != SB_OK) return rc;
  }
  return SB_OK;
}

int sb_stencil_check(const sb_stencil_term *terms, int n, const int64_t radius27[27]) {
  const std::vector<sb_stencil_vterm> v = stencil_vterms_of(terms, n);
  return sb_stencil_vcheck(terms ? v.data() : nullptr, n, radius27);
}

// The colouring m (1, 2 or 8) and the colour condition on every src term with o != 0 (DESIGN.md section 2.9): under
// m = 2 the cell at p + o has another colour than p's iff o_x + o_y + o_z is odd, under m = 8 iff some o_a is odd.
static int stencil_colours_ok(const sb_stencil_vterm *terms, int n, int m) {
  if (m != 1 && m != 2 && m != 8) return fail(SB_ERR_INVALID, "ncolours %d: a colouring has 1, 2 or 8 colours", m);
  for (int t = 0; t < n && m > 1; ++t) {
    const int32_t *o = terms[t].offset;
    if (terms[t].source != 0 || (!o[0] && !o[1] && !o[2])) continue;
    const bool other = m == 2 ? ((o[0] + o[1] + o[2]) & 1) != 0 : ((o[0] | o[1] | o[2]) & 1) != 0;
    if (!other)
      return fail(SB_ERR_INVALID, "term %d: offset (%d, %d, %d) reads a cell of its own colour under %d colours", t, int(o[0]), int(o[1]),
                  int(o[2]), m);
  }
  return SB_OK;
}

// The cells of colour c under the colouring m in the box [lo, lo + e) (global coordinates).
static int64_t stencil_colour_cells(const int64_t lo[3], const int64_t e[3], int m, int c) {
  if (m == 1) return e[0] * e[1] * e[2];
  int64_t n[3][2]; // n[a][q]: the coordinates of the box on axis a of parity q
  for (int a = 0; a < 3; ++a) {
    const int q0 = int(((lo[a] % 2) + 2) % 2);
    n[a][q0] = (e[a] + 1) / 2;
    n[a][q0 ^ 1] = e[a] / 2;
  }
  if (m == 8) return n[0][c & 1] * n[1][(c >> 1) & 1] * n[2][(c >> 2) & 1];
  int64_t total = 0;
  for (int qx = 0; qx < 2; ++qx)
    for (int qy = 0; qy < 2; ++qy) total += n[0][qx] * n[1][qy] * n[2][(c - qx - qy) & 1];
  return total;
}

int sb_stencil_ccheck(const sb_stencil_vterm *terms, int n, const int64_t radius27[27], int ncolours) {
  int rc = sb_stencil_vcheck(terms, n, radius27);
  if (rc != SB_OK) return rc;
  return stencil_colours_ok(terms, n, ncolours);
}

int sb_stencil_relax(const sb_stencil_term *A, int n, double omega, sb_stencil_term *out, int cap) {
  const std::vector<sb_stencil_vterm> v = stencil_vterms_of(A, n);
  int rc = stencil_terms_ok(A ? v.data() : nullptr, n);
  if (rc != SB_OK) return rc;
  if (!std::isfinite(omega)) return fail(SB_ERR_INVALID, "sb_stencil_relax: omega = %g must be finite", omega);
  if (cap < 0 || (cap > 0 && !out)) return fail(SB_ERR_INVALID, "sb_stencil_relax: bad output buffer");
  int centre = -1;
  for (int t = 0; t < n; ++t) {
    const sb_stencil_term &T = A[t];
    if (T.source == 1) return fail(SB_ERR_INVALID, "sb_stencil_relax: term %d reads aux; A reads src only (f goes on aux)", t);
    if (T.offset[0] || T.offset[1] || T.offset[2]) continue;
    if (centre >= 0) return fail(SB_ERR_INVALID, "sb_stencil_relax: terms %d and %d are both at offset (0, 0, 0); A needs one centre term", centre, t);
    centre = t;
  }
  if (centre < 0) return fail(SB_ERR_INVALID, "sb_stencil_relax: A has no term at offset (0, 0, 0)");
  const double ac = A[centre].weight;
  if (ac == 0.0) return fail(SB_ERR_INVALID, "sb_stencil_relax: the centre weight of A is 0");
  if (n + 1 > SB_STENCIL_MAX_TERMS)
    return fail(SB_ERR_INVALID, "sb_stencil_relax: A has %d terms, so the update would have %d (at most %d)", n, n + 1, SB_STENCIL_MAX_TERMS);
  std::vector<sb_stencil_term> r;
  r.push_back(sb_stencil_term{0, {0, 0, 0}, 1.0 - omega});
  for (int t = 0; t < n; ++t)
    if (t != centre) {
      const double num = -omega * A[t].weight;
      r.push_back(sb_stencil_term{0, {A[t].offset[0], A[t].offset[1], A[t].offset[2]}, num / ac});
    }
  r.push_back(sb_stencil_term{1, {0, 0, 0}, omega / ac});
  for (int i = 0; i < int(r.size()) && i < cap; ++i) out[i] = r[size_t(i)];
  return int(r.size());
}

int sb_stencil_div_grad(const double spacing[3], sb_stencil_vterm *out, int cap) {
  if (!spacing) return fail(SB_ERR_INVALID, "sb_stencil_div_grad needs spacing[3]");
  for (int a = 0; a < 3; ++a)
    if (!(spacing[a] > 0.0) || !std::isfinite(spacing[a])) return fail(SB_ERR_INVALID, "spacing[%d] = %g must be finite and > 0", a, spacing[a]);
  if (cap < 0 || (cap > 0 && !out)) return fail(SB_ERR_INVALID, "sb_stencil_div_grad: bad output buffer");
  const int total = 12;
  for (int a = 0, i = 0; a < 3; ++a) {
    const double h2 = spacing[a] * spacing[a];
    const double inv = 1.0 / h2;
    // (src offset, weight, coefficient offset) along axis a, in units of e_a
    const int rows[4][3] = {{1, 1, 1}, {0, -1, 1}, {0, -1, 0}, {-1, 1, 0}};
    for (const auto &r : rows) {
      sb_stencil_vterm t{0, {0, 0, 0}, a, {0, 0, 0}, r[1] * inv};
      t.offset[a] = r[0];
      t.coef_offset[a] = r[2];
      if (i < cap) out[i] = t;
      ++i;
    }
  }
  return total;
}

int sb_stencil_laplacian(int order, const double spacing[3], sb_stencil_term *out, int cap) {
  // c_0 .. c_R of the central second difference, as exact quotients rounded once to double
  static const double c2[] = {-2.0, 1.0};
  static const double c4[] = {-5.0 / 2.0, 4.0 / 3.0, -1.0 / 12.0};
  static const double c6[] = {-49.0 / 18.0, 3.0 / 2.0, -3.0 / 20.0, 1.0 / 90.0};
  static const double c8[] = {-205.0 / 72.0, 8.0 / 5.0, -1.0 / 5.0, 8.0 / 315.0, -1.0 / 560.0};
  const double *c = order == 2 ? c2 : order == 4 ? c4 : order == 6 ? c6 : order == 8 ? c8 : nullptr;
  if (!c) return fail(SB_ERR_INVALID, "Laplacian order %d: 2, 4, 6 or 8", order);
  if (!spacing) return fail(SB_ERR_INVALID, "sb_stencil_laplacian needs spacing[3]");
  for (int a = 0; a < 3; ++a)
    if (!(spacing[a] > 0.0) || !std::isfinite(spacing[a])) return fail(SB_ERR_INVALID, "spacing[%d] = %g must be finite and > 0", a, spacing[a]);
  if (cap < 0 || (cap > 0 && !out)) return fail(SB_ERR_INVALID, "sb_stencil_laplacian: bad output buffer");
  const int R = order / 2, total = 1 + 6 * R;
  double inv[3];
  for (int a = 0; a < 3; ++a) {
    const double h2 = spacing[a] * spacing[a];
    inv[a] = 1.0 / h2;
  }
  std::vector<sb_stencil_term> terms;
  const double cx = c[0] * inv[0], cy = c[0] * inv[1], cz = c[0] * inv[2];
  const double cxy = cx + cy;
  terms.push_back(sb_stencil_term{0, {0, 0, 0}, cxy + cz});
  for (int k = 1; k <= R; ++k)
    for (int a = 0; a < 3; ++a)
      for (int side = -1; side <= 1; side += 2) {
        sb_stencil_term t{0, {0, 0, 0}, c[k] * inv[a]};
        t.offset[a] = side * k;
        terms.push_back(t);
      }
  for (int i = 0; i < total && i < cap; ++i) out[i] = terms[size_t(i)];
  return total;
}

static int stencil_plan_build(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                              sb_pitched src, sb_pitched aux, const sb_pitched *coef, int ncoef, int ncolours, int colour,
                              const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi,
                              const double *omega);

int sb_stencil_plan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_term *terms, int n, sb_pitched dst,
                           sb_pitched src, sb_pitched aux, const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo,
                           const int64_t *hi) {
  if (!out) return fail(SB_ERR_INVALID, "sb_stencil_plan_create needs an output handle");
  const std::vector<sb_stencil_vterm> v = stencil_vterms_of(terms, n);
  return sb_stencil_vplan_create(out, device, dtype, terms ? v.data() : nullptr, n, dst, src, aux, nullptr, 0, acc_origin, zsize, nbox,
                                 lo, hi);
}

int sb_stencil_vplan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                            sb_pitched src, sb_pitched aux, const sb_pitched *coef, int ncoef, const int64_t acc_origin[3],
                            int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi) {
  return sb_stencil_cplan_create(out, device, dtype, terms, n, dst, src, aux, coef, ncoef, 1, 0, acc_origin, zsize, nbox, lo, hi);
}

int sb_stencil_cplan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                            sb_pitched src, sb_pitched aux, const sb_pitched *coef, int ncoef, int ncolours, int colour,
                            const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi) {
  return stencil_plan_build(out, device, dtype, terms, n, dst, src, aux, coef, ncoef, ncolours, colour, acc_origin, zsize, nbox, lo, hi, nullptr);
}

int sb_stencil_dplan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                            sb_pitched src, sb_pitched f, const sb_pitched *coef, int ncoef, double omega, int ncolours, int colour,
                            const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi) {
  return stencil_plan_build(out, device, dtype, terms, n, dst, src, f, coef, ncoef, ncolours, colour, acc_origin, zsize, nbox, lo, hi, &omega);
}

// sb_stencil_cplan_create, and with omega non-NULL sb_stencil_dplan_create (aux is f)
static int stencil_plan_build(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                              sb_pitched src, sb_pitched aux, const sb_pitched *coef, int ncoef, int ncolours, int colour,
                              const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi,
                              const double *omega) {
  if (!out) return fail(SB_ERR_INVALID, "sb_stencil_plan_create needs an output handle");
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) return fail(SB_ERR_INVALID, "dtype %d must be SB_DTYPE_F32 or SB_DTYPE_F64", dtype);
  const int es = dtype == SB_DTYPE_F32 ? 4 : 8;
  int rc = stencil_terms_ok(terms, n);
  if (rc != SB_OK) return rc;
  const bool diag = omega != nullptr;
  unsigned long long centre = 0;
  if (diag) {
    for (int t = 0; t < n; ++t) {
      if (terms[t].source == 1) return fail(SB_ERR_INVALID, "sb_stencil_dplan_create: term %d reads aux; A reads src only (f goes on aux)", t);
      if (!terms[t].offset[0] && !terms[t].offset[1] && !terms[t].offset[2]) centre |= 1ull << t;
    }
    if (!centre) return fail(SB_ERR_INVALID, "sb_stencil_dplan_create: A has no term at offset (0, 0, 0), so no diagonal");
    if (!std::isfinite(*omega)) return fail(SB_ERR_INVALID, "sb_stencil_dplan_create: omega = %g must be finite", *omega);
    if (!aux.ptr) return fail(SB_ERR_INVALID, "sb_stencil_dplan_create: f is NULL");
  }
  if ((rc = stencil_colours_ok(terms, n, ncolours)) != SB_OK) return rc;
  if (colour < 0 || colour >= ncolours) return fail(SB_ERR_INVALID, "colour %d: 0 .. %d under %d colours", colour, ncolours - 1, ncolours);
  if (ncoef < 0 || ncoef > SB_STENCIL_MAX_COEFS) return fail(SB_ERR_INVALID, "ncoef %d: 0 to %d coefficient fields", ncoef, SB_STENCIL_MAX_COEFS);
  if (ncoef > 0 && !coef) return fail(SB_ERR_INVALID, "ncoef %d, but the coefficient array is NULL", ncoef);
  bool has_aux = diag; // the diagonal mode reads f on aux
  int rm[3] = {0, 0, 0}, rp[3] = {0, 0, 0}, R = 1;
  // coefficient fields the op references, renumbered 0 .. nf - 1 in order of their index, with their reach per axis
  int fmap[SB_STENCIL_MAX_COEFS] = {-1, -1, -1, -1}, fsrc[SB_STENCIL_MAX_COEFS] = {}, nf = 0;
  int crm[SB_STENCIL_MAX_COEFS][3] = {}, crp[SB_STENCIL_MAX_COEFS][3] = {};
  for (int t = 0; t < n; ++t) {
    has_aux = has_aux || terms[t].source == 1;
    for (int a = 0; a < 3; ++a) {
      const int o = terms[t].offset[a];
      rm[a] = std::max(rm[a], -o);
      rp[a] = std::max(rp[a], o);
      R = std::max(R, std::abs(o));
    }
    const int k = terms[t].coef;
    if (k >= ncoef) return fail(SB_ERR_INVALID, "term %d names coefficient field %d, but ncoef is %d", t, k, ncoef);
    if (k >= 0 && !coef[k].ptr) return fail(SB_ERR_INVALID, "coefficient field %d is NULL", k);
  }
  for (int k = 0; k < ncoef; ++k)
    for (int t = 0; t < n; ++t)
      if (terms[t].coef == k) {
        if (fmap[k] < 0) {
          fmap[k] = nf;
          fsrc[nf++] = k;
        }
        for (int a = 0; a < 3; ++a) {
          crm[fmap[k]][a] = std::max(crm[fmap[k]][a], -terms[t].coef_offset[a]);
          crp[fmap[k]][a] = std::max(crp[fmap[k]][a], terms[t].coef_offset[a]);
        }
      }
  if (has_aux && !aux.ptr) return fail(SB_ERR_INVALID, "the op has a term on aux, but aux is NULL");
  if (!dst.ptr || !src.ptr) return fail(SB_ERR_INVALID, "dst and src must not be NULL");
  if (dst.ptr == src.ptr && ncolours == 1) return fail(SB_ERR_INVALID, "dst must not be src (dst may be %s)", diag ? "f" : "aux");
  for (int f = 0; f < nf; ++f)
    if (coef[fsrc[f]].ptr == dst.ptr) return fail(SB_ERR_INVALID, "coefficient field %d is dst (coefficients are read only)", fsrc[f]);
  std::vector<const sb_pitched *> bufs = {&dst, &src};
  std::vector<std::string> names = {"dst", "src"};
  if (has_aux) {
    bufs.push_back(&aux);
    names.push_back("aux");
  }
  for (int f = 0; f < nf; ++f) {
    bufs.push_back(&coef[fsrc[f]]);
    names.push_back("coefficient field " + std::to_string(fsrc[f]));
  }
  if ((rc = stencil_buffers_ok(bufs, names, src, "src", es)) != SB_OK) return rc;
  if (!acc_origin || zsize < 1) return fail(SB_ERR_INVALID, "sb_stencil_plan_create needs acc_origin and zsize >= 1");
  if (nbox < 0 || (nbox > 0 && (!lo || !hi))) return fail(SB_ERR_INVALID, "nbox %d: needs nbox >= 0 and lo / hi arrays", nbox);
  const int64_t size[3] = {src.pitch / es, src.ysize, zsize};
  PlanBoxes B;
  int64_t written = 0;
  rc = plan_boxes(nbox, lo, hi, acc_origin, 8, [&](int b, const int64_t l[3], const int64_t e[3]) {
    int rc = stencil_box_reads_ok(b, l, e, rm, rp, size, "the op reads");
    for (int f = 0; f < nf && rc == SB_OK; ++f)
      rc = stencil_box_reads_ok(b, l, e, crm[f], crp[f], size, "coefficient field " + std::to_string(fsrc[f]) + " is read at");
    written += stencil_colour_cells(&lo[3 * b], e, ncolours, colour);
    return rc;
  }, B);
  if (rc != SB_OK) return rc;
  sb::OpColour col{ncolours, colour, {}};
  for (int a = 0; a < 3; ++a) col.par[a] = int(((acc_origin[a] % 2) + 2) % 2);
  sb::OpDiag dg{diag ? 1 : 0, centre, diag ? *omega : 0.0, diag ? float(*omega) : 0.0f};

  sb::OpCommon com{};
  com.dst = static_cast<char *>(dst.ptr);
  com.src = static_cast<const char *>(src.ptr);
  com.aux = has_aux ? static_cast<const char *>(aux.ptr) : nullptr;
  com.pitch = src.pitch;
  com.slice = src.pitch * src.ysize;
  com.n = n;
  com.has_aux = has_aux ? 1 : 0;
  for (int t = 0; t < n; ++t) {
    com.source[t] = (signed char)terms[t].source;
    com.w[t] = terms[t].weight;
    com.wf[t] = float(terms[t].weight); // round to nearest
  }

  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  int sms = 0;
  SB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  std::unique_ptr<sb_stencil_plan> p(new sb_stencil_plan());
  p->device = device;
  p->bytes = B.cells * es * ((has_aux ? 2 : 1) + nf) + written * es;
  if (!B.thick.empty()) {
    const int per_sm = sb::op_tile_prepare(R, es, device, nf, ncolours > 1, diag);
    if (per_sm <= 0) return fail(SB_ERR_CUDA, "the R = %d tile kernel cannot be configured: %s", R, cudaGetErrorString(cudaGetLastError()));
    const int SW = sb::op_tile_sw(R), P = sb::op_tile_plane(R), NS = 2 * R + 1;
    const int CSW = sb::op_tile_sw(1), CP = sb::op_tile_plane(1), CS = sb::kOpCoefSlots;
    for (const PlanBox &b : B.thick) {
      sb::OpDTileParams tp{};
      tp.c = com;
      tp.col = col;
      tp.dg = dg;
      tp.k.nf = nf;
      for (int f = 0; f < nf; ++f) {
        tp.k.coef[f] = static_cast<const char *>(coef[fsrc[f]].ptr);
        for (int a = 0; a < 3; ++a) {
          tp.k.crm[f][a] = crm[f][a];
          tp.k.crp[f][a] = crp[f][a];
        }
      }
      for (int t = 0; t < n; ++t) {
        const int f = terms[t].coef < 0 ? -1 : fmap[terms[t].coef];
        tp.k.cfield[t] = (signed char)f;
        const int32_t *c = terms[t].coef_offset;
        for (int s = 0; s < CS && f >= 0; ++s) tp.k.coff[s][t] = short((f * CS + (s + c[2] + CS) % CS) * CP + c[1] * CSW + c[0]);
      }
      tp.src_end = com.src + com.slice * zsize;
      for (int a = 0; a < 3; ++a) {
        tp.lo[a] = b.lo[a];
        tp.ext[a] = b.ext[a];
        tp.rm[a] = rm[a];
        tp.rp[a] = rp[a];
      }
      // each chunk reloads rm + rp planes
      int grid = 0;
      if ((rc = tile_grid(tp, tp.ext, sb::kOpTileX, sb::kOpTileY, sms, per_sm, 16, "tile kernel", grid)) != SB_OK) return rc;
      for (int c = 0; c < NS; ++c)
        for (int t = 0; t < n; ++t) {
          const int32_t *o = terms[t].offset;
          tp.toff[c][t] = ((c + o[2] + NS) % NS) * P + o[1] * SW + o[0];
        }
      p->launches.push_back([tp, R, es, grid](cudaStream_t s) { return sb::launch_op_tile(tp, R, es, grid, s); });
    }
  }
  sb::OpDCellParams cp{};
  cp.c = com;
  cp.col = col;
  cp.dg = dg;
  for (int t = 0; t < n; ++t)
    cp.goff[t] = (long long)terms[t].offset[2] * com.slice + (long long)terms[t].offset[1] * com.pitch + (long long)terms[t].offset[0] * es;
  for (int f = 0; f < nf; ++f) cp.coef[f] = static_cast<const char *>(coef[fsrc[f]].ptr);
  for (int t = 0; t < n; ++t) {
    const int32_t *c = terms[t].coef_offset;
    cp.cfield[t] = (signed char)(terms[t].coef < 0 ? -1 : fmap[terms[t].coef]);
    cp.cgoff[t] = (long long)c[2] * com.slice + (long long)c[1] * com.pitch + (long long)c[0] * es;
  }
  const bool has_coef = nf > 0;
  cell_groups(B.thin, cp, &sb::OpDCellParams::n, sms, [&](const sb::OpDCellParams &g, int grid) {
    p->launches.push_back([g, es, has_coef, grid](cudaStream_t s) { return sb::launch_op_cells(g, es, has_coef, grid, s); });
  });
  *out = p.release();
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- linear stencil systems
// The limits every system obeys, whatever the domain: counts, indices, and each term's offsets as for an operator.
static int stencil_sys_terms_ok(const sb_stencil_sys_term *terms, int n, int nin, int nout) {
  if (nin < 1 || nin > SB_STENCIL_SYS_MAX_INPUTS) return fail(SB_ERR_INVALID, "a system has 1 to %d inputs, not %d", SB_STENCIL_SYS_MAX_INPUTS, nin);
  if (nout < 1 || nout > SB_STENCIL_SYS_MAX_OUTPUTS) return fail(SB_ERR_INVALID, "a system has 1 to %d outputs, not %d", SB_STENCIL_SYS_MAX_OUTPUTS, nout);
  if (!terms || n < 1 || n > SB_STENCIL_SYS_MAX_TERMS)
    return fail(SB_ERR_INVALID, "a system has 1 to %d terms, not %d", SB_STENCIL_SYS_MAX_TERMS, terms ? n : 0);
  for (int t = 0; t < n; ++t) {
    const sb_stencil_sys_term &T = terms[t];
    if (T.output < 0 || T.output >= nout) return fail(SB_ERR_INVALID, "term %d: output %d must be 0 .. %d", t, int(T.output), nout - 1);
    if (T.input < 0 || T.input >= nin) return fail(SB_ERR_INVALID, "term %d: input %d must be 0 .. %d", t, int(T.input), nin - 1);
    int rc = stencil_offset_ok(t, T.offset);
    if (rc != SB_OK || (rc = stencil_coef_ok(t, T.coef, T.coef_offset, nin, "input")) != SB_OK) return rc;
  }
  return SB_OK;
}

int sb_stencil_sys_check(const sb_stencil_sys_term *terms, int n, int nin, int nout, const int64_t radius27[27]) {
  if (!radius27) return fail(SB_ERR_INVALID, "sb_stencil_sys_check needs radius27");
  int rc = stencil_sys_terms_ok(terms, n, nin, nout);
  if (rc != SB_OK) return rc;
  for (int t = 0; t < n; ++t) {
    if ((rc = stencil_offset_in_reach(t, "offset", terms[t].offset, radius27)) != SB_OK) return rc;
    if (terms[t].coef >= 0 && (rc = stencil_offset_in_reach(t, "coefficient offset", terms[t].coef_offset, radius27)) != SB_OK) return rc;
  }
  return SB_OK;
}

// The difference D_a of input `in` into output `out` with the given stagger, times sign (+1 or -1, exact): two terms.
static void stencil_diff_terms(int stagger, int a, double h, int out, int in, double sign, std::vector<sb_stencil_sys_term> &v) {
  const double w = stagger == 0 ? 0.5 / h : 1.0 / h;
  const int hi = stagger >= 0 ? 1 : 0, lo = stagger <= 0 ? -1 : 0; // the offsets along a of the + and the - term
  sb_stencil_sys_term t{out, in, {0, 0, 0}, -1, {0, 0, 0}, sign * w};
  t.offset[a] = hi;
  v.push_back(t);
  t.offset[a] = lo;
  t.weight = -(sign * w);
  v.push_back(t);
}

static int stencil_table_ok(const char *name, int stagger, const double spacing[3], const sb_stencil_sys_term *out, int cap) {
  if (stagger < -1 || stagger > 1) return fail(SB_ERR_INVALID, "%s: stagger %d must be -1 (backward), 0 (central) or +1 (forward)", name, stagger);
  if (!spacing) return fail(SB_ERR_INVALID, "%s needs spacing[3]", name);
  for (int a = 0; a < 3; ++a)
    if (!(spacing[a] > 0.0) || !std::isfinite(spacing[a])) return fail(SB_ERR_INVALID, "spacing[%d] = %g must be finite and > 0", a, spacing[a]);
  if (cap < 0 || (cap > 0 && !out)) return fail(SB_ERR_INVALID, "%s: bad output buffer", name);
  return SB_OK;
}

static int stencil_table_put(const std::vector<sb_stencil_sys_term> &v, sb_stencil_sys_term *out, int cap) {
  for (int i = 0; i < int(v.size()) && i < cap; ++i) out[i] = v[size_t(i)];
  return int(v.size());
}

int sb_stencil_grad(int stagger, const double spacing[3], sb_stencil_sys_term *out, int cap) {
  int rc = stencil_table_ok("sb_stencil_grad", stagger, spacing, out, cap);
  if (rc != SB_OK) return rc;
  std::vector<sb_stencil_sys_term> v;
  for (int a = 0; a < 3; ++a) stencil_diff_terms(stagger, a, spacing[a], a, 0, 1.0, v);
  return stencil_table_put(v, out, cap);
}

int sb_stencil_div(int stagger, const double spacing[3], sb_stencil_sys_term *out, int cap) {
  int rc = stencil_table_ok("sb_stencil_div", stagger, spacing, out, cap);
  if (rc != SB_OK) return rc;
  std::vector<sb_stencil_sys_term> v;
  for (int a = 0; a < 3; ++a) stencil_diff_terms(stagger, a, spacing[a], 0, a, 1.0, v);
  return stencil_table_put(v, out, cap);
}

int sb_stencil_curl(int stagger, const double spacing[3], sb_stencil_sys_term *out, int cap) {
  int rc = stencil_table_ok("sb_stencil_curl", stagger, spacing, out, cap);
  if (rc != SB_OK) return rc;
  std::vector<sb_stencil_sys_term> v;
  for (int j = 0; j < 3; ++j) { // output j = D_{j+1} in_{j+2} - D_{j+2} in_{j+1}
    const int a = (j + 1) % 3, b = (j + 2) % 3;
    stencil_diff_terms(stagger, a, spacing[a], j, b, 1.0, v);
    stencil_diff_terms(stagger, b, spacing[b], j, a, -1.0, v);
  }
  return stencil_table_put(v, out, cap);
}

int sb_stencil_sys_plan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_sys_term *terms, int n,
                               const sb_pitched *outputs, int nout, const sb_pitched *inputs, int nin, const int64_t acc_origin[3],
                               int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi) {
  constexpr int NI = SB_STENCIL_SYS_MAX_INPUTS, NO = SB_STENCIL_SYS_MAX_OUTPUTS;
  static_assert(NI == sb::kSysMaxInputs && NO == sb::kSysMaxOutputs && SB_STENCIL_SYS_MAX_TERMS == sb::kSysMaxTerms, "one set of limits");
  if (!out) return fail(SB_ERR_INVALID, "sb_stencil_sys_plan_create needs an output handle");
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) return fail(SB_ERR_INVALID, "dtype %d must be SB_DTYPE_F32 or SB_DTYPE_F64", dtype);
  const int es = dtype == SB_DTYPE_F32 ? 4 : 8;
  int rc = stencil_sys_terms_ok(terms, n, nin, nout);
  if (rc != SB_OK) return rc;
  if (!outputs || !inputs) return fail(SB_ERR_INVALID, "sb_stencil_sys_plan_create needs the output and input arrays");
  // the inputs the terms read, each with its reach per axis and side, and whether any read has a non-zero offset
  bool used[NI] = {}, moved[NI] = {};
  int rm[NI][3] = {}, rp[NI][3] = {}, count[NO] = {};
  auto reads = [&](int i, const int32_t o[3]) {
    used[i] = true;
    for (int a = 0; a < 3; ++a) {
      rm[i][a] = std::max(rm[i][a], -o[a]);
      rp[i][a] = std::max(rp[i][a], o[a]);
      moved[i] = moved[i] || o[a] != 0;
    }
  };
  for (int t = 0; t < n; ++t) {
    ++count[terms[t].output];
    reads(terms[t].input, terms[t].offset);
    if (terms[t].coef >= 0) reads(terms[t].coef, terms[t].coef_offset);
  }
  for (int j = 0; j < nout; ++j) {
    if (!count[j]) return fail(SB_ERR_INVALID, "output %d has no terms", j);
    if (!outputs[j].ptr) return fail(SB_ERR_INVALID, "output %d is NULL", j);
    for (int k = 0; k < j; ++k)
      if (outputs[k].ptr == outputs[j].ptr) return fail(SB_ERR_INVALID, "outputs %d and %d are the same buffer", k, j);
  }
  for (int i = 0; i < nin; ++i) {
    if (!used[i]) continue;
    if (!inputs[i].ptr) return fail(SB_ERR_INVALID, "input %d is read by a term, but it is NULL", i);
    for (int j = 0; j < nout && moved[i]; ++j)
      if (outputs[j].ptr == inputs[i].ptr)
        return fail(SB_ERR_INVALID, "output %d is input %d, which a term reads at a non-zero offset (an output may be an input read only at offset 0)", j, i);
  }
  std::vector<const sb_pitched *> bufs;
  std::vector<std::string> names;
  for (int j = 0; j < nout; ++j) {
    bufs.push_back(&outputs[j]);
    names.push_back("output " + std::to_string(j));
  }
  for (int i = 0; i < nin; ++i)
    if (used[i]) {
      bufs.push_back(&inputs[i]);
      names.push_back("input " + std::to_string(i));
    }
  if ((rc = stencil_buffers_ok(bufs, names, outputs[0], "output 0", es)) != SB_OK) return rc;
  if (!acc_origin || zsize < 1) return fail(SB_ERR_INVALID, "sb_stencil_sys_plan_create needs acc_origin and zsize >= 1");
  if (nbox < 0 || (nbox > 0 && (!lo || !hi))) return fail(SB_ERR_INVALID, "nbox %d: needs nbox >= 0 and lo / hi arrays", nbox);
  const int64_t pitch = outputs[0].pitch, slice = pitch * outputs[0].ysize;
  const int64_t size[3] = {pitch / es, outputs[0].ysize, zsize};
  PlanBoxes B;
  rc = plan_boxes(nbox, lo, hi, acc_origin, 8, [&](int b, const int64_t l[3], const int64_t e[3]) {
    int rc = SB_OK;
    for (int i = 0; i < nin && rc == SB_OK; ++i)
      if (used[i]) rc = stencil_box_reads_ok(b, l, e, rm[i], rp[i], size, "input " + std::to_string(i) + " is read at");
    return rc;
  }, B);
  if (rc != SB_OK) return rc;

  // the read inputs renumbered 0 .. nr - 1 (ring r of the tile kernel); each ring's plane size; the shared row width fits
  // the widest window shifted onto 16-byte phase
  int ri[NI], src_of[NI], nr = 0, rx = 0;
  for (int i = 0; i < nin; ++i) {
    ri[i] = used[i] ? nr : -1;
    if (used[i]) {
      src_of[nr++] = i;
      rx = std::max(rx, rm[i][0] + rp[i][0]);
    }
  }
  const int V = 16 / es;
  const int sw = (V - 1 + sb::kOpTileX + rx + V - 1) / V * V;
  int base[NI] = {}, ns[NI] = {};
  size_t ring_elems = 0;
  for (int r = 0; r < nr; ++r) {
    const int i = src_of[r];
    ns[r] = rm[i][2] + rp[i][2] + 2;
    base[r] = int(ring_elems);
    ring_elems += size_t(ns[r]) * size_t(sb::kOpTileY + rm[i][1] + rp[i][1]) * size_t(sw);
  }
  const size_t smem = size_t(sb::kSysTableBytes) + ring_elems * size_t(es);
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  int sms = 0, optin = 0;
  SB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  SB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
  if (!B.thick.empty() && smem > size_t(optin))
    return fail(SB_ERR_INVALID, "the system's tile kernel needs %zu bytes of shared memory per block, the device allows %d", smem, optin);

  // the terms sorted by output (stable): the rule sums each output's terms in list order
  std::vector<int> order;
  sb::SysTerms com{};
  for (int j = 0; j < nout; ++j) {
    com.first[j] = int(order.size());
    for (int t = 0; t < n; ++t)
      if (terms[t].output == j) order.push_back(t);
    com.out[j] = static_cast<char *>(outputs[j].ptr);
  }
  com.first[nout] = n;
  com.pitch = pitch;
  com.slice = slice;
  com.n = n;
  com.nout = nout;
  for (int k = 0; k < n; ++k) {
    const sb_stencil_sys_term &T = terms[order[size_t(k)]];
    com.in[k] = (signed char)ri[T.input];
    com.cin[k] = (signed char)(T.coef < 0 ? -1 : ri[T.coef]);
    com.w[k] = T.weight;
    com.wf[k] = float(T.weight); // round to nearest
  }

  std::unique_ptr<sb_stencil_plan> p(new sb_stencil_plan());
  p->device = device;
  p->bytes = B.cells * es * (nr + nout);
  if (!B.thick.empty()) {
    const int per_sm = sb::sys_tile_prepare(es, device, smem);
    if (per_sm <= 0) return fail(SB_ERR_CUDA, "the system tile kernel cannot be configured: %s", cudaGetErrorString(cudaGetLastError()));
    for (const PlanBox &b : B.thick) {
      sb::SysTileParams tp{};
      tp.c = com;
      tp.nr = nr;
      tp.sw = sw;
      int shift[NI] = {};
      for (int r = 0; r < nr; ++r) {
        const int i = src_of[r];
        tp.in[r] = static_cast<const char *>(inputs[i].ptr);
        tp.vec[r] = pitch % 16 == 0; // else rows alternate between 16-byte phases: elements one by one
        shift[r] = tp.vec[r] ? int((uintptr_t(tp.in[r]) + uintptr_t(int64_t(b.lo[0] - rm[i][0]) * es)) % 16) / es : 0;
        tp.shift[r] = shift[r];
        tp.ns[r] = ns[r];
        tp.base[r] = base[r];
        for (int a = 0; a < 3; ++a) {
          tp.rm[r][a] = rm[i][a];
          tp.rp[r][a] = rp[i][a];
        }
      }
      // a read's shared offset within its plane, from the cell's own slot position wy * sw + lane
      auto inplane = [&](int r, const int32_t o[3]) { return (tp.rm[r][1] + o[1]) * sw + tp.rm[r][0] + shift[r] + o[0]; };
      for (int k = 0; k < n; ++k) {
        const sb_stencil_sys_term &T = terms[order[size_t(k)]];
        tp.oz[k] = (signed char)T.offset[2];
        tp.inpl[k] = inplane(com.in[k], T.offset);
        if (com.cin[k] >= 0) {
          tp.coz[k] = (signed char)T.coef_offset[2];
          tp.cinpl[k] = inplane(com.cin[k], T.coef_offset);
        }
      }
      for (int a = 0; a < 3; ++a) {
        tp.lo[a] = b.lo[a];
        tp.ext[a] = b.ext[a];
      }
      // z chunks as for an operator
      int grid = 0;
      if ((rc = tile_grid(tp, tp.ext, sb::kOpTileX, sb::kOpTileY, sms, per_sm, 16, "tile kernel", grid)) != SB_OK) return rc;
      p->launches.push_back([tp, es, smem, grid](cudaStream_t s) { return sb::launch_sys_tile(tp, es, smem, grid, s); });
    }
  }
  sb::SysCellParams cp{};
  cp.c = com;
  for (int r = 0; r < nr; ++r) cp.in[r] = static_cast<const char *>(inputs[src_of[r]].ptr);
  for (int k = 0; k < n; ++k) {
    const sb_stencil_sys_term &T = terms[order[size_t(k)]];
    for (int a = 0; a < 3; ++a) {
      cp.o[k][a] = (signed char)T.offset[a];
      cp.co[k][a] = (signed char)T.coef_offset[a];
    }
  }
  cell_groups(B.thin, cp, &sb::SysCellParams::nb, sms, [&](const sb::SysCellParams &g, int grid) {
    p->launches.push_back([g, es, grid](cudaStream_t s) { return sb::launch_sys_cells(g, es, grid, s); });
  });
  *out = p.release();
  return SB_OK;
}

int sb_stencil_plan_launch(sb_stencil_plan *p, void *stream) { return run_launches(p, stream); }

int64_t sb_stencil_plan_bytes(const sb_stencil_plan *p) { return p ? p->bytes : 0; }

int sb_stencil_plan_destroy(sb_stencil_plan *p) {
  delete p;
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- multigrid transfers
static int64_t floor_half(int64_t v) { return v >= 0 ? v / 2 : -((1 - v) / 2); }

int sb_transfer_check(const int64_t fine_dim[3], const int64_t coarse_dim[3], const int64_t *fine_origin, const int64_t *fine_size,
                      const int64_t *coarse_origin, const int64_t *coarse_size, const int64_t coarse_radius27[27]) {
  if (!fine_dim || !coarse_dim || !fine_origin || !fine_size || !coarse_origin || !coarse_size)
    return fail(SB_ERR_INVALID, "sb_transfer_check needs both dims and the origin and size arrays");
  for (int a = 0; a < 3; ++a) {
    if (fine_dim[a] < 1 || coarse_dim[a] < 1) return fail(SB_ERR_INVALID, "a partition has at least one subdomain on every axis");
    if (fine_dim[a] != coarse_dim[a])
      return fail(SB_ERR_INVALID, "the fine partition is %lld x %lld x %lld subdomains, the coarse one %lld x %lld x %lld: they must be the same",
                  (long long)fine_dim[0], (long long)fine_dim[1], (long long)fine_dim[2], (long long)coarse_dim[0], (long long)coarse_dim[1],
                  (long long)coarse_dim[2]);
  }
  const int64_t n = fine_dim[0] * fine_dim[1] * fine_dim[2];
  for (int64_t k = 0; k < n; ++k) {
    const long long i = (long long)(k % fine_dim[0]), j = (long long)((k / fine_dim[0]) % fine_dim[1]),
                    l = (long long)(k / (fine_dim[0] * fine_dim[1]));
    for (int a = 0; a < 3; ++a) {
      const int64_t fo = fine_origin[3 * k + a], co = coarse_origin[3 * k + a], fs = fine_size[3 * k + a], cs = coarse_size[3 * k + a];
      if (fo != 2 * co)
        return fail(SB_ERR_INVALID, "subdomain (%lld, %lld, %lld): fine origin %lld on axis %c is not twice the coarse origin %lld", i, j, l,
                    (long long)fo, "xyz"[a], (long long)co);
      if (fs != 2 * cs)
        return fail(SB_ERR_INVALID, "subdomain (%lld, %lld, %lld): fine size %lld on axis %c is not twice the coarse size %lld", i, j, l,
                    (long long)fs, "xyz"[a], (long long)cs);
    }
  }
  if (coarse_radius27)
    for (int z = -1; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x)
          if ((x || y || z) && coarse_radius27[(z + 1) * 9 + (y + 1) * 3 + (x + 1)] < 1)
            return fail(SB_ERR_INVALID, "the coarse radius in direction (%d, %d, %d) is 0: prolongation reads one ghost layer in all 26 directions",
                        x, y, z);
  return SB_OK;
}

// sb_transfer_plan_create, and with face >= 0 (a restriction) sb_transfer_fplan_create
static int transfer_plan_build(sb_transfer_plan **out, int device, int dtype, int kind, sb_pitched dst, const int64_t dst_acc_origin[3],
                               int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3], int64_t src_zsize, sb_pitched aux,
                               const int64_t lo[3], const int64_t hi[3], int face, const char *fn);

int sb_transfer_plan_create(sb_transfer_plan **out, int device, int dtype, int kind, sb_pitched dst, const int64_t dst_acc_origin[3],
                            int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3], int64_t src_zsize, sb_pitched aux,
                            const int64_t lo[3], const int64_t hi[3]) {
  if (kind != SB_TRANSFER_RESTRICT && kind != SB_TRANSFER_PROLONG)
    return fail(SB_ERR_INVALID, "kind %d must be SB_TRANSFER_RESTRICT or SB_TRANSFER_PROLONG", kind);
  return transfer_plan_build(out, device, dtype, kind, dst, dst_acc_origin, dst_zsize, src, src_acc_origin, src_zsize, aux, lo, hi, -1,
                             "sb_transfer_plan_create");
}

int sb_transfer_fplan_create(sb_transfer_plan **out, int device, int dtype, int axis, sb_pitched dst, const int64_t dst_acc_origin[3],
                             int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3], int64_t src_zsize,
                             const int64_t lo[3], const int64_t hi[3]) {
  if (axis < 0 || axis > 2) return fail(SB_ERR_INVALID, "sb_transfer_fplan_create: axis %d must be 0, 1 or 2", axis);
  return transfer_plan_build(out, device, dtype, SB_TRANSFER_RESTRICT, dst, dst_acc_origin, dst_zsize, src, src_acc_origin, src_zsize,
                             sb_pitched{nullptr, 0, 0}, lo, hi, axis, "sb_transfer_fplan_create");
}

static int transfer_plan_build(sb_transfer_plan **out, int device, int dtype, int kind, sb_pitched dst, const int64_t dst_acc_origin[3],
                               int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3], int64_t src_zsize, sb_pitched aux,
                               const int64_t lo[3], const int64_t hi[3], int face, const char *fn) {
  if (!out) return fail(SB_ERR_INVALID, "%s needs an output handle", fn);
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) return fail(SB_ERR_INVALID, "dtype %d must be SB_DTYPE_F32 or SB_DTYPE_F64", dtype);
  const int es = dtype == SB_DTYPE_F32 ? 4 : 8;
  const bool prolong = kind == SB_TRANSFER_PROLONG, has_aux = aux.ptr != nullptr;
  if (!dst.ptr || !src.ptr) return fail(SB_ERR_INVALID, "dst and src must not be NULL");
  if (dst.ptr == src.ptr) return fail(SB_ERR_INVALID, "dst must not be src");
  if (has_aux && !prolong) return fail(SB_ERR_INVALID, "a restriction takes no aux");
  if (!dst_acc_origin || !src_acc_origin || !lo || !hi) return fail(SB_ERR_INVALID, "%s needs both acc_origins, lo and hi", fn);
  if (dst_zsize < 1 || src_zsize < 1) return fail(SB_ERR_INVALID, "dst_zsize and src_zsize must be >= 1");
  int rc = stencil_buffers_ok({&dst}, {"dst"}, dst, "dst", es);
  if (rc == SB_OK) rc = stencil_buffers_ok({&src}, {"src"}, src, "src", es);
  if (rc == SB_OK && has_aux) rc = stencil_buffers_ok({&aux}, {"aux"}, dst, "dst", es);
  if (rc != SB_OK) return rc;
  const int64_t dsize[3] = {dst.pitch / es, dst.ysize, dst_zsize}, ssize[3] = {src.pitch / es, src.ysize, src_zsize};
  int64_t l[3], e[3];
  bool empty = false;
  for (int a = 0; a < 3; ++a) {
    if (lo[a] > hi[a]) return fail(SB_ERR_INVALID, "lo > hi on axis %c", "xyz"[a]);
    l[a] = lo[a] - dst_acc_origin[a];
    e[a] = hi[a] - lo[a];
    empty = empty || e[a] == 0;
  }
  std::unique_ptr<sb_transfer_plan> p(new sb_transfer_plan());
  p->device = device;
  if (empty) {
    *out = p.release();
    return SB_OK;
  }
  const int zero[3] = {0, 0, 0};
  if ((rc = stencil_box_reads_ok(0, l, e, zero, zero, dsize, "dst is written at")) != SB_OK) return rc;
  // src reads [rl, rl + re) (allocation coordinates) that the checks cover
  int64_t rl[3], re[3];
  for (int a = 0; a < 3; ++a) {
    if (prolong) {
      rl[a] = floor_half(lo[a]) - 1 - src_acc_origin[a];
      re[a] = floor_half(hi[a] - 1) + 2 - floor_half(lo[a]) + 1;
    } else {
      rl[a] = 2 * lo[a] - src_acc_origin[a];
      re[a] = 2 * e[a];
    }
  }
  if ((rc = stencil_box_reads_ok(0, rl, re, zero, zero, ssize, prolong ? "the prolongation reads coarse" : "the restriction reads fine")) != SB_OK)
    return rc;
  if (over_2_32_cells(e)) return fail(SB_ERR_INVALID, "a box of more than 2^32 cells");
  for (int a = 0; a < 3 && prolong; ++a) { // a child's dst coordinate is 2 * (its parent's src coordinate) + off, in int
    const int64_t off = 2 * src_acc_origin[a] - dst_acc_origin[a];
    if (off < -(1ll << 31) || off >= (1ll << 31))
      return fail(SB_ERR_INVALID, "the prolongation's offset 2 * src_acc_origin - dst_acc_origin = %lld on axis %c does not fit 32 bits",
                  (long long)off, "xyz"[a]);
  }

  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  int sms = 0;
  SB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  const int64_t cells = e[0] * e[1] * e[2];
  if (!prolong) {
    sb::RestrictParams r{};
    r.dst = static_cast<char *>(dst.ptr);
    r.src = static_cast<const char *>(src.ptr);
    r.dpitch = dst.pitch;
    r.dslice = dst.pitch * dst.ysize;
    r.spitch = src.pitch;
    r.sslice = src.pitch * src.ysize;
    for (int a = 0; a < 3; ++a) {
      r.lo[a] = int(l[a]);
      r.ext[a] = int(e[a]);
      r.flo[a] = int(rl[a]);
    }
    p->bytes = (face >= 0 ? 4 + 1 : 8 + 1) * cells * es;
    if (face >= 0)
      p->launches.push_back([r, es, face](cudaStream_t s) { return sb::launch_face_restrict(r, es, face, s); });
    else
      p->launches.push_back([r, es](cudaStream_t s) { return sb::launch_restrict(r, es, s); });
  } else {
    sb::ProlongParams q{};
    q.dst = static_cast<char *>(dst.ptr);
    q.aux = has_aux ? static_cast<const char *>(aux.ptr) : nullptr;
    q.src = static_cast<const char *>(src.ptr);
    q.dpitch = dst.pitch;
    q.dslice = dst.pitch * dst.ysize;
    q.spitch = src.pitch;
    q.sslice = src.pitch * src.ysize;
    int64_t reads = 1;
    for (int a = 0; a < 3; ++a) {
      q.lo[a] = int(l[a]);
      q.ext[a] = int(e[a]);
      q.off[a] = int(2 * src_acc_origin[a] - dst_acc_origin[a]);
      q.plo[a] = int(floor_half(lo[a]) - src_acc_origin[a]);
      q.pext[a] = int(floor_half(hi[a] - 1) - floor_half(lo[a]) + 1);
      // the cells the rule reads: a child at an even coordinate reads its parent's lower neighbour, at an odd one the upper
      q.rlo[a] = int(floor_half(lo[a] - 1) - src_acc_origin[a]);
      q.rhi[a] = int(floor_half(hi[a]) + 1 - src_acc_origin[a]);
      reads *= q.rhi[a] - q.rlo[a];
    }
    p->bytes = reads * es + cells * es * (has_aux ? 2 : 1);
    const int per_sm = sb::prolong_ctas_per_sm(es);
    if (per_sm <= 0) return fail(SB_ERR_CUDA, "the prolongation kernel cannot be configured: %s", cudaGetErrorString(cudaGetLastError()));
    // over the parents, chunks of at least 8 parent planes (each chunk reloads 2 planes)
    int grid = 0;
    if ((rc = tile_grid(q, q.pext, sb::kProlongX, sb::kProlongY, sms, per_sm, 8, "prolongation kernel", grid)) != SB_OK) return rc;
    p->launches.push_back([q, es, grid](cudaStream_t s) { return sb::launch_prolong(q, es, grid, s); });
  }
  *out = p.release();
  return SB_OK;
}

static int transfer_oplan_build(const char *fn, sb_transfer_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n,
                                sb_pitched dst, const int64_t dst_acc_origin[3], int64_t dst_zsize, sb_pitched src,
                                const int64_t src_acc_origin[3], int64_t src_zsize, sb_pitched aux, const sb_pitched *coef, int ncoef,
                                int nbox, const int64_t *lo, const int64_t *hi);

int sb_transfer_oplan_create(sb_transfer_plan **out, int device, int dtype, const sb_stencil_term *terms, int n, sb_pitched dst,
                             const int64_t dst_acc_origin[3], int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3],
                             int64_t src_zsize, sb_pitched aux, int nbox, const int64_t *lo, const int64_t *hi) {
  const std::vector<sb_stencil_vterm> vt = stencil_vterms_of(terms, n);
  return transfer_oplan_build("sb_transfer_oplan_create", out, device, dtype, terms ? vt.data() : nullptr, n, dst, dst_acc_origin, dst_zsize,
                              src, src_acc_origin, src_zsize, aux, nullptr, 0, nbox, lo, hi);
}

int sb_transfer_voplan_create(sb_transfer_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                              const int64_t dst_acc_origin[3], int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3],
                              int64_t src_zsize, sb_pitched aux, const sb_pitched *coef, int ncoef, int nbox, const int64_t *lo,
                              const int64_t *hi) {
  return transfer_oplan_build("sb_transfer_voplan_create", out, device, dtype, terms, n, dst, dst_acc_origin, dst_zsize, src, src_acc_origin,
                              src_zsize, aux, coef, ncoef, nbox, lo, hi);
}

static int transfer_oplan_build(const char *fn, sb_transfer_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n,
                                sb_pitched dst, const int64_t dst_acc_origin[3], int64_t dst_zsize, sb_pitched src,
                                const int64_t src_acc_origin[3], int64_t src_zsize, sb_pitched aux, const sb_pitched *coef, int ncoef,
                                int nbox, const int64_t *lo, const int64_t *hi) {
  if (!out) return fail(SB_ERR_INVALID, "%s needs an output handle", fn);
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) return fail(SB_ERR_INVALID, "dtype %d must be SB_DTYPE_F32 or SB_DTYPE_F64", dtype);
  const int es = dtype == SB_DTYPE_F32 ? 4 : 8;
  int rc = stencil_terms_ok(terms, n);
  if (rc != SB_OK) return rc;
  if (ncoef < 0 || ncoef > SB_STENCIL_MAX_COEFS) return fail(SB_ERR_INVALID, "ncoef %d: 0 to %d coefficient fields", ncoef, SB_STENCIL_MAX_COEFS);
  if (ncoef > 0 && !coef) return fail(SB_ERR_INVALID, "ncoef %d, but the coefficient array is NULL", ncoef);
  bool aux_term = false, used[SB_STENCIL_MAX_COEFS] = {};
  for (int t = 0; t < n; ++t) {
    aux_term = aux_term || terms[t].source == 1;
    for (int a = 0; a < 3; ++a)
      if (terms[t].offset[a] < -1 || terms[t].offset[a] > 1)
        return fail(SB_ERR_INVALID, "term %d: offset (%d, %d, %d) reaches beyond 1 cell, the fused restriction's limit", t,
                    int(terms[t].offset[0]), int(terms[t].offset[1]), int(terms[t].offset[2]));
    const int k = terms[t].coef;
    if (k >= ncoef) return fail(SB_ERR_INVALID, "term %d names coefficient field %d, but ncoef is %d", t, k, ncoef);
    if (k >= 0 && !coef[k].ptr) return fail(SB_ERR_INVALID, "coefficient field %d is NULL", k);
    if (k >= 0) used[k] = true;
  }
  if (aux_term && !aux.ptr) return fail(SB_ERR_INVALID, "a term reads aux, but aux is NULL");
  if (!dst.ptr || !src.ptr) return fail(SB_ERR_INVALID, "dst and src must not be NULL");
  if (dst.ptr == src.ptr) return fail(SB_ERR_INVALID, "dst must not be src");
  if (aux_term && dst.ptr == aux.ptr) return fail(SB_ERR_INVALID, "dst must not be aux");
  for (int k = 0; k < ncoef; ++k)
    if (used[k] && coef[k].ptr == dst.ptr) return fail(SB_ERR_INVALID, "coefficient field %d is dst (coefficients are read only)", k);
  if (!dst_acc_origin || !src_acc_origin) return fail(SB_ERR_INVALID, "%s needs both acc_origins", fn);
  if (nbox < 0 || (nbox > 0 && (!lo || !hi))) return fail(SB_ERR_INVALID, "nbox %d boxes need lo and hi arrays", nbox);
  if (dst_zsize < 1 || src_zsize < 1) return fail(SB_ERR_INVALID, "dst_zsize and src_zsize must be >= 1");
  rc = stencil_buffers_ok({&dst}, {"dst"}, dst, "dst", es);
  if (rc == SB_OK) rc = stencil_buffers_ok({&src}, {"src"}, src, "src", es);
  if (rc == SB_OK && aux_term) rc = stencil_buffers_ok({&aux}, {"aux"}, src, "src", es);
  for (int k = 0; k < ncoef && rc == SB_OK; ++k)
    if (used[k]) rc = stencil_buffers_ok({&coef[k]}, {"coefficient field " + std::to_string(k)}, src, "src", es);
  if (rc != SB_OK) return rc;
  int nf = 0;
  for (int k = 0; k < ncoef; ++k) nf += used[k] ? 1 : 0;
  const int64_t dsize[3] = {dst.pitch / es, dst.ysize, dst_zsize}, ssize[3] = {src.pitch / es, src.ysize, src_zsize};
  const int zero[3] = {0, 0, 0}, one[3] = {1, 1, 1};
  // the fine cell 2 * (global lo) of a coarse box at l on axis a (dst allocation coordinates), in src allocation coordinates
  auto fine_lo = [&](int64_t l, int a) { return 2 * (l + dst_acc_origin[a]) - src_acc_origin[a]; };
  PlanBoxes B;
  rc = plan_boxes(nbox, lo, hi, dst_acc_origin, 4, [&](int b, const int64_t l[3], const int64_t e[3]) {
    const int64_t fl[3] = {fine_lo(l[0], 0), fine_lo(l[1], 1), fine_lo(l[2], 2)}, fe[3] = {2 * e[0], 2 * e[1], 2 * e[2]};
    int rc = stencil_box_reads_ok(b, l, e, zero, zero, dsize, "dst is written at");
    if (rc == SB_OK) rc = stencil_box_reads_ok(b, fl, fe, one, one, ssize, "the fused restriction reads fine");
    return rc;
  }, B);
  if (rc != SB_OK) return rc;

  sb::RopCommon com{};
  com.dst = static_cast<char *>(dst.ptr);
  com.src = static_cast<const char *>(src.ptr);
  com.aux = aux_term ? static_cast<const char *>(aux.ptr) : nullptr;
  com.dpitch = dst.pitch;
  com.dslice = dst.pitch * dst.ysize;
  com.spitch = src.pitch;
  com.sslice = src.pitch * src.ysize;
  com.n = n;
  for (int t = 0; t < n; ++t) {
    com.source[t] = (signed char)terms[t].source;
    for (int a = 0; a < 3; ++a) com.off[t][a] = (signed char)terms[t].offset[a];
    com.w[t] = terms[t].weight;
    com.wf[t] = float(terms[t].weight); // round to nearest
  }
  std::unique_ptr<sb_transfer_plan> p(new sb_transfer_plan());
  p->device = device;
  p->bytes = B.cells * es * (8 * ((aux_term ? 2 : 1) + nf) + 1);
  if (B.cells == 0) {
    *out = p.release();
    return SB_OK;
  }
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess)
    return fail(SB_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(cudaGetLastError()));
  // the launches take the coefficient parameters only with coefficient terms (nf > 0): the plain kernels their base
  if (!B.thick.empty()) {
    const int per_sm = sb::rop_tile_ctas_per_sm(es, nf > 0);
    if (per_sm <= 0) return fail(SB_ERR_CUDA, "the fused restriction's tile kernel cannot be configured: %s", cudaGetErrorString(cudaGetLastError()));
    for (const PlanBox &b : B.thick) {
      sb::RopVTileParams tp{};
      tp.c = com;
      for (int a = 0; a < 3; ++a) {
        tp.lo[a] = b.lo[a];
        tp.ext[a] = b.ext[a];
        tp.flo[a] = int(fine_lo(b.lo[a], a));
        tp.rlo[a] = tp.flo[a] - 1;
        tp.rhi[a] = tp.flo[a] + 2 * b.ext[a] + 1;
      }
      for (int c = 0; c < 3; ++c)
        for (int t = 0; t < n; ++t) {
          const int32_t *o = terms[t].offset;
          tp.toff[c][t] = ((c + o[2] + 3) % 3) * sb::kRopPlane + o[1] * sb::kRopSW + o[0];
        }
      // each chunk reloads 2 fine planes
      int grid = 0;
      if ((rc = tile_grid(tp, tp.ext, sb::kRestrictX, sb::kRestrictY, sms, per_sm, 4, "fused restriction's tile kernel", grid)) != SB_OK) return rc;
      for (int k = 0; k < ncoef; ++k) tp.coef[k] = static_cast<const char *>(coef[k].ptr);
      for (int t = 0; t < n; ++t) {
        const int32_t *c = terms[t].coef_offset;
        tp.cfield[t] = (signed char)terms[t].coef;
        tp.cgoff[t] = (long long)c[2] * com.sslice + (long long)c[1] * com.spitch + (long long)c[0] * es;
      }
      if (nf == 0)
        p->launches.push_back([base = sb::RopTileParams(tp), es, grid](cudaStream_t s) { return sb::launch_rop_tile(base, es, grid, s); });
      else
        p->launches.push_back([tp, es, grid](cudaStream_t s) { return sb::launch_rop_vtile(tp, es, grid, s); });
    }
  }
  sb::RopVCellParams cp{};
  cp.c = com;
  for (int k = 0; k < ncoef; ++k) cp.coef[k] = static_cast<const char *>(coef[k].ptr);
  for (int t = 0; t < n; ++t) {
    cp.cfield[t] = (signed char)terms[t].coef;
    for (int a = 0; a < 3; ++a) cp.coff[t][a] = (signed char)terms[t].coef_offset[a];
  }
  cell_groups(B.thin, cp, &sb::RopVCellParams::n, sms, [&](sb::RopVCellParams &g, int grid) {
    for (int m = 0; m < g.n; ++m)
      for (int a = 0; a < 3; ++a) g.flo[m][a] = int(fine_lo(g.lo[m][a], a));
    if (nf == 0)
      p->launches.push_back([base = sb::RopCellParams(g), es, grid](cudaStream_t s) { return sb::launch_rop_cells(base, es, grid, s); });
    else
      p->launches.push_back([g, es, grid](cudaStream_t s) { return sb::launch_rop_vcells(g, es, grid, s); });
  });
  *out = p.release();
  return SB_OK;
}

int sb_transfer_plan_launch(sb_transfer_plan *p, void *stream) { return run_launches(p, stream); }

int64_t sb_transfer_plan_bytes(const sb_transfer_plan *p) { return p ? p->bytes : 0; }

int sb_transfer_plan_destroy(sb_transfer_plan *p) {
  delete p;
  return SB_OK;
}

// ----------------------------------------------------------------------------------------- device plumbing
int sb_device_count(int *count) {
  cudaError_t e = cudaGetDeviceCount(count);
  if (e != cudaSuccess) {
    *count = 0;
    cudaGetLastError();
    return fail(SB_ERR_NOGPU, "cudaGetDeviceCount: %s", cudaGetErrorString(e));
  }
  return SB_OK;
}

int sb_malloc(void **ptr, size_t bytes, int device) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaMalloc(ptr, bytes));
  return SB_OK;
}

int sb_free(void *ptr, int device) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaFree(ptr));
  return SB_OK;
}

int sb_memset(void *ptr, int value, size_t bytes, int device, void *stream) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaMemsetAsync(ptr, value, bytes, static_cast<cudaStream_t>(stream)));
  return SB_OK;
}

int sb_memcpy(void *dst, const void *src, size_t bytes, int device, void *stream) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDefault, static_cast<cudaStream_t>(stream)));
  return SB_OK;
}

int sb_stream_sync(int device, void *stream) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  return SB_OK;
}

int sb_device_sync(int device) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaDeviceSynchronize());
  return SB_OK;
}

int sb_enable_peer(int src_device, int dst_device, int *ok) {
  *ok = 0;
  if (src_device == dst_device) {
    *ok = 1;
    return SB_OK;
  }
  int can = 0;
  SB_CUDA(cudaDeviceCanAccessPeer(&can, src_device, dst_device));
  if (!can) return SB_OK;
  DeviceGuard guard(src_device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", src_device);
  cudaError_t e = cudaDeviceEnablePeerAccess(dst_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) {
    cudaGetLastError();
    e = cudaSuccess;
  }
  SB_CUDA(e);
  *ok = 1;
  return SB_OK;
}

int sb_ipc_export(void *ptr, void *handle64) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  SB_CUDA(cudaIpcGetMemHandle(&h, ptr));
  std::memcpy(handle64, &h, sizeof(h));
  return SB_OK;
}

int sb_ipc_import(const void *handle64, int device, void **ptr) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle64, sizeof(h));
  SB_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return SB_OK;
}

int sb_ipc_close(void *ptr, int device) {
  DeviceGuard guard(device);
  if (!guard.ok) return fail(SB_ERR_NOGPU, "cannot select CUDA device %d", device);
  SB_CUDA(cudaIpcCloseMemHandle(ptr));
  return SB_OK;
}

} // extern "C"
