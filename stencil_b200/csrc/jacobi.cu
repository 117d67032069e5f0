// 7-point jacobi kernels for sm_90a (see jacobi.cuh).
//
// jacobi_march_kernel: register-blocked z-march.  A warp owns a strip of 32*VX cells in x and RY
// rows in y; each lane keeps the z-1 / z / z+1 values of its VX*RY columns in registers, so every
// cell of the subdomain is fetched from HBM exactly once (as the z+1 "centre" of its own column)
// with 16-byte vector loads.  x-neighbours come from the adjacent lane by warp shuffle (lanes 0
// and 31 fetch one scalar), y-neighbours inside the RY rows from registers and across warps from
// L1 (the neighbouring warp loaded that row one step earlier).  Eight warps are stacked in y, the
// z axis is cut into chunks so that the grid has several waves on the GPU's SMs, and an optional
// prefetch.global.L2 runs a few planes ahead of the march to deepen the memory pipeline without
// spending registers.  Algorithmic traffic: one read + one write per cell (2*sizeof(T) B/cell).
//
// Numerics: sum order ((((((0+px)+mx)+py)+my)+pz)+mz) as in bin/jacobi3d.cu:66-77, then an exact
// IEEE division by 6 done as q = v*c; r = fma(-6,q,v); q' = fma(r,c,q) with c = RN(1/6)
// (Markstein's correction: q' is the correctly rounded quotient), so results are bit-identical
// to the CPU oracle's `v / 6` in both FP32 and FP64.
#include "jacobi.cuh"

#include <map>
#include <mutex>
#include <utility>

namespace sb {
namespace {

template <typename T> struct Num;
template <> struct Num<float> {
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float div6(float v) {
    const float c = 1.0f / 6.0f;
    const float q = __fmul_rn(v, c);
    const float r = __fmaf_rn(-6.0f, q, v);
    return __fmaf_rn(r, c, q);
  }
};
template <> struct Num<double> {
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double div6(double v) {
    const double c = 1.0 / 6.0;
    const double q = __dmul_rn(v, c);
    const double r = __fma_rn(-6.0, q, v);
    return __fma_rn(r, c, q);
  }
};

template <typename T, int N> struct alignas(sizeof(T) * N) Vec { T v[N]; };

// dist() of bin/jacobi3d.cu:31-33: int64(__fsqrt_rn(float(d2)))
__device__ __forceinline__ bool in_sphere(int d2, int rad) { return (int)__fsqrt_rn((float)d2) <= rad; }

template <typename T> __device__ __forceinline__ T stencil_value(T px, T mx, T py, T my, T pz, T mz) {
  T v = Num<T>::add(T(0), px);
  v = Num<T>::add(v, mx);
  v = Num<T>::add(v, py);
  v = Num<T>::add(v, my);
  v = Num<T>::add(v, pz);
  v = Num<T>::add(v, mz);
  return Num<T>::div6(v);
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// x-face cells of a boundary tile, parked while it marches (fused kernel): [side][warp = row][plane of the chunk]
__shared__ unsigned long long g_xstage[2 * 8 * 32];
template <typename T> __device__ __forceinline__ T *xstage_row(int side, int warp) { return reinterpret_cast<T *>(g_xstage) + (side * 8 + warp) * 32; }
// ... and the y-face row of a boundary tile (512 bytes per plane: 32 lanes x one 16-byte vector), all planes of the chunk
__shared__ uint4 g_ystage[32 * 32];
// ... and its z-face plane (8 rows x 512 bytes).  A tile on both z faces (a subdomain of one chunk) parks the -z plane.
__shared__ uint4 g_zstage[8 * 32];

// Register-blocked z-march (see the file header).  Everything that does not change along z is hoisted
// out of the loop -- clamped row offsets, store masks, the (y - cy)^2 term of the sphere test -- so a
// z-step is: RY centre loads for plane z+1, 2 halo-row loads and RY edge scalars for plane z, the
// shuffles, 9 FP64 ops per cell and RY stores.  The loop is unrolled by three with the roles of the
// three register planes rotating, so there are no register-to-register plane copies.
//
// SHIFT variant (RY = 1): when the row pitch is only half-vector aligned (FP32 rows of 514 floats =
// 2056 B are 8 mod 16) consecutive rows alternate between two 16-byte phases.  Each warp then
// starts its strip VX/2 cells earlier on the odd-phase rows, so the HBM-facing accesses (centre
// loads, stores) stay full 128-bit vectors on every row; only the two L1-resident neighbour rows
// (y-1, y+1), which have the opposite phase, are fetched as two half vectors.
//
// Boundary variants (RY = 1; the boundary CTAs of the fused kernel), MODE bits:
//   1 EDGE   the cells just outside the subdomain may come from somewhere else -- a periodic self-neighbour is read in place
//            from the opposite face of src (pointer set-up before the loop).  The loop itself is the plain one.
//   2 XPUSH  the x neighbour of the first / last column may come from a dense received array, and the tile's own x-face
//            cells are parked in shared memory as the march goes (one predicated STS per step).
//   4 YPUSH  the warp that owns a y-face row parks it in shared memory as well (one predicated STS.128 per step); stores
//            into the neighbour never sit between two steps of the march.
// z faces cost the loop nothing: the first plane of the bottom chunk and the last plane of the top chunk are computed by
// two steps taken out of the loop (the top one FIRST, from three planes loaded for it alone -- 2 planes in 32 read twice by
// 1 CTA in 16), which park their result for the neighbour as well, and which know about a periodic self-neighbour along
// z (the plane beyond the top is the bottom plane).
// The kernel is latency- and issue-bound at once (53 % issue utilisation with 8 warps per scheduler): every instruction
// added to the loop shows in the run time, so each boundary CTA runs the leanest variant that serves its faces.
template <typename T, int VX, int RY, bool SHIFT, int MODE>
__device__ __forceinline__ void march_body(const JacobiParams &p, const int bx, const int by, const int bz, const bool wait_barrier = false) {
  static_assert(!SHIFT || (RY == 1 && VX >= 2), "the phase-shifted variant handles one row per warp");
  static_assert(!MODE || RY == 1, "the boundary variants handle one row per warp");
  static_assert(MODE == 0 || (MODE & 1), "XPUSH / YPUSH imply EDGE");
  constexpr bool EDGE = (MODE & 1) != 0; // EDGE
  constexpr bool XP = (MODE & 2) != 0;
  constexpr bool YP = (MODE & 4) != 0;
  using V = Vec<T, VX>;
  constexpr int WY = 8; // warps stacked in y
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;

  const long long S = p.slice, P = p.pitch;
  const int y = p.lo[1] + (by * WY + warp) * RY;         // first row of this warp
  // phase of this row inside a 16-byte vector, in elements (0 unless SHIFT)
  const int shift = SHIFT ? (int)((((unsigned long long)y * (unsigned long long)P) & (sizeof(T) * VX - 1)) / sizeof(T)) : 0;
  const int x0w = p.x0a + bx * 32 * VX - shift; // first cell of this warp's strip (allocation index)
  const int x = x0w + lane * VX;                              // first cell of this lane
  const int z0 = p.lo[2] + bz * p.zchunk;
  const int z1 = min(z0 + p.zchunk, p.hi[2]);
  if (y >= p.hi[1] || x0w >= p.hi[0]) { // warp-uniform
    if (wait_barrier) __syncthreads();
    return;
  }

  // does this lane's vector lie inside the allocation row?
  // SHIFT: a vector may hang over either end of its row into the neighbouring row of the same allocation.  That is valid
  // memory for every vector that holds a compute cell or the ghost cell next to one (rows 1 .. ny of planes 0 .. nz+1 have a
  // row before and after them); lanes further out -- rows much shorter than a strip put them several rows beyond the last
  // row of the allocation -- read (and discard) an aligned vector inside the row instead.
  const bool xin = SHIFT ? (x + VX >= p.lo[0] && x <= p.hi[0]) : (x + VX <= p.raw[0]);
  const int xsafe = SHIFT ? (p.x0a - shift + VX) : (p.x0a >= 0 ? p.x0a : p.x0a + VX);
  const int xs = xin ? x : xsafe;
  const long long xoff = (long long)xs * (long long)sizeof(T);

  // row byte offsets inside a plane; rows beyond the allocation are clamped (their results are masked)
  auto yo = [&](int yy) { return (long long)clampi(yy, 0, p.raw[1] - 1) * P; };
  const char *__restrict__ src = p.src;
  const char *pc[RY]; // centre rows, plane z+1
  const char *ph[RY]; // edge scalar of each row, plane z
  char *pw[RY];       // output rows, plane z
  // A region that ends inside a strip: when the vector after the last compute cell would hang over the end of the row
  // (ghost width 1, the ghost cell is its first element), the next lane loads a stand-in vector instead (xin above), so the
  // lane holding the last cell loads the ghost cell as its edge scalar, like lane 31 at the end of a strip.
  const bool tail_lane = !SHIFT && lane != 31 && x + VX == p.hi[0] && x + 2 * VX > p.raw[0];
  const bool edge_lane = (lane == 0) || (lane == 31) || tail_lane;
  long long phstep = S; // per-plane advance of ph (XPUSH: a dense x-ghost array is z fastest)
  int hxv = lane == 0 ? x - 1 : x + VX;
  bool far = false; // this lane's edge scalar / patched element comes from the other end of the row
  if (EDGE && p.xwrap) { // periodic self-neighbour: the cell beyond a face is the first / last cell of the same row
    if (hxv == p.lo[0] - 1) hxv = p.hi[0] - 1, far = edge_lane;
    else if (hxv == p.hi[0]) hxv = p.lo[0], far = edge_lane;
  }
  const int hx = clampi(hxv, 0, p.raw[0] - 1);
#pragma unroll
  for (int j = 0; j < RY; ++j) {
    pc[j] = src + (long long)(z0 + 1) * S + yo(y + j) + xoff;
    ph[j] = src + (long long)z0 * S + yo(y + j) + (long long)hx * (long long)sizeof(T);
    if (XP) { // the x neighbour of the first / last compute cell may come from a dense received array [y][z]
      const int side = (lane == 0 && x == p.lo[0]) ? 0 : ((lane == 31 && x + VX == p.hi[0]) ? 1 : -1);
      if (side >= 0 && p.xghost_ptr[side]) {
        ph[j] = p.xghost_ptr[side] + (long long)(y + j) * p.xghost_pitch[side] + (long long)z0 * (long long)sizeof(T);
        phstep = (long long)sizeof(T);
      }
    }
    pw[j] = p.dst + (long long)z0 * S + (long long)(y + j) * P + (long long)x * (long long)sizeof(T);
  }
  int yu = y - 1, yd = y + RY;
  if (EDGE && p.ywrap) { // periodic self-neighbour: the row beyond a face is the opposite face row
    if (yu == p.lo[1] - 1) yu = p.hi[1] - 1;
    if (yd == p.hi[1]) yd = p.lo[1];
  }
  const char *pu = src + (long long)z0 * S + yo(yu) + xoff; // row above the strip, plane z
  const char *pd = src + (long long)z0 * S + yo(yd) + xoff; // row below the strip, plane z

  // SHIFT + periodic self-neighbour along x: on phase-shifted rows the ghost cell just outside a face sits INSIDE a lane's
  // vector (the strip starts VX / 2 cells early), where the edge lanes' scalar cannot replace it: that element is patched
  // with the cell of the opposite face.  A ghost cell only matters as the x neighbour of a compute cell, i.e. while its
  // vector is the CURRENT plane, so the scalar loaded beside plane z+1's vector is selected in one step later, when it has
  // long arrived.  (Selected into plane z+1 right away, the select made the warp wait for that plane before it had even
  // asked for the rows above and below: two memory latencies per step, the x-face tiles of FP32 512^3 ran at half speed.)
  // Every lane loads a scalar (its own first element where nothing is patched): no divergent branch around a load.
  int wrap_i = -1;
  const bool xpatch = EDGE && SHIFT && p.xwrap; // kernel-uniform
  const char *wrap_p = pc[0]; // the scalar of plane z+1
  if (xpatch) {
#pragma unroll
    for (int i = 0; i < VX; ++i) {
      const int xi = x + i;
      const int xw = xi == p.lo[0] - 1 ? p.hi[0] - 1 : (xi == p.hi[0] ? p.lo[0] : -1);
      if (xw >= 0) wrap_i = i, wrap_p = src + (long long)(z0 + 1) * S + yo(y) + (long long)xw * (long long)sizeof(T);
    }
  }
  T wA = T(0), wB = T(0), wC = T(0); // the scalar that belongs into each register plane's vector (loaded with it; no copies:
                                     // a copy right behind the load would make the warp wait for it)
  const long long zspan = (long long)(p.hi[2] - p.lo[2]) * S; // a periodic self-neighbour along z is this many bytes away

  // store masks
  bool row_ok[RY];
#pragma unroll
  for (int j = 0; j < RY; ++j) row_ok[j] = (y + j < p.hi[1]);
  const bool full = (x >= p.lo[0]) && (x + VX <= p.hi[0]);
  unsigned cell_ok = 0;
#pragma unroll
  for (int i = 0; i < VX; ++i)
    if (x + i >= p.lo[0] && x + i < p.hi[0]) cell_ok |= 1u << i;

  // sphere test pieces that are constant along z
  const int rr = (p.rad + 1) * (p.rad + 1);
  int dy2[RY];
#pragma unroll
  for (int j = 0; j < RY; ++j) {
    const int dyv = y + j + p.org[1] - p.cy;
    dy2[j] = dyv * dyv;
  }
  const int gx0 = x + p.org[0];

  // ---- What this warp contributes to the neighbours' halos (see jacobi_fused_kernel): parked in shared memory while it
  // marches, stored into the neighbour by finish_tile -- which derives its own indices, so nothing of it is live here.
  //  x faces: the lane holding the first / last cell of the row parks it every step (one predicated STS);
  //  y faces: the warp that owns the first / last row parks its vector every step (one predicated STS.128);
  //  z faces: the first plane of the bottom chunk and the last plane of the top chunk are parked by the two steps taken
  //           out of the loop (below).
  int xsi = -1;       // which element of this lane's vector is an x-face cell (-1: none; a lane never holds both faces: ex >= 16)
  T *xsp = nullptr;   // where that cell of the current plane is parked
  uint4 *ysp = nullptr; // YPUSH: where this lane's vector of the current plane is parked (null: not a y-face row)
  if (XP && row_ok[0]) {
#pragma unroll
    for (int i = 0; i < VX; ++i) {
      if (x + i == p.lo[0] && p.push_ptr[0]) xsi = i, xsp = xstage_row<T>(0, warp);
      if (x + i == p.hi[0] - 1 && p.push_ptr[1]) xsi = i, xsp = xstage_row<T>(1, warp);
    }
  }
  if (YP && sizeof(V) == 16 && row_ok[0]) {
    // (a tile on both y faces -- a subdomain of at most 8 rows -- parks the -y row; finish_tile copies the other one)
    if ((y == p.lo[1] && p.push_ptr[2]) || (y == p.hi[1] - 1 && p.push_ptr[3] && !(by == 0 && p.push_ptr[2]))) ysp = g_ystage + lane;
  }

  // boundary CTAs of the fused kernel: the flag poll issued before all this set-up must have completed before any load
  if (wait_barrier) __syncthreads();
  V A[RY], B[RY], C[RY];
  const int zlast = p.raw[2] - 1; // last plane that may be touched (prefetch guard)
  int z = z0;
  // XPUSH: the x neighbour of the first / last compute cell may come from a dense received array [y][z] (z fastest), which
  // is not part of the rows the march prefetches: a load per step put an L2 miss on every fourth step's critical path
  // (a quarter of the tiles sit on x faces).  The chunk's 256-byte line of this row is
  // pulled into L1 here, one plane per lane; the edge lane's loads then hit.
  if (XP) {
    const int gside = (x0w == p.lo[0] && p.xghost_ptr[0]) ? 0 : ((x0w + 32 * VX == p.hi[0] && p.xghost_ptr[1]) ? 1 : -1);
    if (gside >= 0 && lane < z1 - z0)
      asm volatile("prefetch.global.L1 [%0];" ::"l"(p.xghost_ptr[gside] + (long long)y * p.xghost_pitch[gside] + (long long)(z0 + lane) * (long long)sizeof(T)));
  }

  // one plane: load z+1, compute z from (z-1, z, z+1), store, advance every running pointer.  ZP (the two steps outside the
  // loop): also store the result into the z neighbours named by zmask (bit 0: -z, bit 1: +z).
  auto step = [&](auto zp_tag, const unsigned zmask, const V(&prev)[RY], const V(&cur)[RY], V(&nxt)[RY], const T &wcur, T &wnext) {
    constexpr bool ZP = decltype(zp_tag)::value;
    if (EDGE && SHIFT && wrap_i >= 0) wnext = *reinterpret_cast<const T *>(wrap_p); // (wrap_i >= 0 only with xpatch;
                                                                                   // testing xpatch too made ptxas spill in the FP32 x-face loop)
#pragma unroll
    for (int j = 0; j < RY; ++j) nxt[j] = *reinterpret_cast<const V *>(pc[j]);
    if (EDGE && SHIFT) wrap_p += S;
    if (p.prefetch > 0 && z + 1 + p.prefetch <= zlast) {
#pragma unroll
      for (int j = 0; j < RY; ++j) asm volatile("prefetch.global.L2 [%0];" ::"l"(pc[j] + (long long)p.prefetch * S));
      // cells read from the other end of the row are in nobody's prefetch stream here: without this every step of an
      // x-face warp waits for DRAM (FP32 512^3, one GPU: 0.290 -> ms per iteration)
      if (EDGE && far) asm volatile("prefetch.global.L2 [%0];" ::"l"(ph[0] + (long long)p.prefetch * S));
      if (EDGE && SHIFT && wrap_i >= 0) asm volatile("prefetch.global.L2 [%0];" ::"l"(wrap_p + (long long)(p.prefetch - 1) * S)); // (wrap_p is already one plane on)
    }
    V up, dn;
    if (SHIFT) { // the rows above / below have the other phase: two aligned half vectors each
      using H = Vec<T, (VX >= 2 ? VX / 2 : 1)>;
      const H u0 = reinterpret_cast<const H *>(pu)[0], u1 = reinterpret_cast<const H *>(pu)[1];
      const H d0 = reinterpret_cast<const H *>(pd)[0], d1 = reinterpret_cast<const H *>(pd)[1];
#pragma unroll
      for (int i = 0; i < VX / 2; ++i) {
        up.v[i] = u0.v[i];
        up.v[i + VX / 2] = u1.v[i];
        dn.v[i] = d0.v[i];
        dn.v[i + VX / 2] = d1.v[i];
      }
    } else {
      up = *reinterpret_cast<const V *>(pu);
      dn = *reinterpret_cast<const V *>(pd);
    }
    const int dzv = z + p.org[2] - p.cz;
    const int dz2 = dzv * dzv;
    T hh[RY];
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      hh[j] = T(0);
      if (edge_lane) hh[j] = *reinterpret_cast<const T *>(ph[j]);
    }
    V cc[RY]; // the current plane as the x direction sees it
#pragma unroll
    for (int j = 0; j < RY; ++j) cc[j] = cur[j];
    if (EDGE && SHIFT && xpatch) {
#pragma unroll
      for (int i = 0; i < VX; ++i) cc[0].v[i] = (wrap_i == i) ? wcur : cc[0].v[i];
    }
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      const T h = hh[j];
      T left = __shfl_up_sync(0xffffffffu, cc[j].v[VX - 1], 1);
      T right = __shfl_down_sync(0xffffffffu, cc[j].v[0], 1);
      if (lane == 0) left = h;
      if (lane == 31 || tail_lane) right = h;
      V out;
#pragma unroll
      for (int i = 0; i < VX; ++i) {
        const T px = (i < VX - 1) ? cc[j].v[i + 1 < VX ? i + 1 : i] : right;
        const T mx = (i > 0) ? cc[j].v[i > 0 ? i - 1 : 0] : left;
        const T py = (j < RY - 1) ? cur[j + 1 < RY ? j + 1 : j].v[i] : dn.v[i];
        const T my = (j > 0) ? cur[j > 0 ? j - 1 : 0].v[i] : up.v[i];
        out.v[i] = stencil_value<T>(px, mx, py, my, nxt[j].v[i], prev[j].v[i]);
      }
      const int dyz2 = dy2[j] + dz2;
      if (dyz2 < rr) { // rare: this row crosses a sphere (exact pre-filter, see oracle/stencil_oracle.c)
#pragma unroll
        for (int i = 0; i < VX; ++i) {
          const int dh = (gx0 + i - p.hot_x) * (gx0 + i - p.hot_x) + dyz2;
          const int dc = (gx0 + i - p.cold_x) * (gx0 + i - p.cold_x) + dyz2;
          if (in_sphere(dh, p.rad)) {
            out.v[i] = T(1);
          } else if (in_sphere(dc, p.rad)) {
            out.v[i] = T(0);
          }
        }
      }
      if (row_ok[j]) {
        if (full) {
          *reinterpret_cast<V *>(pw[j]) = out;
        } else {
#pragma unroll
          for (int i = 0; i < VX; ++i)
            if (cell_ok & (1u << i)) reinterpret_cast<T *>(pw[j])[i] = out.v[i];
        }
      }
      if (XP && xsi >= 0) {
        T v = out.v[0];
#pragma unroll
        for (int i = 1; i < VX; ++i)
          if (xsi == i) v = out.v[i];
        *xsp++ = v;
      }
      if (YP && ysp) {
        *reinterpret_cast<V *>(ysp) = out;
        ysp += 32;
      }
      if (ZP && sizeof(V) == 16 && zmask) *reinterpret_cast<V *>(g_zstage + warp * 32 + lane) = out; // leaves in finish_tile
      pc[j] += S;
      ph[j] += XP ? phstep : S;
      pw[j] += S;
    }
    pu += S;
    pd += S;
    ++z;
  };
  using NoZ = std::integral_constant<bool, false>;
  using WithZ = std::integral_constant<bool, true>;

  // the last plane of the top chunk first (EDGE): its +z neighbour plane may be the bottom plane (zwrap), and its result
  // may have to go to the +z neighbour -- neither is the loop's business.  Every running pointer moves up, the step runs,
  // and they all come back.
  int zend = z1;
  if (EDGE && z1 == p.hi[2] && (p.zwrap || p.push_ptr[5])) {
    const int up = z1 - 1 - z0;
    const long long d = (long long)up * S;
#pragma unroll
    for (int j = 0; j < RY; ++j) pc[j] += d, ph[j] += (long long)up * (XP ? phstep : S), pw[j] += d;
    pu += d, pd += d, z += up;
    if (XP) xsp += up;
    if (YP && ysp) ysp += 32 * up;
    if (SHIFT) wrap_p += d;
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      const char *pa = pc[j] - 2 * S;
      const bool below = p.zwrap && up == 0 && z0 == p.lo[2]; // a one-plane subdomain chunk: its own plane, twice
      if (below) pa += zspan;
      A[j] = *reinterpret_cast<const V *>(pa);
      B[j] = *reinterpret_cast<const V *>(pc[j] - S);
      if (p.zwrap) pc[j] -= zspan;
    }
    if (xpatch && wrap_i >= 0) wB = *reinterpret_cast<const T *>(wrap_p - S);
    if (SHIFT && p.zwrap) wrap_p -= zspan;
    const unsigned zmask = (p.push_ptr[5] && !(z0 == p.lo[2] && p.push_ptr[4])) ? 2u : 0u; // (on both z faces: finish_tile copies)
    step(WithZ{}, zmask, A, B, C, wB, wC);
    const long long back = (long long)(up + 1) * S;
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      pc[j] -= back, ph[j] -= (long long)(up + 1) * (XP ? phstep : S), pw[j] -= back;
      if (p.zwrap) pc[j] += zspan;
    }
    pu -= back, pd -= back, z -= up + 1;
    if (XP) xsp -= up + 1;
    if (YP && ysp) ysp -= 32 * (up + 1);
    if (SHIFT) {
      wrap_p -= back;
      if (p.zwrap) wrap_p += zspan;
    }
    zend = z1 - 1;
  }
  if (z < zend) {
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      // plane z0-1 (a periodic self-neighbour along z: the ghost plane below the subdomain is its own top plane, read in place)
      const char *pa = pc[j] - 2 * S;
      const bool below = EDGE && p.zwrap && z0 == p.lo[2];
      if (below) pa += zspan;
      A[j] = *reinterpret_cast<const V *>(pa);
      B[j] = *reinterpret_cast<const V *>(pc[j] - S); // plane z0
    }
    if (xpatch && wrap_i >= 0) wB = *reinterpret_cast<const T *>(wrap_p - S);
    if (EDGE && z0 == p.lo[2] && p.push_ptr[4] && !(z1 == p.hi[2] && p.push_ptr[5])) { // the first plane of the bottom chunk is parked for the -z neighbour
      step(WithZ{}, 1u, A, B, C, wB, wC);
#pragma unroll
      for (int j = 0; j < RY; ++j) A[j] = B[j], B[j] = C[j];
      wB = wC;
    }
  }
  while (z < zend) {
    step(NoZ{}, 0u, A, B, C, wB, wC);
    if (z >= zend) break;
    step(NoZ{}, 0u, B, C, A, wC, wA);
    if (z >= zend) break;
    step(NoZ{}, 0u, C, A, B, wA, wB);
  }
}

// Rows per warp and minimum CTAs per SM of the march kernel: fewer rows -> fewer registers -> more warps in flight.
constexpr int kMarchRows = 1;
constexpr int kMarchCtasPerSm = 4;

template <typename T, int VX, bool SHIFT>
__global__ void __launch_bounds__(256, kMarchCtasPerSm) jacobi_march_kernel(const __grid_constant__ JacobiParams p, int tiles_x, int tiles_y) {
  int b = blockIdx.x;
  const int bx = b % tiles_x;
  b /= tiles_x;
  march_body<T, VX, kMarchRows, SHIFT, 0>(p, bx, b % tiles_y, b / tiles_y);
}

// The tail column of phase-shifted rows (fused kernel).  FP32 rows of 514 floats alternate between two 16-byte phases, so
// 512 compute cells starting at cell 1 touch 129 aligned vectors of every row: four strips of 32 lanes and one vector
// more, with 1 or 3 compute cells in it.  As a fifth strip that vector costs a whole warp per row and step (a fifth of all
// warps of the launch, and two more strips of every row count as x-face tiles).  Here it is a tile of its own kind: one
// THREAD per row, 256 rows per CTA, marching the same z chunk with the planes z-1 / z / z+1 of its vector in registers,
// the neighbours in x and y as scalar loads (L2: the main strips fetch the same sectors).  It reads periodic
// self-neighbours in place and stores its cells of the y / z faces into the neighbours itself, step by step (a handful
// of stores per tile).  Not used when the +x face must be pushed (the launcher then keeps the fifth strip).
template <typename T, int VX>
__device__ __forceinline__ void march_column(const JacobiParams &p, const int xcol, const int cy, const int bz, const bool wait_barrier) {
  using V = Vec<T, VX>;
  const long long S = p.slice, P = p.pitch, es = (long long)sizeof(T);
  const int y = p.lo[1] + cy * 256 + (int)threadIdx.x;
  const int z0 = p.lo[2] + bz * p.zchunk;
  const int z1 = min(z0 + p.zchunk, p.hi[2]);
  if (wait_barrier) __syncthreads();
  if (y >= p.hi[1]) return;
  const int shift = (int)((((unsigned long long)y * (unsigned long long)P) & (sizeof(T) * VX - 1)) / sizeof(T));
  const int xv = xcol - shift;              // first cell of this row's tail vector (16-byte aligned; >= lo: there are main strips)
  const int n = min(p.hi[0] - xv, VX);      // compute cells in it (1 .. VX)
  int yu = y - 1, yd = y + 1;
  if (p.ywrap) {
    if (yu == p.lo[1] - 1) yu = p.hi[1] - 1;
    if (yd == p.hi[1]) yd = p.lo[1];
  }
  const int xr = p.xwrap ? p.lo[0] : p.hi[0]; // the cell beyond the +x face: the ghost cell, or this row's first cell
  const char *row = p.src + (long long)y * P, *rowu = p.src + (long long)yu * P, *rowd = p.src + (long long)yd * P;
  char *orow = p.dst + (long long)y * P;
  auto plane = [&](int zz) { // byte offset of plane zz, a periodic self-neighbour along z read in place
    if (p.zwrap) {
      if (zz == p.lo[2] - 1) zz = p.hi[2] - 1;
      else if (zz == p.hi[2]) zz = p.lo[2];
    }
    return (long long)zz * S;
  };
  const int rr = (p.rad + 1) * (p.rad + 1);
  const int dyv = y + p.org[1] - p.cy;
  const int dy2 = dyv * dyv;
  const int gx0 = xv + p.org[0];
  char *ypush = (y == p.lo[1] && p.push_ptr[2]) ? p.push_ptr[2] : nullptr; // this row is a y face of the subdomain
  long long yslice = p.push_slice[2];
  if (y == p.hi[1] - 1 && p.push_ptr[3] && !ypush) ypush = p.push_ptr[3], yslice = p.push_slice[3];
  char *ypush2 = (y == p.hi[1] - 1 && p.push_ptr[3] && ypush != p.push_ptr[3]) ? p.push_ptr[3] : nullptr; // a one-row subdomain: both

  V prev = *reinterpret_cast<const V *>(row + plane(z0 - 1) + (long long)xv * es);
  V cur = *reinterpret_cast<const V *>(row + (long long)z0 * S + (long long)xv * es);
  for (int z = z0; z < z1; ++z) {
    const V nxt = *reinterpret_cast<const V *>(row + plane(z + 1) + (long long)xv * es);
    const long long pz = (long long)z * S;
    const T left = *reinterpret_cast<const T *>(row + pz + (long long)(xv - 1) * es);
    const T right = *reinterpret_cast<const T *>(row + pz + (long long)xr * es);
    const int dzv = z + p.org[2] - p.cz;
    const int dyz2 = dy2 + dzv * dzv;
#pragma unroll
    for (int i = 0; i < VX; ++i) {
      if (i >= n) continue;
      const long long xo = (long long)(xv + i) * es;
      const T px = (i + 1 < VX && i + 1 < n) ? cur.v[i + 1 < VX ? i + 1 : i] : right;
      const T mx = (i > 0) ? cur.v[i > 0 ? i - 1 : 0] : left;
      const T py = *reinterpret_cast<const T *>(rowd + pz + xo);
      const T my = *reinterpret_cast<const T *>(rowu + pz + xo);
      T out = stencil_value<T>(px, mx, py, my, nxt.v[i], prev.v[i]);
      if (dyz2 < rr) {
        const int dh = (gx0 + i - p.hot_x) * (gx0 + i - p.hot_x) + dyz2;
        const int dc = (gx0 + i - p.cold_x) * (gx0 + i - p.cold_x) + dyz2;
        if (in_sphere(dh, p.rad)) {
          out = T(1);
        } else if (in_sphere(dc, p.rad)) {
          out = T(0);
        }
      }
      *reinterpret_cast<T *>(orow + pz + xo) = out;
      if (ypush) *reinterpret_cast<T *>(ypush + xo + (long long)z * yslice) = out;
      if (ypush2) *reinterpret_cast<T *>(ypush2 + xo + (long long)z * p.push_slice[3]) = out;
      if (z == p.lo[2] && p.push_ptr[4]) *reinterpret_cast<T *>(p.push_ptr[4] + (long long)y * p.push_pitch[4] + xo) = out;
      if (z == p.hi[2] - 1 && p.push_ptr[5]) *reinterpret_cast<T *>(p.push_ptr[5] + (long long)y * p.push_pitch[5] + xo) = out;
    }
    prev = cur;
    cur = nxt;
  }
}

// ---------------------------------------------------------------------------------------------------- fused iteration
// launch_jacobi_fused: the march over the WHOLE compute region of a subdomain, with the halo exchange of the next
// iteration and the ordering between ranks inside the kernel.
//
//  * Tiles are walked x fastest, then y, then z (measured: gathering the boundary tiles at the start or the end of the
//    grid costs 10 %, their 512-byte row segments lose the DRAM locality of whole rows).  Tiles that touch no face of
//    the subdomain (64 % at 512^3) run the plain loop; a boundary tile runs the leanest variant of the loop that serves
//    its faces (march_body MODE).  The kernel is latency- and issue-bound at once: every instruction added to a loop
//    shows in the run time.
//  * Pushing.  A boundary tile parks its face cells in shared memory while it marches -- the x column (one STS per step),
//    the y row (one STS.128 per step of the warp that owns it), the z plane (the two steps taken out of the loop) -- and
//    stores them into the neighbour when the march is over (finish_tile): x columns as one 256-byte line per row into a
//    dense array, y rows and z planes as 512-byte rows into the ghost cells.  Stores into the neighbour never sit between
//    two steps of the march (measured: a warp then runs at NVLink latency), nothing is counted, nothing crosses CTAs,
//    and no global load follows the march (tried: a copy pass over the finished tile costs microseconds per CTA under a
//    saturated memory system, and re-reading through a "last CTA of a group" costs an L1 invalidation per fence).
//  * A tile that pushes stays longer (8 to 128 NVLink stores, a few in flight at a time), so the walk is rotated on every
//    axis: it neither starts nor ends with such tiles (launch_fused).
//  * Ordering between ranks: ONE release per kernel.  The first CTA of iteration e writes e into every neighbour rank's
//    mailbox (st.release.sys; the kernel boundary has completed iteration e - 1, pushes and reads alike, and nothing of
//    this kernel is outstanding yet).  Before its first load a boundary tile polls the word of the neighbour across its
//    face (own memory, ld.acquire.sys by one thread): "the neighbour has started iteration e" says both "the ghost cells
//    I read are filled" and "the neighbour is done reading the ghost cells I am about to overwrite".  Inner tiles never
//    wait.  Tried first: one flag per boundary tile, released by the tile after its pushes -- the releasing warp waits for
//    an NVLink round trip and keeps its CTA's registers (4 x 256 x 64 = the whole file), so it was slower on 8 ranks;
//    what the per-kernel flag costs instead is the skew between the ranks' kernel starts, a few microseconds in the
//    first wave.  Every acquire also invalidates the SM's whole L1 (CCTL.IVALL): exactly one per face and tile.
constexpr int kMaxGroups = SB_FUSED_MAX_GROUPS;

template <typename T, int VX, bool SHIFT> __device__ __noinline__ void finish_tile(const JacobiParams &p, const FusedSync &s, int nx, int ny, int nz);

template <typename T, int VX, bool SHIFT, int EDGE>
__device__ __forceinline__ void fused_body(const JacobiParams &p, const FusedSync &s, int nx, int ny, int nz) {
  int b = blockIdx.x;
  // The first CTA of iteration e tells every neighbour rank "my iteration e - 1 is complete" (the kernel boundary has
  // made all its stores visible; nothing of this kernel is outstanding yet, so the release costs nothing).
  if (EDGE >= 2 && s.any_signal && b == 0 && threadIdx.x < 6 && s.signal_row[threadIdx.x])
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(s.signal_row[threadIdx.x]), "r"(s.signal_value) : "memory");
  if (SHIFT && s.col_cy) { // the first CTAs of the launch are the tail-column tiles (march_column)
    const int ncol = s.col_cy * nz;
    if (b < ncol) {
      const int cy = b % s.col_cy;
      int cz = b / s.col_cy + s.zrot;
      if (cz >= nz) cz -= nz;
      unsigned cf = 0; // faces of the subdomain this tile pushes to (x: none, see launch_fused)
      if (cy == 0 && p.push_ptr[2]) cf |= 4u;
      if (cy == s.col_cy - 1 && p.push_ptr[3]) cf |= 8u;
      if (cz == 0 && p.push_ptr[4]) cf |= 16u;
      if (cz == nz - 1 && p.push_ptr[5]) cf |= 32u;
      const bool cw = s.any_wait && cf;
      if (cw && threadIdx.x == 0) {
#pragma unroll
        for (int f = 2; f < 6; ++f)
          if ((cf >> f & 1u) && s.wait_row[f]) {
            uint32_t v;
            while (true) {
              asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(s.wait_row[f]) : "memory");
              if ((int32_t)(v - s.wait_value) >= 0) break;
              __nanosleep(100);
            }
          }
      }
      march_column<T, VX>(p, s.col_x, cy, cz, cw);
      return;
    }
    b -= ncol;
  }
  int bx = b % nx + s.xrot;
  b /= nx;
  int by = b % ny + s.yrot;
  int bz = b / ny + s.zrot;
  if (bx >= nx) bx -= nx;
  if (by >= ny) by -= ny;
  if (bz >= nz) bz -= nz;
  // the faces this CTA's cells lie on (phase-shifted rows end one strip later than the others, so with SHIFT the last TWO
  // strips along x may hold cells of the +x face)
  const int nxhi = SHIFT ? (s.col_cy ? 0 : min(nx, 2)) : 1; // (with tail-column tiles no strip holds a cell of the +x face)
  unsigned touch = 0;
  if (bx == 0) touch |= 1u;
  if (bx >= nx - nxhi) touch |= 2u;
  if (by == 0) touch |= 4u;
  if (by == ny - 1) touch |= 8u;
  if (bz == 0) touch |= 16u;
  if (bz == nz - 1) touch |= 32u;
  if (!touch) { // CTAs that touch no face take the plain loop
    march_body<T, VX, 1, SHIFT, 0>(p, bx, by, bz);
    return;
  }
  unsigned faces = 0; // faces with a push
#pragma unroll
  for (int f = 0; f < 6; ++f)
    if ((touch >> f & 1u) && p.push_ptr[f]) faces |= 1u << f;
  // the leanest loop that serves this tile's faces (march_body): x pushes or dense x ghosts, y pushes, or neither
  const bool needx = EDGE >= 2 && (((touch & 1u) && (p.push_ptr[0] || p.xghost_ptr[0])) || ((touch & 2u) && (p.push_ptr[1] || p.xghost_ptr[1])));
  const bool needy = EDGE >= 2 && (faces & 12u);

  // poll first, synchronise late: the barrier that publishes the poll to the other warps sits inside march_body, after its
  // address set-up and right before its first load
  const bool waits = s.any_wait && faces;
  if (waits && threadIdx.x == 0) {
    const uint32_t want = s.wait_value;
    // ld.acquire.sys = LDG.STRONG.SYS + CCTL.IVALL (the SM's L1 is dropped, so that ghost cells fetched before the
    // neighbour wrote them cannot be served from it).  Alternatives tried: relaxed loads + one fence.acq_rel.sys were slower
    // (MEMBAR.ALL.SYS at the start of every boundary CTA); three acquiring threads gained nothing over one.
    auto poll = [&](const uint32_t *slot) {
      uint32_t v;
      while (true) {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(slot) : "memory");
        if ((int32_t)(v - want) >= 0) break; // wrap-safe "v >= want"
        __nanosleep(100);
      }
    };
#pragma unroll
    for (int f = 0; f < 6; ++f)
      if ((faces >> f & 1u) && s.wait_row[f]) poll(s.wait_row[f]);
  }

  if (needy)
    march_body<T, VX, 1, SHIFT, 7>(p, bx, by, bz, waits);
  else if (needx)
    march_body<T, VX, 1, SHIFT, 3>(p, bx, by, bz, waits);
  else
    march_body<T, VX, 1, SHIFT, 1>(p, bx, by, bz, waits);
  if (EDGE >= 2) finish_tile<T, VX, SHIFT>(p, s, nx, ny, nz);
}

// After the march of a boundary CTA: ship what the loop could not, then tell the neighbours.  Everything is derived again
// from the block and thread indices (read through an opaque asm, so that the compiler keeps no tile coordinates, masks or
// face pointers alive across the marching loop -- with them the 64-register loop spilled and reloaded constants).
//  x faces: the column parked in shared memory, one plane per lane: a 256-byte line of the dense array per row and chunk.
//  (z faces went out from the registers of the two steps taken out of the loop, see march_body.)
//  y faces the loop could not serve (y_store_in_loop): copied from this lane's own stores, plane by plane.
//  Signalling: only warp 0 stays -- the others arrive at a named barrier and exit (a CTA's registers return to the SM when
//  its LAST warp exits, and the release below waits for an NVLink round trip).
template <typename T, int VX, bool SHIFT> __device__ __noinline__ void finish_tile(const JacobiParams &p, const FusedSync &s, int nx, int ny, int nz) {
  using V = Vec<T, VX>;
  int b, tid;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
  asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
  if (SHIFT && s.col_cy) b -= s.col_cy * nz; // (tail-column tiles never come here)
  int bx = b % nx + s.xrot;
  b /= nx;
  int by = b % ny + s.yrot;
  int bz = b / ny + s.zrot;
  if (bx >= nx) bx -= nx;
  if (by >= ny) by -= ny;
  if (bz >= nz) bz -= nz;
  const int lane = tid & 31, warp = tid >> 5;
  const long long S = p.slice, P = p.pitch, es = (long long)sizeof(T);
  const int y = p.lo[1] + by * 8 + warp;
  const int shift = SHIFT ? (int)((((unsigned long long)y * (unsigned long long)P) & (sizeof(T) * VX - 1)) / sizeof(T)) : 0;
  const int x0w = p.x0a + bx * 32 * VX - shift;
  const int x = x0w + lane * VX;
  const int z0 = p.lo[2] + bz * p.zchunk;
  const int z1 = min(z0 + p.zchunk, p.hi[2]);
  if (y < p.hi[1] && x0w < p.hi[0]) { // warp-uniform: this warp marched
    const bool full = (x >= p.lo[0]) && (x + VX <= p.hi[0]);
    unsigned cell_ok = 0;
    int xside = -1;
#pragma unroll
    for (int i = 0; i < VX; ++i) {
      if (x + i >= p.lo[0] && x + i < p.hi[0]) cell_ok |= 1u << i;
      if (x + i == p.lo[0] && p.push_ptr[0]) xside = 0;
      if (x + i == p.hi[0] - 1 && p.push_ptr[1]) xside = 1;
    }
#pragma unroll
    for (int side = 0; side < 2; ++side) {
      if (!__ballot_sync(0xffffffffu, xside == side)) continue; // warp-uniform
      __syncwarp();
      if (lane < z1 - z0) {
        char *t = p.xdense[side] ? p.push_ptr[side] + (long long)y * p.push_pitch[side] + (long long)(z0 + lane) * es
                                 : p.push_ptr[side] + (long long)(z0 + lane) * p.push_slice[side] + (long long)y * p.push_pitch[side];
        *reinterpret_cast<T *>(t) = xstage_row<T>(side, warp)[lane];
      }
    }
    // z faces: the plane this very thread parked; a tile on both z faces (or one marching narrow vectors) reads its own
    // stores back instead
    const bool zlo = z0 == p.lo[2] && p.push_ptr[4], zhi = z1 == p.hi[2] && p.push_ptr[5];
    if ((zlo || zhi) && cell_ok) {
      const bool parked = sizeof(V) == 16 && !(zlo && zhi);
#pragma unroll
      for (int side = 0; side < 2; ++side) {
        if (!(side == 0 ? zlo : zhi)) continue;
        char *t = p.push_ptr[4 + side] + (long long)y * p.push_pitch[4 + side] + (long long)x * es;
        V v;
        if (parked) {
          v = *reinterpret_cast<const V *>(g_zstage + warp * 32 + lane);
        } else {
          const char *r = p.dst + (long long)(side == 0 ? z0 : z1 - 1) * S + (long long)y * P + (long long)x * es;
#pragma unroll
          for (int i = 0; i < VX; ++i) v.v[i] = (cell_ok & (1u << i)) ? __ldcg(reinterpret_cast<const T *>(r) + i) : T(0);
        }
        if (full && ((unsigned long long)t % sizeof(V)) == 0) {
          *reinterpret_cast<V *>(t) = v;
        } else {
#pragma unroll
          for (int i = 0; i < VX; ++i)
            if (cell_ok & (1u << i)) reinterpret_cast<T *>(t)[i] = v.v[i];
        }
      }
    }
  }
  // y faces: the parked row leaves with every warp taking its share of the planes (stores into the neighbour are slow one
  // after the other, not side by side); vectors narrower than 16 bytes and the second row of a tile on both y faces are
  // copied from the tile's own stores instead
  {
    const int ylo = (by == 0 && p.push_ptr[2]) ? 1 : 0, yhi = (by == ny - 1 && p.push_ptr[3]) ? 1 : 0; // CTA-uniform
    if (ylo | yhi) {
      const int ydir = ylo ? 2 : 3;
      const int yrow = ylo ? p.lo[1] : p.hi[1] - 1;
      // the owner row's strip (its phase decides where the lanes' vectors start)
      const int rshift = SHIFT ? (int)((((unsigned long long)yrow * (unsigned long long)P) & (sizeof(T) * VX - 1)) / sizeof(T)) : 0;
      const int rx0 = p.x0a + bx * 32 * VX - rshift;
      const int rx = rx0 + lane * VX;
      unsigned rcell = 0;
#pragma unroll
      for (int i = 0; i < VX; ++i)
        if (rx + i >= p.lo[0] && rx + i < p.hi[0]) rcell |= 1u << i;
      const bool rfull = (rx >= p.lo[0]) && (rx + VX <= p.hi[0]);
      if (sizeof(V) == 16 && rx0 < p.hi[0]) {
        __syncthreads(); // every warp's march is over: the parked planes are complete
        for (int pl = warp; pl < z1 - z0; pl += 8) {
          const V v = *reinterpret_cast<const V *>(g_ystage + pl * 32 + lane);
          char *t = p.push_ptr[ydir] + (long long)rx * es + (long long)(z0 + pl) * p.push_slice[ydir];
          if (rfull && ((unsigned long long)t % sizeof(V)) == 0) {
            *reinterpret_cast<V *>(t) = v;
          } else {
#pragma unroll
            for (int i = 0; i < VX; ++i)
              if (rcell & (1u << i)) reinterpret_cast<T *>(t)[i] = v.v[i];
          }
        }
      }
      // the slow way: this warp's own row, read back plane by plane
      const bool slow_lo = sizeof(V) != 16 && ylo && y == p.lo[1];
      const bool slow_hi = yhi && y == p.hi[1] - 1 && (sizeof(V) != 16 || ylo);
      if ((slow_lo || slow_hi) && y < p.hi[1] && x0w < p.hi[0]) {
        unsigned cell_ok = 0;
#pragma unroll
        for (int i = 0; i < VX; ++i)
          if (x + i >= p.lo[0] && x + i < p.hi[0]) cell_ok |= 1u << i;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          if (k == 0 ? !slow_lo : !slow_hi) continue;
          const char *r = p.dst + (long long)y * P + (long long)x * es;
          char *t = p.push_ptr[2 + k] + (long long)x * es;
          for (int zz = z0; zz < z1; ++zz) {
#pragma unroll
            for (int i = 0; i < VX; ++i)
              if (cell_ok & (1u << i)) reinterpret_cast<T *>(t + (long long)zz * p.push_slice[2 + k])[i] = __ldcg(reinterpret_cast<const T *>(r + (long long)zz * S) + i);
          }
        }
      }
    }
  }
}

// EDGE 1: no face is pushed (every neighbour is this subdomain itself, read in place); 2: pushes, per-tile flags.
// 64 registers, 4 CTAs per SM.  (Tried: a 56-register build, so that a new CTA fits beside warps lingering in signal_tile
// -- it spills loop invariants and was 4 % slower at N = 2; one loop for all CTAs instead of the per-tile choice: the
// inner 64 % pay for the boundary code.)
template <typename T, int VX, bool SHIFT, int EDGE>
__global__ void __launch_bounds__(256, 4)
    jacobi_fused_kernel(const __grid_constant__ JacobiParams p, const __grid_constant__ FusedSync s, int nx, int ny, int nz) {
  fused_body<T, VX, SHIFT, EDGE>(p, s, nx, ny, nz);
}

// One thread per cell: thin regions (the +-x exterior slabs are 1..r cells wide in x).
// Threads run fastest along y there so a warp's accesses land in 32 different rows but the
// same few sectors per row; z-neighbours of consecutive planes hit L2.
template <typename T> __global__ void __launch_bounds__(256) jacobi_cell_kernel(const __grid_constant__ JacobiParams p) {
  const int ex = p.hi[0] - p.lo[0], ey = p.hi[1] - p.lo[1], ez = p.hi[2] - p.lo[2];
  const long long total = (long long)ex * ey * ez;
  const int rr = (p.rad + 1) * (p.rad + 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    // y fastest, then x, then z
    const int yy = (int)(i % ey);
    const long long t = i / ey;
    const int xx = (int)(t % ex);
    const int zz = (int)(t / ex);
    const int x = p.lo[0] + xx, y = p.lo[1] + yy, z = p.lo[2] + zz;
    const char *c = p.src + (long long)z * p.slice + (long long)y * p.pitch + (long long)x * (long long)sizeof(T);
    const T px = *reinterpret_cast<const T *>(c + sizeof(T));
    const T mx = *reinterpret_cast<const T *>(c - sizeof(T));
    const T py = *reinterpret_cast<const T *>(c + p.pitch);
    const T my = *reinterpret_cast<const T *>(c - p.pitch);
    const T pz = *reinterpret_cast<const T *>(c + p.slice);
    const T mz = *reinterpret_cast<const T *>(c - p.slice);
    T val = stencil_value<T>(px, mx, py, my, pz, mz);
    const int gx = x + p.org[0], gy = y + p.org[1], gz = z + p.org[2];
    const int dyz2 = (gy - p.cy) * (gy - p.cy) + (gz - p.cz) * (gz - p.cz);
    if (dyz2 < rr) {
      const int dh = (gx - p.hot_x) * (gx - p.hot_x) + dyz2;
      const int dc = (gx - p.cold_x) * (gx - p.cold_x) + dyz2;
      if (in_sphere(dh, p.rad)) {
        val = T(1);
      } else if (in_sphere(dc, p.rad)) {
        val = T(0);
      }
    }
    *reinterpret_cast<T *>(p.dst + (long long)z * p.slice + (long long)y * p.pitch + (long long)x * (long long)sizeof(T)) = val;
  }
}

// All exterior slabs of a subdomain in one launch (bin/jacobi3d.cu:324-342 issues up to six).  One thread
// per cell; inside a region threads run fastest along x when the slab is wide in x (coalesced rows)
// and along y when it is an x-face (1..r cells wide), so a warp always touches few sectors per row.
template <typename T>
__global__ void __launch_bounds__(256) jacobi_regions_kernel(const __grid_constant__ JacobiParams p, const __grid_constant__ JacobiRegions rg) {
  const long long total = rg.first[rg.n];
  const int rr = (p.rad + 1) * (p.rad + 1);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int k = 0;
    while (k + 1 < rg.n && i >= rg.first[k + 1]) ++k;
    const unsigned li = (unsigned)(i - rg.first[k]);
    const unsigned ex = rg.ext[k][0], ey = rg.ext[k][1];
    unsigned xx, yy, zz;
    if (ex >= 32) { // x fastest
      xx = li % ex;
      const unsigned t = li / ex;
      yy = t % ey;
      zz = t / ey;
    } else { // y fastest
      yy = li % ey;
      const unsigned t = li / ey;
      xx = t % ex;
      zz = t / ex;
    }
    const int x = rg.lo[k][0] + (int)xx, y = rg.lo[k][1] + (int)yy, z = rg.lo[k][2] + (int)zz;
    const long long off = (long long)z * p.slice + (long long)y * p.pitch + (long long)x * (long long)sizeof(T);
    const char *c = p.src + off;
    const T px = *reinterpret_cast<const T *>(c + sizeof(T));
    const T mx = *reinterpret_cast<const T *>(c - sizeof(T));
    const T py = *reinterpret_cast<const T *>(c + p.pitch);
    const T my = *reinterpret_cast<const T *>(c - p.pitch);
    const T pz = *reinterpret_cast<const T *>(c + p.slice);
    const T mz = *reinterpret_cast<const T *>(c - p.slice);
    T val = stencil_value<T>(px, mx, py, my, pz, mz);
    const int gx = x + p.org[0], gy = y + p.org[1], gz = z + p.org[2];
    const int dyz2 = (gy - p.cy) * (gy - p.cy) + (gz - p.cz) * (gz - p.cz);
    if (dyz2 < rr) {
      const int dh = (gx - p.hot_x) * (gx - p.hot_x) + dyz2;
      const int dc = (gx - p.cold_x) * (gx - p.cold_x) + dyz2;
      if (in_sphere(dh, p.rad)) {
        val = T(1);
      } else if (in_sphere(dc, p.rad)) {
        val = T(0);
      }
    }
    *reinterpret_cast<T *>(p.dst + off) = val;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) fill_kernel(char *dst, long long pitch, long long slice, int lx, int ly, int lz, int ex,
                                                   int ey, int ez, T value) {
  const long long total = (long long)ex * ey * ez;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % ex);
    const long long t = i / ex;
    const int yy = (int)(t % ey);
    const int zz = (int)(t / ey);
    reinterpret_cast<T *>(dst + (long long)(lz + zz) * slice + (long long)(ly + yy) * pitch)[lx + xx] = value;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) sqdiff_kernel(const char *a, const char *b, long long pitch, long long slice, int lx,
                                                     int ly, int lz, int ex, int ey, int ez, double *out) {
  const long long total = (long long)ex * ey * ez;
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int xx = (int)(i % ex);
    const long long t = i / ex;
    const int yy = (int)(t % ey);
    const int zz = (int)(t / ey);
    const long long off = (long long)(lz + zz) * slice + (long long)(ly + yy) * pitch;
    const double d = (double)reinterpret_cast<const T *>(a + off)[lx + xx] - (double)reinterpret_cast<const T *>(b + off)[lx + xx];
    acc += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  __shared__ double wsum[8];
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int w = 0; w < 8; ++w) s += wsum[w];
    atomicAdd(out, s);
  }
}

template <typename T, int VX, bool SHIFT> int launch_fused(const JacobiParams &p, FusedSync s, cudaStream_t stream) {
  const int x0a = p.x0a;
  int tiles_x = (p.hi[0] - x0a + (SHIFT ? VX / 2 : 0) + 32 * VX - 1) / (32 * VX);
  const int ny = p.hi[1] - p.lo[1], nz = p.hi[2] - p.lo[2];
  const int tiles_z = (nz + p.zchunk - 1) / p.zchunk;
  const int tiles_y = (ny + 7) / 8;
  if ((long long)tiles_z * tiles_y > kMaxGroups || (long long)tiles_z * tiles_x > kMaxGroups || (long long)tiles_y * tiles_x > kMaxGroups) return -2;
  // Phase-shifted rows whose last strip holds at most one vector of compute cells (FP32 512^3: 1 or 3 cells per row): that
  // vector becomes tail-column tiles (march_column), the strips before it the main grid.  Not when the +x face is pushed:
  // its cells would have to be parked by the column tiles.
  s.col_cy = s.col_x = 0;
  if (SHIFT && tiles_x >= 2 && !p.push_ptr[1]) {
    const int xcol = x0a + (tiles_x - 1) * 32 * VX; // first cell of the last strip on rows of phase 0
    if (p.hi[0] - (xcol - VX / 2) <= VX && xcol - VX / 2 >= p.lo[0]) {
      s.col_cy = (ny + 255) / 256;
      s.col_x = xcol;
      tiles_x -= 1;
    }
  }
  const long long blocks = (long long)tiles_x * tiles_y * tiles_z + (long long)s.col_cy * tiles_z;
  s.any_wait = s.any_signal = 0;
  for (int f = 0; f < 6; ++f) {
    if (s.wait_row[f]) s.any_wait = 1;
    if (s.signal_row[f]) s.any_signal = 1;
  }
  const bool dense_ghosts = p.xghost_ptr[0] || p.xghost_ptr[1];
  bool any_push = false;
  for (int f = 0; f < 6; ++f) any_push = any_push || p.push_ptr[f];
  // The walk over the tiles (x fastest, then y, then z) starts at a rotated origin: boundary tiles stay longer than inner
  // ones (pushes after the march, three extra plane loads in the top chunk), so the walk should not end with them, and z
  // starts in the middle, which keeps the z-face tiles out of the first wave, where every boundary tile waits for the
  // neighbour rank's kernel to start.  (Measured on and off, one and two ranks: within the run-to-run noise.)
  s.xrot = tiles_x - 1;
  s.yrot = tiles_y - 1;
  s.zrot = tiles_z / 2;
  if (!any_push && !dense_ghosts) // every face is a periodic self-neighbour read in place (one GPU)
    jacobi_fused_kernel<T, VX, SHIFT, 1><<<(unsigned)blocks, 256, 0, stream>>>(p, s, tiles_x, tiles_y, tiles_z);
  else
    jacobi_fused_kernel<T, VX, SHIFT, 2><<<(unsigned)blocks, 256, 0, stream>>>(p, s, tiles_x, tiles_y, tiles_z);
  return 1;
}

template <typename T, int VX, bool SHIFT> int launch_march(const JacobiParams &p, cudaStream_t stream) {
  const int x0a = p.x0a;
  // a shifted row starts VX/2 cells early, so the last tile must reach VX/2 cells further
  const int tiles_x = (p.hi[0] - x0a + (SHIFT ? VX / 2 : 0) + 32 * VX - 1) / (32 * VX);
  const int ny = p.hi[1] - p.lo[1], nz = p.hi[2] - p.lo[2];
  const int tiles_z = (nz + p.zchunk - 1) / p.zchunk;
  const int tiles_y = (ny + 8 * kMarchRows - 1) / (8 * kMarchRows);
  const long long blocks = (long long)tiles_x * tiles_y * tiles_z;
  jacobi_march_kernel<T, VX, SHIFT><<<(unsigned)blocks, 256, 0, stream>>>(p, tiles_x, tiles_y);
  return 1;
}

// regions narrower than this in x take the one-thread-per-cell kernel
constexpr int kThinX = 16;
// grid cap of the exterior-slab kernel
constexpr int kRegionsCtasPerSm = 32;

// SMs of the current device: the grid-stride kernels below cap their grids at a few CTAs per SM
long long sm_count() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 1;
}

} // namespace

int launch_jacobi_regions(const JacobiParams &p, const JacobiRegions &r, int dtype_size, cudaStream_t stream) {
  const long long total = r.first[r.n];
  if (r.n <= 0 || total <= 0) return 0;
  long long blocks = (total + 255) / 256;
  if (blocks > sm_count() * kRegionsCtasPerSm) blocks = sm_count() * kRegionsCtasPerSm;
  if (dtype_size == 4)
    jacobi_regions_kernel<float><<<(unsigned)blocks, 256, 0, stream>>>(p, r);
  else
    jacobi_regions_kernel<double><<<(unsigned)blocks, 256, 0, stream>>>(p, r);
  return 1;
}

static int pick_vectors(JacobiParams &p, int dtype_size, bool *shift);

int launch_jacobi(const JacobiParams &p_in, int dtype_size, cudaStream_t stream) {
  JacobiParams p = p_in;
  const int ex = p.hi[0] - p.lo[0], ey = p.hi[1] - p.lo[1], ez = p.hi[2] - p.lo[2];
  if (ex <= 0 || ey <= 0 || ez <= 0) return 0;

  if (ex < kThinX) {
    const long long total = (long long)ex * ey * ez;
    long long blocks = (total + 255) / 256;
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    if (dtype_size == 4)
      jacobi_cell_kernel<float><<<(unsigned)blocks, 256, 0, stream>>>(p);
    else
      jacobi_cell_kernel<double><<<(unsigned)blocks, 256, 0, stream>>>(p);
    return 1;
  }

  // z chunk: the caller's, else 32 planes
  if (p.zchunk <= 0) p.zchunk = 32;
  if (p.zchunk > ez) p.zchunk = ez;
  p.prefetch = 2;

  bool shift = false;
  const int vx = pick_vectors(p, dtype_size, &shift);
  if (dtype_size == 8) {
    if (vx == 2) return shift ? launch_march<double, 2, true>(p, stream) : launch_march<double, 2, false>(p, stream);
    return launch_march<double, 1, false>(p, stream);
  }
  if (vx == 4) return shift ? launch_march<float, 4, true>(p, stream) : launch_march<float, 4, false>(p, stream);
  if (vx == 2) return launch_march<float, 2, false>(p, stream);
  return launch_march<float, 1, false>(p, stream);
}

// Vector width and strip origin for a launch.  Rows whose pitch and slice are multiples of 16 bytes all have the phase
// of the allocation base: LocalDomain places the base so that the first COMPUTE cell is 16-byte aligned (the whole
// compute region of 512 cells is then exactly 8 strips of 32 lanes x 2 doubles); any other common phase of src and dst
// works as well.  Returns VX (1 = scalar fallback) and sets p.x0a; `shift` reports the alternating-phase case.
// Unshifted rows: a vector that holds compute cells but hangs over the end of its row is replaced by a stand-in load
// (march_body, xin), which would feed wrong values to those cells.  Such a region (e.g. 30 or 130 floats with one ghost
// cell behind a 12-byte lead) takes the scalar path, in launch_jacobi and launch_jacobi_fused alike.  A vector that holds
// only the ghost cell is handled in march_body (tail_lane), unless the lane before it is lane 0 of a strip (below).
static int pick_vectors(JacobiParams &p, int dtype_size, bool *shift) {
  const unsigned long long s = (unsigned long long)(uintptr_t)p.src, d = (unsigned long long)(uintptr_t)p.dst;
  const int full = 16 / dtype_size;
  *shift = false;
  auto origin = [&](int vx, unsigned phase) {
    const int xal = int(((16u - phase) & 15u) / unsigned(dtype_size)) % vx; // x (mod vx) of the aligned cells
    int r = (p.lo[0] - xal) % vx;
    if (r < 0) r += vx;
    p.x0a = p.lo[0] - r;
    return vx;
  };
  int vx;
  if (p.pitch % 16 == 0 && p.slice % 16 == 0 && (s & 15) == (d & 15) && (s & 15) % dtype_size == 0) {
    // with a non-zero phase the first vector may start before x = 0: still inside the (256-byte aligned) allocation,
    // whose first `phase` bytes are the lead pad
    vx = origin(full, unsigned(s & 15));
  } else if ((s & 15) == 0 && (d & 15) == 0 && p.slice % 16 == 0 && p.pitch % 16 == 8) {
    *shift = true;
    return origin(full, 0); // (shifted rows may hang over either end of a row: march_body xin)
  } else if (dtype_size == 4 && ((s | d | (unsigned long long)p.pitch | (unsigned long long)p.slice) % 8 == 0)) {
    vx = origin(2, 0);
  } else {
    return origin(1, 0);
  }
  const int last = p.x0a + ((p.hi[0] - 1 - p.x0a) / vx) * vx; // first cell of the last vector holding compute cells
  if (last + vx > p.raw[0]) return origin(1, 0);               // the overhang above
  // march_body's tail_lane takes the ghost cell as the right neighbour through the lane's one edge scalar; lane 0 of a strip
  // needs that scalar for its left neighbour (e.g. 66 or 130 doubles with one ghost cell behind an 8-byte lead)
  if (last + vx == p.hi[0] && last + 2 * vx > p.raw[0] && (last - p.x0a) / vx % 32 == 0) return origin(1, 0);
  return vx;
}

int launch_jacobi_fused(const JacobiParams &p_in, const FusedSync &sync, int dtype_size, cudaStream_t stream) {
  JacobiParams p = p_in;
  const int ex = p.hi[0] - p.lo[0], ey = p.hi[1] - p.lo[1], ez = p.hi[2] - p.lo[2];
  if (ex <= 0 || ey <= 0 || ez <= 0) return 0;
  // H100 80GB HBM3 (400 W), 512^3 FP64, one GPU, 1-plane L2 prefetch: 8-plane chunks take 0.78 ms per iteration, 16-plane
  // chunks 0.80 ms, 32 planes with a 2-plane prefetch 0.88 ms; deeper prefetch is slower (DESIGN.md section 2.2)
  p.prefetch = 1;
  bool shift = false;
  const int vx = pick_vectors(p, dtype_size, &shift);
  // z chunk (the x faces are staged at most 32 planes at a time): 8 planes by default, 16 or 32 where shorter chunks would
  // give a face more tiles than launch_fused's group limit (8: subdomains up to 512 cells in z at 512 cells in y; 16: up to
  // ~720 cells in y and z)
  const long long tiles_x = (p.hi[0] - p.x0a + (shift ? vx / 2 : 0) + 32 * vx - 1) / (32 * vx), tiles_y = (ey + 7) / 8;
  const long long across = tiles_x > tiles_y ? tiles_x : tiles_y;
  p.zchunk = ((ez + 7) / 8) * across <= kMaxGroups ? 8 : (((ez + 15) / 16) * across <= kMaxGroups ? 16 : 32);
  if (p.zchunk > ez) p.zchunk = ez;
  // x wrap (periodic self-neighbour read in place) works through the edge lanes' scalar load, so the first compute cell
  // must open lane 0 of the first strip and the last one must close lane 31 of the last strip; otherwise the ghost
  // column is read by a vector load or a shuffle and the x faces are pushed into the ghost cells like any other face
  // (phase-shifted FP32 rows: always possible -- a ghost cell inside a vector is patched, one beside lane 0 / 31 is the
  // edge scalar, see march_body)
  if (p.xwrap && !shift && !(p.x0a == p.lo[0] && (p.hi[0] - p.lo[0]) % (32 * vx) == 0)) p.xwrap = 0;
  if (p.xwrap) p.push_ptr[0] = p.push_ptr[1] = nullptr;
  if (p.xghost_ptr[0] || p.xghost_ptr[1]) {
    // a dense received x array is read by the edge lanes' scalar load: same layout conditions as the wrap
    if (shift || p.x0a != p.lo[0] || (p.hi[0] - p.lo[0]) % (32 * vx) != 0) return -1;
  }
  if (dtype_size == 8) {
    if (vx == 2) return shift ? launch_fused<double, 2, true>(p, sync, stream) : launch_fused<double, 2, false>(p, sync, stream);
    return launch_fused<double, 1, false>(p, sync, stream);
  }
  if (vx == 4) return shift ? launch_fused<float, 4, true>(p, sync, stream) : launch_fused<float, 4, false>(p, sync, stream);
  if (vx == 2) return launch_fused<float, 2, false>(p, sync, stream);
  return launch_fused<float, 1, false>(p, sync, stream);
}

int launch_fill(char *dst, long long pitch, long long slice, const int lo[3], const int hi[3], int dtype_size, double value,
                cudaStream_t stream) {
  const int ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
  if (ex <= 0 || ey <= 0 || ez <= 0) return 0;
  long long blocks = ((long long)ex * ey * ez + 255) / 256;
  if (blocks > sm_count() * 16) blocks = sm_count() * 16;
  if (dtype_size == 4)
    fill_kernel<float><<<(unsigned)blocks, 256, 0, stream>>>(dst, pitch, slice, lo[0], lo[1], lo[2], ex, ey, ez, (float)value);
  else
    fill_kernel<double><<<(unsigned)blocks, 256, 0, stream>>>(dst, pitch, slice, lo[0], lo[1], lo[2], ex, ey, ez, value);
  return 1;
}

int launch_sqdiff(const char *a, const char *b, long long pitch, long long slice, const int lo[3], const int hi[3],
                  int dtype_size, double *out_dev, cudaStream_t stream) {
  cudaMemsetAsync(out_dev, 0, sizeof(double), stream);
  const int ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
  if (ex <= 0 || ey <= 0 || ez <= 0) return 0;
  long long blocks = ((long long)ex * ey * ez + 255) / 256;
  if (blocks > sm_count() * 8) blocks = sm_count() * 8;
  if (dtype_size == 4)
    sqdiff_kernel<float><<<(unsigned)blocks, 256, 0, stream>>>(a, b, pitch, slice, lo[0], lo[1], lo[2], ex, ey, ez, out_dev);
  else
    sqdiff_kernel<double><<<(unsigned)blocks, 256, 0, stream>>>(a, b, pitch, slice, lo[0], lo[1], lo[2], ex, ey, ez, out_dev);
  return 1;
}

} // namespace sb
