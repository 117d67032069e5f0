// Linear stencil operators for sm_90a, constant and variable coefficients (see stencil_op.cuh and include/stencil_b200.h).
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
//
// Coefficient fields (HAS_COEF, a compile-time switch, so the plain instantiations are the code they were): a term may
// carry a field C read at p + c, |c_a| <= 1, and contributes (T(w) * C) * S.  The tile kernel keeps a ring of
// kOpCoefSlots halo'd planes per referenced field behind the src ring, filled one plane ahead by cp.async (no register
// staging), each field's window cut to its own reach; the term table carries each term's coefficient offset per slot.
// The cell kernel reads coefficients through __ldg at per-term byte offsets.
//
// Coloured application (COL, DESIGN.md section 2.9; again a compile-time switch): only the cells of colour c of the
// colouring m (2 or 8, from global coordinates) are written, and dst may be src.  In a tile row the cells of a colour
// alternate along x, so each lane computes one of them (cell 2 * lane + s); the cell kernel skips the other cells.
// src is read with plain loads, since the launch may write it.
//
// Diagonal relaxation (DIAG, DESIGN.md section 2.12; with COL, a compile-time switch): a cell of the colour gets
// u + omega ((f - A u) / d), f on aux and d the sum of the offset-0 terms' factors, formed in the same term loop.
#include "stencil_op.cuh"

#include <cstring>
#include <type_traits>

namespace sb {
namespace {

template <typename T> struct OpNum;
template <> struct OpNum<float> {
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float w(const OpCommon &c, int t) { return c.wf[t]; }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
};
template <> struct OpNum<double> {
  static __device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
  static __device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
  static __device__ __forceinline__ double w(const OpCommon &c, int t) { return c.w[t]; }
  static __device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
  static __device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }
};

// one element global -> shared, asynchronously (cp.async, sm_80+); completion by cp_async_wait_all
template <typename T> __device__ __forceinline__ void cp_async_elem(T *dst, const T *src) {
  const unsigned s = unsigned(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;\n" ::"r"(s), "l"(src), "n"(int(sizeof(T))) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

// A load of src.  The coloured kernels may run in place (dst == src), so they read src with plain loads: the
// non-coherent path may not see what this launch writes.  What they then race on is only what they never use.
template <bool COL, typename V> __device__ __forceinline__ V src_load(const V *a) {
  if constexpr (COL) return *a;
  else return __ldg(a);
}

template <bool HAS_COEF, bool COL, bool DIAG = false>
using OpTileParamsOf = typename std::conditional<
    DIAG, OpDTileParams,
    typename std::conditional<COL, OpCTileParams, typename std::conditional<HAS_COEF, OpVTileParams, OpTileParams>::type>::type>::type;

// COL: the coloured kernel.  Each warp row holds 32 cells of the colour at most (one colour of two alternates along x),
// so each lane computes one of them: the cell 2 * lane + s of the row, with s the row's colour phase.  DIAG (always with
// COL): the diagonal relaxation; under m = 1 each lane computes the cells 2 * lane and 2 * lane + 1.
template <typename T, int R, bool HAS_COEF, bool COL, bool DIAG = false>
__global__ void __launch_bounds__(kOpThreads, 2) op_tile_kernel(const __grid_constant__ OpTileParamsOf<HAS_COEF, COL, DIAG> p) {
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
            buf[i] = src_load<COL>(reinterpret_cast<const uint4 *>(ca));
          } else { // a chunk that would leave the allocation: its wanted elements one by one
            T e[V];
#pragma unroll
            for (int v = 0; v < V; ++v) {
              const char *a = ca + v * ES;
              e[v] = (a >= wa && a < wb) ? src_load<COL>(reinterpret_cast<const T *>(a)) : T(0);
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

  // coefficient rings: field f's kOpCoefSlots planes of (kOpTileX + 2) x (kOpTileY + 2) after the src ring; plane z of
  // its window (its own reach only) goes element by element through cp.async, so no registers hold it in flight
  constexpr int CSW = op_tile_sw(1), CP = op_tile_plane(1);
  T *const cring = ring + NS * P;
  auto coef_plane = [&](int f, int z) {
    if constexpr (HAS_COEF) {
      const int cxa = x0 - p.k.crm[f][0], w = xe + p.k.crp[f][0] - cxa;
      const int cya = y0 - p.k.crm[f][1], rows = ye + p.k.crp[f][1] - cya;
      const char *plane = p.k.coef[f] + (long long)z * p.c.slice;
      T *dst = cring + (f * kOpCoefSlots + ((z - z0 + 1) & (kOpCoefSlots - 1))) * CP + (1 - p.k.crm[f][1]) * CSW + (1 - p.k.crm[f][0]);
      for (int j = wy; j < rows; j += kOpThreads / 32) { // warps own rows, lanes columns
        const T *row = reinterpret_cast<const T *>(plane + (long long)(cya + j) * p.c.pitch) + cxa;
        for (int i = lane; i < w; i += 32) cp_async_elem(dst + j * CSW + i, row + i);
      }
    }
  };
  if constexpr (HAS_COEF) {
    if (z0 < z1)
      for (int f = 0; f < p.k.nf; ++f)
        for (int z = z0 - p.k.crm[f][2]; z <= z0 + p.k.crp[f][2]; ++z) coef_plane(f, z);
  }

  for (int z = z0 - p.rm[2]; z < z0 + p.rp[2]; ++z) {
    fetch(z);
    store(slot_of(z));
  }
  if (z0 < z1) fetch(z0 + p.rp[2]);

  const int y = y0 + wy, xA = x0 + lane, xB = xA + 32;
  const bool okA = y < ye && xA < xe, okB = y < ye && xB < xe;
  const T *own = ring + (wy + R) * SW + lane + R;
  const T *const cown = cring + (wy + 1) * CSW + lane + 1;
  // the coloured kernel's plane zc (cell: the byte offset of this warp's row): this lane's cell of the colour, if any
  auto coloured_row = [&](int zc, long long cell) {
    if constexpr (COL) {
      const int gx = x0 + p.col.par[0], gy = y + p.col.par[1], gz = zc + p.col.par[2], c = p.col.c;
      const bool on = p.col.m == 2 || (((gy ^ (c >> 1)) | (gz ^ (c >> 2))) & 1) == 0; // m = 8: the row's y and z parities
      const int s = (p.col.m == 2 ? c - gx - gy - gz : c - gx) & 1;                   // the x parity of the colour's cells
      const int xl = 2 * lane + s, x = x0 + xl;
      if (!on || y >= ye || x >= xe) return;
      const long long at = cell + x * ES;
      const T a = p.c.has_aux ? *reinterpret_cast<const T *>(p.c.aux + at) : T(0); // before the write: dst may be aux
      const T *const o1 = ring + (wy + R) * SW + R + xl;
      const int sl = slot_of(zc);
      T acc = T(0);
      for (int t = 0; t < p.c.n; ++t) {
        const T v = p.c.source[t] == 0 ? o1[p.toff[sl][t]] : a;
        T w = OpNum<T>::w(p.c, t);
        if constexpr (HAS_COEF) {
          const T *const co1 = cring + (wy + 1) * CSW + 1 + xl;
          const int cs = (zc - z0 + 1) & (kOpCoefSlots - 1);
          if (p.k.cfield[t] >= 0) w = OpNum<T>::mul(w, co1[p.k.coff[cs][t]]);
        }
        const T m = OpNum<T>::mul(w, v);
        acc = t == 0 ? m : OpNum<T>::add(acc, m);
      }
      *reinterpret_cast<T *>(p.c.dst + at) = acc;
    }
  };
  // DIAG: the cells of the colour in this warp's row of plane zc, each u + omega ((f - A u) / d); f is aux
  auto diag_row = [&](int zc, long long cell) {
    if constexpr (DIAG) {
      const int gx = x0 + p.col.par[0], gy = y + p.col.par[1], gz = zc + p.col.par[2], c = p.col.c, m = p.col.m;
      const bool on = m <= 2 || (((gy ^ (c >> 1)) | (gz ^ (c >> 2))) & 1) == 0;
      const int s = m == 1 ? 0 : (m == 2 ? c - gx - gy - gz : c - gx) & 1;
      if (!on || y >= ye) return;
      const int sl = slot_of(zc);
      for (int k = 0; k < (m == 1 ? 2 : 1); ++k) {
        const int xl = 2 * lane + s + k, x = x0 + xl;
        if (x >= xe) break;
        const long long at = cell + x * ES;
        const T f = *reinterpret_cast<const T *>(p.c.aux + at); // before the write: dst may be aux
        const T *const o1 = ring + (wy + R) * SW + R + xl;
        T acc = T(0), d = T(0);
        bool first = true;
        for (int t = 0; t < p.c.n; ++t) {
          T w = OpNum<T>::w(p.c, t);
          if constexpr (HAS_COEF) {
            const T *const co1 = cring + (wy + 1) * CSW + 1 + xl;
            const int cs = (zc - z0 + 1) & (kOpCoefSlots - 1);
            if (p.k.cfield[t] >= 0) w = OpNum<T>::mul(w, co1[p.k.coff[cs][t]]);
          }
          const T mt = OpNum<T>::mul(w, o1[p.toff[sl][t]]);
          acc = t == 0 ? mt : OpNum<T>::add(acc, mt);
          if ((p.dg.centre >> t) & 1ull) {
            d = first ? w : OpNum<T>::add(d, w);
            first = false;
          }
        }
        const T u = o1[sl * P];
        const T om = sizeof(T) == 4 ? T(p.dg.omegaf) : T(p.dg.omega);
        *reinterpret_cast<T *>(p.c.dst + at) = OpNum<T>::add(u, OpNum<T>::mul(om, OpNum<T>::div(OpNum<T>::sub(f, acc), d)));
      }
    }
  };
  for (int zc = z0; zc < z1; ++zc) {
    store(slot_of(zc + p.rp[2])); // the slot of plane zc + rp - (2R + 1), which no cell of plane zc reads
    if constexpr (HAS_COEF) cp_async_wait_all(); // this thread's coefficient planes up to zc + crp have landed
    __syncthreads();
    if (zc + 1 < z1) fetch(zc + 1 + p.rp[2]);
    if constexpr (HAS_COEF) {
      if (zc + 1 < z1) // into the slot of plane zc - 2 (or older), which no cell of plane zc reads
        for (int f = 0; f < p.k.nf; ++f) coef_plane(f, zc + 1 + p.k.crp[f][2]);
    }
    const long long cell = (long long)zc * p.c.slice + (long long)y * p.c.pitch;
    if constexpr (DIAG) {
      diag_row(zc, cell);
      __syncthreads();
      continue;
    } else if constexpr (COL) {
      coloured_row(zc, cell);
      __syncthreads();
      continue;
    }
    T auxA = T(0), auxB = T(0);
    if (p.c.has_aux) { // read before the cell is written: dst may be aux
      if (okA) auxA = *reinterpret_cast<const T *>(p.c.aux + cell + xA * ES);
      if (okB) auxB = *reinterpret_cast<const T *>(p.c.aux + cell + xB * ES);
    }
    const int c = slot_of(zc);
    const int cs = (zc - z0 + 1) & (kOpCoefSlots - 1);
    (void)cs;
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
      T mA, mB;
      if constexpr (HAS_COEF) { // (T(w) * C) * S
        T wA = w, wB = w;
        if (p.k.cfield[t] >= 0) {
          const int o = p.k.coff[cs][t];
          wA = OpNum<T>::mul(w, cown[o]);
          wB = OpNum<T>::mul(w, cown[o + 32]);
        }
        mA = OpNum<T>::mul(wA, vA);
        mB = OpNum<T>::mul(wB, vB);
      } else {
        mA = OpNum<T>::mul(w, vA);
        mB = OpNum<T>::mul(w, vB);
      }
      accA = t == 0 ? mA : OpNum<T>::add(accA, mA);
      accB = t == 0 ? mB : OpNum<T>::add(accB, mB);
    }
    if (okA) *reinterpret_cast<T *>(p.c.dst + cell + xA * ES) = accA;
    if (okB) *reinterpret_cast<T *>(p.c.dst + cell + xB * ES) = accB;
    __syncthreads();
  }
}

template <bool HAS_COEF, bool COL, bool DIAG = false>
using OpCellParamsOf = typename std::conditional<
    DIAG, OpDCellParams,
    typename std::conditional<COL, OpCCellParams, typename std::conditional<HAS_COEF, OpVCellParams, OpCellParams>::type>::type>::type;

// COL: the coloured kernel; a thread whose cell is of another colour does nothing.  DIAG (always with COL): the
// diagonal relaxation, every cell under m = 1.
template <typename T, bool HAS_COEF, bool COL, bool DIAG = false>
__global__ void __launch_bounds__(256) op_cell_kernel(const __grid_constant__ OpCellParamsOf<HAS_COEF, COL, DIAG> p) {
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
    if constexpr (DIAG) {
      const int gx = p.lo[k][0] + int(xx) + p.col.par[0], gy = p.lo[k][1] + int(yy) + p.col.par[1], gz = p.lo[k][2] + int(zz) + p.col.par[2];
      const int colour = p.col.m == 1 ? 0 : p.col.m == 2 ? (gx + gy + gz) & 1 : (gx & 1) | (gy & 1) << 1 | (gz & 1) << 2;
      if (colour != p.col.c) continue;
    } else if constexpr (COL) {
      const int gx = p.lo[k][0] + int(xx) + p.col.par[0], gy = p.lo[k][1] + int(yy) + p.col.par[1], gz = p.lo[k][2] + int(zz) + p.col.par[2];
      const int colour = p.col.m == 2 ? (gx + gy + gz) & 1 : (gx & 1) | (gy & 1) << 1 | (gz & 1) << 2;
      if (colour != p.col.c) continue;
    }
    const long long off = (long long)(p.lo[k][2] + (int)zz) * p.c.slice + (long long)(p.lo[k][1] + (int)yy) * p.c.pitch +
                          (long long)(p.lo[k][0] + (int)xx) * (long long)sizeof(T);
    const char *s = p.c.src + off;
    if constexpr (DIAG) { // u + omega ((f - A u) / d); f is aux, read before the write (dst may be aux)
      const T f = *reinterpret_cast<const T *>(p.c.aux + off);
      T acc = T(0), d = T(0);
      bool first = true;
      for (int t = 0; t < p.c.n; ++t) {
        T w = OpNum<T>::w(p.c, t);
        if constexpr (HAS_COEF) {
          const int fi = p.cfield[t];
          if (fi >= 0) w = OpNum<T>::mul(w, __ldg(reinterpret_cast<const T *>(p.coef[fi] + off + p.cgoff[t])));
        }
        const T m = OpNum<T>::mul(w, *reinterpret_cast<const T *>(s + p.goff[t]));
        acc = t == 0 ? m : OpNum<T>::add(acc, m);
        if ((p.dg.centre >> t) & 1ull) {
          d = first ? w : OpNum<T>::add(d, w);
          first = false;
        }
      }
      const T u = *reinterpret_cast<const T *>(s);
      const T om = sizeof(T) == 4 ? T(p.dg.omegaf) : T(p.dg.omega);
      *reinterpret_cast<T *>(p.c.dst + off) = OpNum<T>::add(u, OpNum<T>::mul(om, OpNum<T>::div(OpNum<T>::sub(f, acc), d)));
      continue;
    }
    const T a = p.c.has_aux ? *reinterpret_cast<const T *>(p.c.aux + off) : T(0); // before the write: dst may be aux
    T acc = T(0);
    for (int t = 0; t < p.c.n; ++t) {
      const T v = p.c.source[t] == 0 ? src_load<COL>(reinterpret_cast<const T *>(s + p.goff[t])) : a;
      T w = OpNum<T>::w(p.c, t);
      if constexpr (HAS_COEF) {
        const int f = p.cfield[t];
        if (f >= 0) w = OpNum<T>::mul(w, __ldg(reinterpret_cast<const T *>(p.coef[f] + off + p.cgoff[t])));
      }
      const T m = OpNum<T>::mul(w, v);
      acc = t == 0 ? m : OpNum<T>::add(acc, m);
    }
    *reinterpret_cast<T *>(p.c.dst + off) = acc;
  }
}

template <typename T, int R, bool COL> const void *tile_fn(bool coef) {
  return coef ? reinterpret_cast<const void *>(&op_tile_kernel<T, R, true, COL>) : reinterpret_cast<const void *>(&op_tile_kernel<T, R, false, COL>);
}
template <typename T, int R> const void *tile_fn(bool coef, bool col, bool diag) {
  if (diag)
    return coef ? reinterpret_cast<const void *>(&op_tile_kernel<T, R, true, true, true>)
                : reinterpret_cast<const void *>(&op_tile_kernel<T, R, false, true, true>);
  return col ? tile_fn<T, R, true>(coef) : tile_fn<T, R, false>(coef);
}

const void *tile_kernel(int R, int es, bool coef, bool col, bool diag) {
  switch (R * 10 + es) {
  case 14: return tile_fn<float, 1>(coef, col, diag);
  case 24: return tile_fn<float, 2>(coef, col, diag);
  case 34: return tile_fn<float, 3>(coef, col, diag);
  case 44: return tile_fn<float, 4>(coef, col, diag);
  case 18: return tile_fn<double, 1>(coef, col, diag);
  case 28: return tile_fn<double, 2>(coef, col, diag);
  case 38: return tile_fn<double, 3>(coef, col, diag);
  case 48: return tile_fn<double, 4>(coef, col, diag);
  default: return nullptr;
  }
}

} // namespace

size_t op_tile_smem(int R, int es, int nf) {
  return (size_t(2 * R + 1) * size_t(op_tile_plane(R)) + size_t(nf) * kOpCoefSlots * size_t(op_tile_plane(1))) * size_t(es);
}

int op_tile_prepare(int R, int es, int device, int nf, bool col, bool diag) {
  const void *fn = tile_kernel(R, es, nf > 0, col, diag);
  if (!fn) return 0;
  // the coefficient kernel's limit covers every field count, so plans with different counts can share it
  const int limit = int(op_tile_smem(R, es, nf > 0 ? kOpMaxCoefs : 0));
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, limit) != cudaSuccess) return 0;
  int ctas = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, fn, kOpThreads, op_tile_smem(R, es, nf)) != cudaSuccess) return 0;
  (void)device;
  return ctas;
}

int launch_op_tile(const OpDTileParams &p, int R, int es, int grid, cudaStream_t stream) {
  if (grid <= 0) return 0;
  const bool coef = p.k.nf > 0, diag = p.dg.on != 0, col = p.col.m > 1;
  const void *fn = tile_kernel(R, es, coef, col, diag);
  if (!fn) return 0;
  // the coloured kernels take the OpCTileParams part, the uncoloured ones the OpVTileParams part, the plain one the
  // OpTileParams part only
  OpDTileParams *const q = const_cast<OpDTileParams *>(&p);
  void *args[] = {diag  ? static_cast<void *>(q)
                  : col ? static_cast<void *>(static_cast<OpCTileParams *>(q))
                  : coef ? static_cast<void *>(static_cast<OpVTileParams *>(q))
                         : static_cast<void *>(static_cast<OpTileParams *>(q))};
  cudaLaunchKernel(fn, dim3(unsigned(grid)), dim3(kOpThreads), args, op_tile_smem(R, es, p.k.nf), stream);
  return 1;
}

int launch_op_cells(const OpDCellParams &p, int es, bool has_coef, int grid, cudaStream_t stream) {
  if (grid <= 0 || p.n <= 0) return 0;
  const OpCCellParams &cc = p;
  const OpVCellParams &v = p;
  const OpCellParams &b = p;
  const unsigned g = unsigned(grid);
  if (p.dg.on) {
    if (es == 4 && has_coef)
      op_cell_kernel<float, true, true, true><<<g, 256, 0, stream>>>(p);
    else if (es == 4)
      op_cell_kernel<float, false, true, true><<<g, 256, 0, stream>>>(p);
    else if (has_coef)
      op_cell_kernel<double, true, true, true><<<g, 256, 0, stream>>>(p);
    else
      op_cell_kernel<double, false, true, true><<<g, 256, 0, stream>>>(p);
  } else if (p.col.m > 1) {
    if (es == 4 && has_coef)
      op_cell_kernel<float, true, true><<<g, 256, 0, stream>>>(cc);
    else if (es == 4)
      op_cell_kernel<float, false, true><<<g, 256, 0, stream>>>(cc);
    else if (has_coef)
      op_cell_kernel<double, true, true><<<g, 256, 0, stream>>>(cc);
    else
      op_cell_kernel<double, false, true><<<g, 256, 0, stream>>>(cc);
  } else if (es == 4 && has_coef)
    op_cell_kernel<float, true, false><<<g, 256, 0, stream>>>(v);
  else if (es == 4)
    op_cell_kernel<float, false, false><<<g, 256, 0, stream>>>(b);
  else if (has_coef)
    op_cell_kernel<double, true, false><<<g, 256, 0, stream>>>(v);
  else
    op_cell_kernel<double, false, false><<<g, 256, 0, stream>>>(b);
  return 1;
}

} // namespace sb
