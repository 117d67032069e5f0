// Astaroth `solve<step>` for sm_90a (H100).  See astaroth.cuh for the reference anchors.
//
// What the reference does (astaroth/user_kernels.h:437-469 with block (32,1,4), astaroth/kernels.cu:67): every thread
// rebuilds value + gradient + full hessian of all 8 fields from global memory -- 8 x 55 neighbour loads per cell, 254
// registers -- and relies on L1 for reuse.
//
// What this file does:
//  * only the derivatives the equations consume (lnrho, entropy: no cross terms; each vector component: two of the
//    three cross terms) -- 296 instead of 440 neighbour values per cell;
//  * tile kernel: a CTA owns a TX x TY column of cells and marches in z.  The halo'd planes z-3..z+3 of all 8 fields
//    live in a shared-memory ring (FP64: 8 fields x 8 slots x 22 x 20 doubles = 220 KiB of the SM's 227 KiB; FP32: 32 x 8
//    tiles, 133 KiB); plane
//    z+4 streams in with cp.async while plane z is computed, one __syncthreads per plane.  Every neighbour value is an
//    LDS with an immediate offset (ring slot bases are 7 registers), x-y reuse never leaves the SM, and HBM sees each
//    input plane once per tile (+ halo overlap served by L2);
//  * cell kernel for thin boxes (the 3-cell exterior slabs): one thread per cell, neighbours through the read-only path.
// Roofline: 8 reads + 8 reads of `out` + 8 writes per cell = 24 x sizeof(T) bytes (16 x for step 0, which ignores the
// previous state); with ~300 shared-memory loads and ~900 FP instructions per cell the FP64 kernel is shared-memory /
// DFMA-issue bound before it is HBM bound.
#include "astaroth.cuh"

#include <cuda.h>

#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>

namespace sb {
namespace {

enum { LNRHO = 0, UUX, UUY, UUZ, AX, AY, AZ, ENTROPY };

template <typename T> struct AcConst {
  T ix, iy, iz, dt, cs2s, gam, cp, lnrho0, lnT0, mu0, nu, zeta, eta;
  T icp, imu0, elnT0; // 1 / cp, 1 / mu0, exp(lnT0): hoisted to the host (team kernel)
};

template <typename T> AcConst<T> make_const(const AcParams &p) {
  AcConst<T> c;
  c.ix = T(p.inv_dsx), c.iy = T(p.inv_dsy), c.iz = T(p.inv_dsz), c.dt = T(p.dt);
  c.cs2s = T(p.cs2_sound), c.gam = T(p.gamma), c.cp = T(p.cp_sound), c.lnrho0 = T(p.lnrho0), c.lnT0 = T(p.lnT0);
  c.mu0 = T(p.mu0), c.nu = T(p.nu_visc), c.zeta = T(p.zeta), c.eta = T(p.eta);
  c.icp = T(1.0 / p.cp_sound), c.imu0 = T(1.0 / p.mu0), c.elnT0 = T(exp(p.lnT0));
  return c;
}

template <typename T> struct AcArgs {
  const T *in[kAcFields];
  T *out[kAcFields];
  int mx, my;
  long long mxy;
  int lo[3], hi[3];
  int zchunk;
  AcConst<T> P;
};

// value, gradient and the second derivatives one field contributes
template <typename T> struct Dv {
  T v, gx, gy, gz, xx, yy, zz, xy, xz, yz;
};

__device__ __forceinline__ double ac_exp(double x) { return exp(x); }
__device__ __forceinline__ float ac_exp(float x) { return expf(x); }

// first / second / cross derivative, same association order as astaroth/user_kernels.h:36-75
template <typename T> __device__ __forceinline__ T d1(T m3, T m2, T m1, T p1, T p2, T p3, T inv) {
  const T c1 = T(3.0) / T(4.0), c2 = -T(3.0) / T(20.0), c3 = T(1.0) / T(60.0);
  T r = c1 * (p1 - m1);
  r += c2 * (p2 - m2);
  r += c3 * (p3 - m3);
  return r * inv;
}
template <typename T> __device__ __forceinline__ T d2(T c, T m3, T m2, T m1, T p1, T p2, T p3, T inv) {
  const T c0 = -T(49.0) / T(18.0), c1 = T(3.0) / T(2.0), c2 = -T(3.0) / T(20.0), c3 = T(1.0) / T(90.0);
  T r = c0 * c;
  r += c1 * (p1 + m1);
  r += c2 * (p2 + m2);
  r += c3 * (p3 + m3);
  return r * inv * inv;
}
// a: the (+,+) diagonal, b: the (+,-) diagonal; am_i = a[3-i], ap_i = a[3+i]
template <typename T>
__device__ __forceinline__ T dc(T am3, T am2, T am1, T ap1, T ap2, T ap3, T bm3, T bm2, T bm1, T bp1, T bp2, T bp3, T inva, T invb) {
  const T fac = T(1.0) / T(720.0);
  const T c1 = T(270.0) * fac, c2 = -T(27.0) * fac, c3 = T(2.0) * fac;
  T r = c1 * (ap1 + am1 - bp1 - bm1);
  r += c2 * (ap2 + am2 - bp2 - bm2);
  r += c3 * (ap3 + am3 - bp3 - bm3);
  return r * inva * invb;
}

// The compiler may not move memory operations across this point.  Used between the pencils of derive<PACE = true>: left
// alone, the scheduler hoists all ~43 shared-memory loads of a field (and of the next field) to the front and issues
// them back to back -- ncu: 2.8 "MIO throttle" stalls per issued instruction with the shared-memory pipe only 55 % busy,
// because every warp alternates between a burst of LDS and a long stretch of FP64.  With the fences a warp issues
// the <= 12 loads of one pencil, then the arithmetic of the previous one: loads and arithmetic interleave at a steady rate.
__device__ __forceinline__ void pace() { asm volatile("" ::: "memory"); }

// `at(dx, dy, dz)` returns the field value at that offset from the cell (offsets are compile-time after inlining).
template <typename T, bool XY, bool XZ, bool YZ, bool PACE = false, typename At> __device__ __forceinline__ Dv<T> derive(At at, const AcConst<T> &P) {
  Dv<T> d;
  const T c = at(0, 0, 0);
  d.v = c;
  {
    const T m3 = at(-3, 0, 0), m2 = at(-2, 0, 0), m1 = at(-1, 0, 0), p1 = at(1, 0, 0), p2 = at(2, 0, 0), p3 = at(3, 0, 0);
    if (PACE) pace();
    d.gx = d1(m3, m2, m1, p1, p2, p3, P.ix);
    d.xx = d2(c, m3, m2, m1, p1, p2, p3, P.ix);
  }
  {
    const T m3 = at(0, -3, 0), m2 = at(0, -2, 0), m1 = at(0, -1, 0), p1 = at(0, 1, 0), p2 = at(0, 2, 0), p3 = at(0, 3, 0);
    if (PACE) pace();
    d.gy = d1(m3, m2, m1, p1, p2, p3, P.iy);
    d.yy = d2(c, m3, m2, m1, p1, p2, p3, P.iy);
  }
  {
    const T m3 = at(0, 0, -3), m2 = at(0, 0, -2), m1 = at(0, 0, -1), p1 = at(0, 0, 1), p2 = at(0, 0, 2), p3 = at(0, 0, 3);
    if (PACE) pace();
    d.gz = d1(m3, m2, m1, p1, p2, p3, P.iz);
    d.zz = d2(c, m3, m2, m1, p1, p2, p3, P.iz);
  }
  d.xy = d.xz = d.yz = T(0);
  if (XY) { // derxy, astaroth/user_kernels.h:96-111
    const T a0 = at(-3, -3, 0), a1 = at(-2, -2, 0), a2 = at(-1, -1, 0), a3 = at(1, 1, 0), a4 = at(2, 2, 0), a5 = at(3, 3, 0);
    const T b0 = at(-3, 3, 0), b1 = at(-2, 2, 0), b2 = at(-1, 1, 0), b3 = at(1, -1, 0), b4 = at(2, -2, 0), b5 = at(3, -3, 0);
    if (PACE) pace();
    d.xy = dc(a0, a1, a2, a3, a4, a5, b0, b1, b2, b3, b4, b5, P.ix, P.iy);
  }
  if (XZ) { // derxz, :112-127
    const T a0 = at(-3, 0, -3), a1 = at(-2, 0, -2), a2 = at(-1, 0, -1), a3 = at(1, 0, 1), a4 = at(2, 0, 2), a5 = at(3, 0, 3);
    const T b0 = at(-3, 0, 3), b1 = at(-2, 0, 2), b2 = at(-1, 0, 1), b3 = at(1, 0, -1), b4 = at(2, 0, -2), b5 = at(3, 0, -3);
    if (PACE) pace();
    d.xz = dc(a0, a1, a2, a3, a4, a5, b0, b1, b2, b3, b4, b5, P.ix, P.iz);
  }
  if (YZ) { // deryz, :148-163
    const T a0 = at(0, -3, -3), a1 = at(0, -2, -2), a2 = at(0, -1, -1), a3 = at(0, 1, 1), a4 = at(0, 2, 2), a5 = at(0, 3, 3);
    const T b0 = at(0, -3, 3), b1 = at(0, -2, 2), b2 = at(0, -1, 1), b3 = at(0, 1, -1), b4 = at(0, 2, -2), b5 = at(0, 3, -3);
    if (PACE) pace();
    d.yz = dc(a0, a1, a2, a3, a4, a5, b0, b1, b2, b3, b4, b5, P.iy, P.iz);
  }
  return d;
}

template <int STEP, typename T> __device__ __forceinline__ T rk3(T prev, T curr, T roc, T dt) {
  // Williamson (1980), astaroth/integration.cuh:14-37
  const T alpha[4] = {0, T(.0), T(-5. / 9.), T(-153. / 128.)};
  const T beta[4] = {0, T(1. / 3.), T(15. / 16.), T(8. / 15.)};
  if (STEP == 0) return curr + beta[STEP + 1] * roc * dt;
  return curr + beta[STEP + 1] * (alpha[STEP + 1] * (T(1.) / beta[STEP]) * (curr - prev) + roc * dt);
}

// continuity / momentum / induction / entropy (astaroth/user_kernels.h:376-428) + the RK3 update (:444-453).
// `prev[f]` is the `out` field before the update (unused for STEP 0), `res[f]` what solve<> writes back.
template <int STEP, typename T>
__device__ __forceinline__ void physics(const Dv<T> &lr, const Dv<T> *u, const Dv<T> *a, const Dv<T> &s, const T *prev, T *res,
                                        const AcConst<T> &P) {
  const T ux = u[0].v, uy = u[1].v, uz = u[2].v;
  const T divu = u[0].gx + u[1].gy + u[2].gz;
  const T cont = -(ux * lr.gx + uy * lr.gy + uz * lr.gz) - divu;
  // induction
  const T Bx = a[2].gy - a[1].gz, By = a[0].gz - a[2].gx, Bz = a[1].gx - a[0].gy;
  const T lax = a[0].xx + a[0].yy + a[0].zz, lay = a[1].xx + a[1].yy + a[1].zz, laz = a[2].xx + a[2].yy + a[2].zz;
  const T indx = (uy * Bz - uz * By) + P.eta * lax;
  const T indy = (uz * Bx - ux * Bz) + P.eta * lay;
  const T indz = (ux * By - uy * Bx) + P.eta * laz;
  // current density j = (grad div A - lap A) / mu0
  const T imu0 = T(1.0) / P.mu0;
  const T jx = imu0 * ((a[0].xx + a[1].xy + a[2].xz) - lax);
  const T jy = imu0 * ((a[0].xy + a[1].yy + a[2].yz) - lay);
  const T jz = imu0 * ((a[0].xz + a[1].yz + a[2].zz) - laz);
  // momentum
  const T S00 = (T(2.0) / T(3.0)) * u[0].gx - (T(1.0) / T(3.0)) * (u[1].gy + u[2].gz);
  const T S01 = (T(1.0) / T(2.0)) * (u[0].gy + u[1].gx);
  const T S02 = (T(1.0) / T(2.0)) * (u[0].gz + u[2].gx);
  const T S11 = (T(2.0) / T(3.0)) * u[1].gy - (T(1.0) / T(3.0)) * (u[0].gx + u[2].gz);
  const T S12 = (T(1.0) / T(2.0)) * (u[1].gz + u[2].gy);
  const T S22 = (T(2.0) / T(3.0)) * u[2].gz - (T(1.0) / T(3.0)) * (u[0].gx + u[1].gy);
  const T arg = P.gam * s.v / P.cp + (P.gam - T(1.0)) * (lr.v - P.lnrho0);
  const T earg = ac_exp(arg);
  const T cs2 = P.cs2s * earg;
  const T rho = ac_exp(lr.v);
  const T inv_rho = T(1.0) / rho;
  const T icp = T(1.0) / P.cp;
  const T gdx = u[0].xx + u[1].xy + u[2].xz, gdy = u[0].xy + u[1].yy + u[2].yz, gdz = u[0].xz + u[1].yz + u[2].zz;
  const T lux = u[0].xx + u[0].yy + u[0].zz, luy = u[1].xx + u[1].yy + u[1].zz, luz = u[2].xx + u[2].yy + u[2].zz;
  const T jxBx = jy * Bz - jz * By, jxBy = jz * Bx - jx * Bz, jxBz = jx * By - jy * Bx;
  const T Sgx = S00 * lr.gx + S01 * lr.gy + S02 * lr.gz;
  const T Sgy = S01 * lr.gx + S11 * lr.gy + S12 * lr.gz;
  const T Sgz = S02 * lr.gx + S12 * lr.gy + S22 * lr.gz;
  T momx = -(u[0].gx * ux + u[0].gy * uy + u[0].gz * uz);
  T momy = -(u[1].gx * ux + u[1].gy * uy + u[1].gz * uz);
  T momz = -(u[2].gx * ux + u[2].gy * uy + u[2].gz * uz);
  momx = momx - cs2 * (icp * s.gx + lr.gx);
  momy = momy - cs2 * (icp * s.gy + lr.gy);
  momz = momz - cs2 * (icp * s.gz + lr.gz);
  momx = momx + inv_rho * jxBx;
  momy = momy + inv_rho * jxBy;
  momz = momz + inv_rho * jxBz;
  momx = momx + P.nu * ((lux + (T(1.0) / T(3.0)) * gdx) + T(2.0) * Sgx);
  momy = momy + P.nu * ((luy + (T(1.0) / T(3.0)) * gdy) + T(2.0) * Sgy);
  momz = momz + P.nu * ((luz + (T(1.0) / T(3.0)) * gdz) + T(2.0) * Sgz);
  momx = momx + P.zeta * gdx;
  momy = momy + P.zeta * gdy;
  momz = momz + P.zeta * gdz;
  // entropy.  exp(lnT) = exp(lnT0 + arg): the reference evaluates a third exp; exp(lnT0) * exp(arg) differs by rounding only
  const T elnT = ac_exp(P.lnT0 + arg);
  const T inv_pT = T(1.0) / (rho * elnT);
  const T SS = (S00 * S00 + S01 * S01 + S02 * S02) + (S01 * S01 + S11 * S11 + S12 * S12) + (S02 * S02 + S12 * S12 + S22 * S22);
  const T RHS = P.eta * P.mu0 * (jx * jx + jy * jy + jz * jz) + T(2.0) * rho * P.nu * SS + P.zeta * rho * divu * divu;
  const T ls = s.xx + s.yy + s.zz, llr = lr.xx + lr.yy + lr.zz;
  const T first = P.gam * icp * ls + (P.gam - T(1.0)) * llr;
  const T s2x = P.gam * icp * s.gx + (P.gam - T(1.0)) * lr.gx;
  const T s2y = P.gam * icp * s.gy + (P.gam - T(1.0)) * lr.gy;
  const T s2z = P.gam * icp * s.gz + (P.gam - T(1.0)) * lr.gz;
  const T t3x = P.gam * (icp * s.gx + lr.gx) + (-lr.gx);
  const T t3y = P.gam * (icp * s.gy + lr.gy) + (-lr.gy);
  const T t3z = P.gam * (icp * s.gz + lr.gz) + (-lr.gz);
  const T chi = T(0.001) / (rho * P.cp);
  const T heat = P.cp * chi * (first + (s2x * t3x + s2y * t3y + s2z * t3z));
  const T ent = -(ux * s.gx + uy * s.gy + uz * s.gz) + inv_pT * RHS + heat;

  res[LNRHO] = rk3<STEP>(prev[LNRHO], lr.v, cont, P.dt);
  res[AX] = rk3<STEP>(prev[AX], a[0].v, indx, P.dt);
  res[AY] = rk3<STEP>(prev[AY], a[1].v, indy, P.dt);
  res[AZ] = rk3<STEP>(prev[AZ], a[2].v, indz, P.dt);
  res[UUX] = rk3<STEP>(prev[UUX], ux, momx, P.dt);
  res[UUY] = rk3<STEP>(prev[UUY], uy, momy, P.dt);
  res[UUZ] = rk3<STEP>(prev[UUZ], uz, momz, P.dt);
  res[ENTROPY] = rk3<STEP>(prev[ENTROPY], s.v, ent, P.dt);
}

template <int STEP, typename T, typename AtF>
__device__ __forceinline__ void solve_cell(AtF atf, const AcArgs<T> &A, long long idx) {
  // atf(f) returns the accessor of field f
  Dv<T> u[3], a[3];
  const Dv<T> lr = derive<T, false, false, false>(atf(LNRHO), A.P);
  const Dv<T> s = derive<T, false, false, false>(atf(ENTROPY), A.P);
  u[0] = derive<T, true, true, false>(atf(UUX), A.P);
  u[1] = derive<T, true, false, true>(atf(UUY), A.P);
  u[2] = derive<T, false, true, true>(atf(UUZ), A.P);
  a[0] = derive<T, true, true, false>(atf(AX), A.P);
  a[1] = derive<T, true, false, true>(atf(AY), A.P);
  a[2] = derive<T, false, true, true>(atf(AZ), A.P);
  T prev[kAcFields], res[kAcFields];
#pragma unroll
  for (int f = 0; f < kAcFields; ++f) prev[f] = (STEP == 0) ? T(0) : A.out[f][idx];
  physics<STEP>(lr, u, a, s, prev, res, A.P);
#pragma unroll
  for (int f = 0; f < kAcFields; ++f) A.out[f][idx] = res[f];
}

// ---------------------------------------------------------------------------------------------- cell kernel
// 128 threads shaped (1 << lgx, 1 << lgy, rest) so that thin boxes keep their lanes busy.
template <int STEP, typename T> __global__ void __launch_bounds__(128) ac_cell_kernel(const __grid_constant__ AcArgs<T> A, int lgx, int lgy) {
  const int t = threadIdx.x;
  const int tx = t & ((1 << lgx) - 1), ty = (t >> lgx) & ((1 << lgy) - 1), tz = t >> (lgx + lgy);
  const int x = A.lo[0] + (blockIdx.x << lgx) + tx;
  const int y = A.lo[1] + (blockIdx.y << lgy) + ty;
  const int z = A.lo[2] + blockIdx.z * (128 >> (lgx + lgy)) + tz;
  if (x >= A.hi[0] || y >= A.hi[1] || z >= A.hi[2]) return;
  const long long idx = (long long)z * A.mxy + (long long)y * A.mx + x;
  const int mx = A.mx;
  const long long mxy = A.mxy;
  auto atf = [&](int f) {
    const T *p = A.in[f] + idx;
    return [p, mx, mxy](int dx, int dy, int dz) { return __ldg(p + dz * mxy + dy * mx + dx); };
  };
  solve_cell<STEP>(atf, A, idx);
}

// ---------------------------------------------------------------------------------------------- tile kernel
template <int BYTES> __device__ __forceinline__ void cp_async(void *smem, const void *gmem) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(s), "l"(gmem), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <int STEP, typename T, int TX, int TY, int NSLOT>
__global__ void __launch_bounds__(TX *TY, 1) ac_tile_kernel(const __grid_constant__ AcArgs<T> A) {
  constexpr int W = TX + 6, H = TY + 6, PL = W * H, NT = TX * TY, NL = (PL + NT - 1) / NT;
  static_assert(NSLOT == 7 || NSLOT == 8, "ring of 7 (synchronous refill) or 8 (refill overlaps the computation) planes");
  extern __shared__ __align__(16) unsigned char ac_smem[];
  T *ring = reinterpret_cast<T *>(ac_smem); // [field][slot][H][W]

  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const int x0 = A.lo[0] + blockIdx.x * TX, y0 = A.lo[1] + blockIdx.y * TY;
  const int z0 = A.lo[2] + blockIdx.z * A.zchunk;
  const int z1 = min(z0 + A.zchunk, A.hi[2]);
  const int mx = A.mx;
  const long long mxy = A.mxy;

  // what this thread fetches of every plane: element k of the halo'd tile -> (shared offset, global offset)
  int goff[NL];
#pragma unroll
  for (int k = 0; k < NL; ++k) {
    const int e = tid + k * NT;
    const int r = e / W, c = e - r * W;
    const int gx = min(x0 - 3 + c, mx - 1), gy = min(y0 - 3 + r, A.my - 1); // partial tiles: stay inside the allocation
    goff[k] = (e < PL) ? gy * mx + gx : -1;
  }
  auto load_plane = [&](int p, int slot) {
#pragma unroll
    for (int f = 0; f < kAcFields; ++f) {
      const T *src = A.in[f] + (long long)p * mxy;
      T *dst = ring + (f * NSLOT + slot) * PL + tid;
#pragma unroll
      for (int k = 0; k < NL; ++k) {
        if (goff[k] >= 0) cp_async<sizeof(T)>(dst + k * NT, src + goff[k]);
      }
    }
  };

  for (int p = z0 - 3; p <= z0 + 3; ++p) load_plane(p, p - z0 + 3);
  cp_async_commit();
  cp_async_wait_all();
  __syncthreads();

  const bool valid = (x0 + tx < A.hi[0]) && (y0 + ty < A.hi[1]);
  const int o0 = (ty + 3) * W + tx + 3;
  long long idx = (long long)z0 * mxy + (long long)(y0 + ty) * mx + (x0 + tx);

  for (int z = z0; z < z1; ++z, idx += mxy) {
    const int zi = z - z0;
    const bool more = z + 1 < z1;
    if (NSLOT == 8) {
      if (more) load_plane(z + 4, (zi + 7) % NSLOT);
      cp_async_commit();
    }
    if (valid) {
      const T *b[7]; // plane z-3+k of field 0 at this thread's cell
#pragma unroll
      for (int k = 0; k < 7; ++k) b[k] = ring + ((zi + k) % NSLOT) * PL + o0;
      auto atf = [&](int f) {
        return [&b, f](int dx, int dy, int dz) { return b[dz + 3][f * NSLOT * PL + dy * W + dx]; };
      };
      solve_cell<STEP>(atf, A, idx);
    }
    if (NSLOT == 8) {
      cp_async_wait_all();
      __syncthreads();
    } else {
      __syncthreads(); // everyone is done with plane z-3 before its slot is refilled
      if (more) {
        load_plane(z + 4, (zi + 7) % NSLOT);
        cp_async_commit();
        cp_async_wait_all();
        __syncthreads();
      }
    }
  }
}

int env_int(const char *name, int dflt);

// ---------------------------------------------------------------------------------------------- team kernel
// Two threads per cell.  The tile kernel above keeps value + gradient + hessian of all 8 fields live until the physics
// runs (238 registers -> 7 warps per SM), and all of its warps alternate between a shared-memory phase (296 LDS) and an
// FP64 phase (~900 instructions) in lock step behind the per-plane barrier: ncu shows the two pipes at 53 % and 31 %,
// never overlapping.  Here
//   team U (threads [0, NC))      derives lnrho, entropy, uux, uuy, uuz and folds every field into a handful of running
//                                 sums the moment it is derived (advection, div u, lap u, grad div u, the six entries of
//                                 the rate-of-strain tensor, ...), then integrates continuity, momentum and entropy;
//   team A (threads [NC, 2 NC))   derives ax, ay, az (curl, laplacian, grad div), integrates the induction equation and
//                                 hands j x B and |j|^2 to team U through 4 words of shared memory per cell.
// Nobody holds more than ~35 live values, the CTA has twice the warps on the same shared-memory ring, and the two teams
// have different LDS : FP64 mixes, so one team's loads overlap the other's arithmetic.  The only intra-plane dependency
// is a named barrier (team A arrives, team U waits) just before team U's final assembly.
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// One plane of the two-team scheme (see ac_team_kernel): team A (induction) or team U (continuity, momentum, entropy) of
// the cell at shared-memory offset o0 of ring plane `zi`, global index idx.  Shared by the cp.async-fed and the TMA-fed kernel.
template <int STEP, typename T, int W, int PL, int NSLOT, int NC, bool PACED>
__device__ __forceinline__ void team_plane(const AcArgs<T> &A, const T *ring, T *xb, int zi, int o0, int cell, bool teamA, bool valid, long long idx) {
  constexpr int NT = 2 * NC;
  const AcConst<T> &P = A.P;
  const T third = T(1.0) / T(3.0), half = T(0.5);
  const T *b[7]; // plane z-3+k of field 0 at this thread's cell
#pragma unroll
  for (int k = 0; k < 7; ++k) b[k] = ring + ((zi + k) % NSLOT) * PL + o0;
  auto atf = [&](int f) {
    return [&b, f](int dx, int dy, int dz) { return b[dz + 3][f * NSLOT * PL + dy * W + dx]; };
  };
  const T ux = b[3][UUX * NSLOT * PL], uy = b[3][UUY * NSLOT * PL], uz = b[3][UUZ * NSLOT * PL];
  if (teamA) {
    if (valid) {
      T pa[3];
#pragma unroll
      for (int i = 0; i < 3; ++i) pa[i] = (STEP == 0) ? T(0) : A.out[AX + i][idx];
      // curl A, laplacian A, grad div A, folded field by field
      T Bx, By, Bz, lax, lay, laz, gx, gy, gz, av[3];
      {
        const Dv<T> d = derive<T, true, true, false, PACED>(atf(AX), P);
        av[0] = d.v;
        By = d.gz, Bz = -d.gy;
        lax = d.xx + d.yy + d.zz;
        gx = d.xx, gy = d.xy, gz = d.xz;
      }
      {
        const Dv<T> d = derive<T, true, false, true, PACED>(atf(AY), P);
        av[1] = d.v;
        Bx = -d.gz, Bz += d.gx;
        lay = d.xx + d.yy + d.zz;
        gx += d.xy, gy += d.yy, gz += d.yz;
      }
      {
        const Dv<T> d = derive<T, false, true, true, PACED>(atf(AZ), P);
        av[2] = d.v;
        Bx += d.gy, By -= d.gx;
        laz = d.xx + d.yy + d.zz;
        gx += d.xz, gy += d.yz, gz += d.zz;
      }
      const T indx = (uy * Bz - uz * By) + P.eta * lax;
      const T indy = (uz * Bx - ux * Bz) + P.eta * lay;
      const T indz = (ux * By - uy * Bx) + P.eta * laz;
      const T jx = P.imu0 * (gx - lax), jy = P.imu0 * (gy - lay), jz = P.imu0 * (gz - laz);
      xb[0 * NC + cell] = jy * Bz - jz * By;
      xb[1 * NC + cell] = jz * Bx - jx * Bz;
      xb[2 * NC + cell] = jx * By - jy * Bx;
      xb[3 * NC + cell] = jx * jx + jy * jy + jz * jz;
      A.out[AX][idx] = rk3<STEP>(pa[0], av[0], indx, P.dt);
      A.out[AY][idx] = rk3<STEP>(pa[1], av[1], indy, P.dt);
      A.out[AZ][idx] = rk3<STEP>(pa[2], av[2], indz, P.dt);
    }
    __threadfence_block();
    bar_arrive(1, NT);
  } else {
    T pl = T(0), ps = T(0), pu[3] = {T(0), T(0), T(0)};
    T lrv = T(0), sv = T(0), cont = T(0), entadv = T(0), heat_in = T(0), arg = T(0);
    T lg[3] = {T(0), T(0), T(0)}, G[3] = {T(0), T(0), T(0)};
    T madv[3], lu[3], gd[3], divu = T(0), S00 = T(0), S11 = T(0), S22 = T(0), S01 = T(0), S02 = T(0), S12 = T(0);
#pragma unroll
    for (int i = 0; i < 3; ++i) madv[i] = lu[i] = gd[i] = T(0);
    if (valid) {
      if (STEP != 0) {
        pl = A.out[LNRHO][idx], ps = A.out[ENTROPY][idx];
#pragma unroll
        for (int i = 0; i < 3; ++i) pu[i] = A.out[UUX + i][idx];
      }
      T llr;
      {
        const Dv<T> d = derive<T, false, false, false, PACED>(atf(LNRHO), P);
        lrv = d.v;
        lg[0] = d.gx, lg[1] = d.gy, lg[2] = d.gz;
        llr = d.xx + d.yy + d.zz;
        cont = -(ux * d.gx + uy * d.gy + uz * d.gz);
      }
      {
        const Dv<T> d = derive<T, false, false, false, PACED>(atf(ENTROPY), P);
        sv = d.v;
        const T ls = d.xx + d.yy + d.zz;
        const T sg[3] = {d.gx, d.gy, d.gz};
        const T first = P.gam * P.icp * ls + (P.gam - T(1.0)) * llr;
        T dot = T(0);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          G[i] = P.icp * sg[i] + lg[i];
          const T s2 = P.gam * P.icp * sg[i] + (P.gam - T(1.0)) * lg[i];
          const T t3 = P.gam * G[i] + (-lg[i]);
          dot += s2 * t3;
        }
        heat_in = first + dot;
        entadv = -(ux * d.gx + uy * d.gy + uz * d.gz);
        arg = P.gam * d.v * P.icp + (P.gam - T(1.0)) * (lrv - P.lnrho0);
      }
      {
        const Dv<T> d = derive<T, true, true, false, PACED>(atf(UUX), P);
        madv[0] = -(d.gx * ux + d.gy * uy + d.gz * uz);
        divu = d.gx;
        lu[0] = d.xx + d.yy + d.zz;
        gd[0] = d.xx, gd[1] = d.xy, gd[2] = d.xz;
        S00 = (T(2.0) * third) * d.gx, S11 = -third * d.gx, S22 = S11;
        S01 = half * d.gy, S02 = half * d.gz;
      }
      {
        const Dv<T> d = derive<T, true, false, true, PACED>(atf(UUY), P);
        madv[1] = -(d.gx * ux + d.gy * uy + d.gz * uz);
        divu += d.gy;
        lu[1] = d.xx + d.yy + d.zz;
        gd[0] += d.xy, gd[1] += d.yy, gd[2] += d.yz;
        S00 -= third * d.gy, S11 += (T(2.0) * third) * d.gy, S22 -= third * d.gy;
        S01 += half * d.gx, S12 = half * d.gz;
      }
      {
        const Dv<T> d = derive<T, false, true, true, PACED>(atf(UUZ), P);
        madv[2] = -(d.gx * ux + d.gy * uy + d.gz * uz);
        divu += d.gz;
        lu[2] = d.xx + d.yy + d.zz;
        gd[0] += d.xz, gd[1] += d.yz, gd[2] += d.zz;
        S00 -= third * d.gz, S11 -= third * d.gz, S22 += (T(2.0) * third) * d.gz;
        S02 += half * d.gx, S12 += half * d.gy;
      }
    }
    bar_sync(1, NT); // team A's j x B and |j|^2 of this plane are in xb
    if (valid) {
      const T jxB[3] = {xb[0 * NC + cell], xb[1 * NC + cell], xb[2 * NC + cell]};
      const T j2 = xb[3 * NC + cell];
      const T earg = ac_exp(arg);
      const T cs2 = P.cs2s * earg;
      const T rho = ac_exp(lrv);
      const T inv_rho = T(1.0) / rho;
      const T Sg[3] = {S00 * lg[0] + S01 * lg[1] + S02 * lg[2], S01 * lg[0] + S11 * lg[1] + S12 * lg[2], S02 * lg[0] + S12 * lg[1] + S22 * lg[2]};
      const T uv[3] = {ux, uy, uz};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        T m = madv[i] - cs2 * G[i];
        m = m + inv_rho * jxB[i];
        m = m + P.nu * ((lu[i] + third * gd[i]) + T(2.0) * Sg[i]);
        m = m + P.zeta * gd[i];
        A.out[UUX + i][idx] = rk3<STEP>(pu[i], uv[i], m, P.dt);
      }
      A.out[LNRHO][idx] = rk3<STEP>(pl, lrv, cont - divu, P.dt);
      // exp(lnT) = exp(lnT0) * exp(arg): the reference evaluates a third exp (rounding-level difference)
      const T inv_pT = T(1.0) / (rho * (P.elnT0 * earg));
      const T SS = (S00 * S00 + S01 * S01 + S02 * S02) + (S01 * S01 + S11 * S11 + S12 * S12) + (S02 * S02 + S12 * S12 + S22 * S22);
      const T RHS = P.eta * P.mu0 * j2 + T(2.0) * rho * P.nu * SS + P.zeta * rho * divu * divu;
      const T chi = T(0.001) / (rho * P.cp);
      const T ent = entadv + inv_pT * RHS + P.cp * chi * heat_in;
      A.out[ENTROPY][idx] = rk3<STEP>(ps, sv, ent, P.dt);
    }
  }
}

template <int STEP, typename T, int TX, int TY, int NSLOT, bool PACED>
__global__ void __launch_bounds__(2 * TX *TY, 1) ac_team_kernel(const __grid_constant__ AcArgs<T> A) {
  constexpr int W = TX + 6, H = TY + 6, PL = W * H, NC = TX * TY, NT = 2 * NC, NL = (PL + NT - 1) / NT;
  static_assert(NSLOT == 8, "ring of 8 planes: 7 in use + 1 in flight");
  extern __shared__ __align__(16) unsigned char ac_smem[];
  T *ring = reinterpret_cast<T *>(ac_smem);      // [field][slot][H][W]
  T *xb = ring + kAcFields * NSLOT * PL;         // [4][NC]: (j x B).xyz, |j|^2 of the plane in progress

  const int tid = threadIdx.x;
  const bool teamA = tid >= NC;
  const int cell = teamA ? tid - NC : tid;
  const int tx = cell % TX, ty = cell / TX;
  const int x0 = A.lo[0] + blockIdx.x * TX, y0 = A.lo[1] + blockIdx.y * TY;
  const int z0 = A.lo[2] + blockIdx.z * A.zchunk;
  const int z1 = min(z0 + A.zchunk, A.hi[2]);
  const int mx = A.mx;
  const long long mxy = A.mxy;
  int goff[NL];
#pragma unroll
  for (int k = 0; k < NL; ++k) {
    const int e = tid + k * NT;
    const int r = e / W, c = e - r * W;
    const int gx = min(x0 - 3 + c, mx - 1), gy = min(y0 - 3 + r, A.my - 1); // partial tiles: stay inside the allocation
    goff[k] = (e < PL) ? gy * mx + gx : -1;
  }
  auto load_plane = [&](int p, int slot) {
#pragma unroll
    for (int f = 0; f < kAcFields; ++f) {
      const T *src = A.in[f] + (long long)p * mxy;
      T *dst = ring + (f * NSLOT + slot) * PL + tid;
#pragma unroll
      for (int k = 0; k < NL; ++k) {
        if (goff[k] >= 0) cp_async<sizeof(T)>(dst + k * NT, src + goff[k]);
      }
    }
  };
  for (int p = z0 - 3; p <= z0 + 3; ++p) load_plane(p, p - z0 + 3);
  cp_async_commit();
  cp_async_wait_all();
  __syncthreads();

  const bool valid = (x0 + tx < A.hi[0]) && (y0 + ty < A.hi[1]);
  const int o0 = (ty + 3) * W + tx + 3;
  long long idx = (long long)z0 * mxy + (long long)(y0 + ty) * mx + (x0 + tx);

  for (int z = z0; z < z1; ++z, idx += mxy) {
    const int zi = z - z0;
    if (z + 1 < z1) load_plane(z + 4, (zi + 7) % NSLOT);
    cp_async_commit();
    team_plane<STEP, T, W, PL, NSLOT, NC, PACED>(A, ring, xb, zi, o0, cell, teamA, valid, idx);
    cp_async_wait_all();
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------- three teams
// With the ring fed by TMA the plane time is the instruction chain of the longest team (team U: 843 instructions against
// team A's 414, each warp at ~6 cycles per instruction: FP64 latency chains with ~3 warps per scheduler).  Three threads
// per cell cut the chain to ~450:
//   team T (thermodynamics)  lnrho, entropy        -> continuity and entropy equations
//   team V (velocity)        uux, uuy, uuz         -> momentum equation
//   team A (induction)       ax, ay, az            -> induction equation
// What one equation needs from another team's fields crosses through 14 words of shared memory per cell:
//   A -> V: j x B (3)   A -> T: |j|^2 (1)   T -> V: cs2, G = grad s / cp + grad lnrho (3), grad lnrho (3), 1 / rho   V -> T: div u, S : S
// ordered by three named barriers (the producer arrives, the consumers wait; no cycle: T publishes before it waits for V).
template <int STEP, typename T, int W, int PL, int NSLOT, int NC, bool PACED>
__device__ __forceinline__ void team3_plane(const AcArgs<T> &A, const T *ring, T *xb, int zi, int o0, int cell, int team, bool valid, long long idx) {
  const AcConst<T> &P = A.P;
  const T third = T(1.0) / T(3.0), half = T(0.5);
  const T *b[7]; // plane z-3+k of field 0 at this thread's cell
#pragma unroll
  for (int k = 0; k < 7; ++k) b[k] = ring + ((zi + k) % NSLOT) * PL + o0;
  auto atf = [&](int f) {
    return [&b, f](int dx, int dy, int dz) { return b[dz + 3][f * NSLOT * PL + dy * W + dx]; };
  };
  const T ux = b[3][UUX * NSLOT * PL], uy = b[3][UUY * NSLOT * PL], uz = b[3][UUZ * NSLOT * PL];
  enum { JXB = 0, J2 = 3, CS2 = 4, GG = 5, LG = 8, IRHO = 11, DIVU = 12, SSQ = 13 };
  constexpr int B_A = 1, B_T = 2, B_V = 3; // named barriers: "team X has published"
  if (team == 2) { // ---- team A: induction
    T pa[3] = {T(0), T(0), T(0)}, av[3] = {T(0), T(0), T(0)};
    T Bx = T(0), By = T(0), Bz = T(0), lax = T(0), lay = T(0), laz = T(0);
    if (valid) {
      if (STEP != 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) pa[i] = A.out[AX + i][idx];
      }
      T gx, gy, gz;
      {
        const Dv<T> d = derive<T, true, true, false, PACED>(atf(AX), P);
        av[0] = d.v;
        By = d.gz, Bz = -d.gy;
        lax = d.xx + d.yy + d.zz;
        gx = d.xx, gy = d.xy, gz = d.xz;
      }
      {
        const Dv<T> d = derive<T, true, false, true, PACED>(atf(AY), P);
        av[1] = d.v;
        Bx = -d.gz, Bz += d.gx;
        lay = d.xx + d.yy + d.zz;
        gx += d.xy, gy += d.yy, gz += d.yz;
      }
      {
        const Dv<T> d = derive<T, false, true, true, PACED>(atf(AZ), P);
        av[2] = d.v;
        Bx += d.gy, By -= d.gx;
        laz = d.xx + d.yy + d.zz;
        gx += d.xz, gy += d.yz, gz += d.zz;
      }
      const T jx = P.imu0 * (gx - lax), jy = P.imu0 * (gy - lay), jz = P.imu0 * (gz - laz);
      xb[(JXB + 0) * NC + cell] = jy * Bz - jz * By;
      xb[(JXB + 1) * NC + cell] = jz * Bx - jx * Bz;
      xb[(JXB + 2) * NC + cell] = jx * By - jy * Bx;
      xb[J2 * NC + cell] = jx * jx + jy * jy + jz * jz;
      __threadfence_block();
    }
    bar_arrive(B_A, 3 * NC); // (outside the branch: a barrier instruction is executed once per warp)
    if (valid) {
      const T indx = (uy * Bz - uz * By) + P.eta * lax;
      const T indy = (uz * Bx - ux * Bz) + P.eta * lay;
      const T indz = (ux * By - uy * Bx) + P.eta * laz;
      A.out[AX][idx] = rk3<STEP>(pa[0], av[0], indx, P.dt);
      A.out[AY][idx] = rk3<STEP>(pa[1], av[1], indy, P.dt);
      A.out[AZ][idx] = rk3<STEP>(pa[2], av[2], indz, P.dt);
    }
  } else if (team == 1) { // ---- team V: momentum
    T pu[3] = {T(0), T(0), T(0)};
    T madv[3] = {T(0), T(0), T(0)}, lu[3] = {T(0), T(0), T(0)}, gd[3] = {T(0), T(0), T(0)};
    T S00 = T(0), S11 = T(0), S22 = T(0), S01 = T(0), S02 = T(0), S12 = T(0);
    if (valid) {
      if (STEP != 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) pu[i] = A.out[UUX + i][idx];
      }
      T divu;
      {
        const Dv<T> d = derive<T, true, true, false, PACED>(atf(UUX), P);
        madv[0] = -(d.gx * ux + d.gy * uy + d.gz * uz);
        divu = d.gx;
        lu[0] = d.xx + d.yy + d.zz;
        gd[0] = d.xx, gd[1] = d.xy, gd[2] = d.xz;
        S00 = (T(2.0) * third) * d.gx, S11 = -third * d.gx, S22 = S11;
        S01 = half * d.gy, S02 = half * d.gz;
      }
      {
        const Dv<T> d = derive<T, true, false, true, PACED>(atf(UUY), P);
        madv[1] = -(d.gx * ux + d.gy * uy + d.gz * uz);
        divu += d.gy;
        lu[1] = d.xx + d.yy + d.zz;
        gd[0] += d.xy, gd[1] += d.yy, gd[2] += d.yz;
        S00 -= third * d.gy, S11 += (T(2.0) * third) * d.gy, S22 -= third * d.gy;
        S01 += half * d.gx, S12 = half * d.gz;
      }
      {
        const Dv<T> d = derive<T, false, true, true, PACED>(atf(UUZ), P);
        madv[2] = -(d.gx * ux + d.gy * uy + d.gz * uz);
        divu += d.gz;
        lu[2] = d.xx + d.yy + d.zz;
        gd[0] += d.xz, gd[1] += d.yz, gd[2] += d.zz;
        S00 -= third * d.gz, S11 -= third * d.gz, S22 += (T(2.0) * third) * d.gz;
        S02 += half * d.gx, S12 += half * d.gy;
      }
      xb[DIVU * NC + cell] = divu;
      xb[SSQ * NC + cell] = (S00 * S00 + S01 * S01 + S02 * S02) + (S01 * S01 + S11 * S11 + S12 * S12) + (S02 * S02 + S12 * S12 + S22 * S22);
      __threadfence_block();
    }
    bar_arrive(B_V, 2 * NC);
    bar_sync(B_T, 2 * NC);
    bar_sync(B_A, 3 * NC);
    if (valid) {
      const T cs2 = xb[CS2 * NC + cell], inv_rho = xb[IRHO * NC + cell];
      const T lg[3] = {xb[(LG + 0) * NC + cell], xb[(LG + 1) * NC + cell], xb[(LG + 2) * NC + cell]};
      const T Sg[3] = {S00 * lg[0] + S01 * lg[1] + S02 * lg[2], S01 * lg[0] + S11 * lg[1] + S12 * lg[2], S02 * lg[0] + S12 * lg[1] + S22 * lg[2]};
      const T uv[3] = {ux, uy, uz};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        T m = madv[i] - cs2 * xb[(GG + i) * NC + cell];
        m = m + inv_rho * xb[(JXB + i) * NC + cell];
        m = m + P.nu * ((lu[i] + third * gd[i]) + T(2.0) * Sg[i]);
        m = m + P.zeta * gd[i];
        A.out[UUX + i][idx] = rk3<STEP>(pu[i], uv[i], m, P.dt);
      }
    }
  } else { // ---- team T: continuity and entropy
    T pl = T(0), ps = T(0), lrv = T(0), sv = T(0), cont = T(0), entadv = T(0), heat_in = T(0), rho = T(1), earg = T(1);
    if (valid) {
      if (STEP != 0) pl = A.out[LNRHO][idx], ps = A.out[ENTROPY][idx];
      T llr, lg[3];
      {
        const Dv<T> d = derive<T, false, false, false, PACED>(atf(LNRHO), P);
        lrv = d.v;
        lg[0] = d.gx, lg[1] = d.gy, lg[2] = d.gz;
        llr = d.xx + d.yy + d.zz;
        cont = -(ux * d.gx + uy * d.gy + uz * d.gz);
      }
      rho = ac_exp(lrv);
      xb[IRHO * NC + cell] = T(1.0) / rho;
#pragma unroll
      for (int i = 0; i < 3; ++i) xb[(LG + i) * NC + cell] = lg[i];
      {
        const Dv<T> d = derive<T, false, false, false, PACED>(atf(ENTROPY), P);
        sv = d.v;
        const T ls = d.xx + d.yy + d.zz;
        const T sg[3] = {d.gx, d.gy, d.gz};
        const T first = P.gam * P.icp * ls + (P.gam - T(1.0)) * llr;
        T dot = T(0);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const T G = P.icp * sg[i] + lg[i];
          xb[(GG + i) * NC + cell] = G;
          const T s2 = P.gam * P.icp * sg[i] + (P.gam - T(1.0)) * lg[i];
          const T t3 = P.gam * G + (-lg[i]);
          dot += s2 * t3;
        }
        heat_in = first + dot;
        entadv = -(ux * d.gx + uy * d.gy + uz * d.gz);
        const T arg = P.gam * d.v * P.icp + (P.gam - T(1.0)) * (lrv - P.lnrho0);
        earg = ac_exp(arg);
        xb[CS2 * NC + cell] = P.cs2s * earg;
      }
      __threadfence_block();
    }
    bar_arrive(B_T, 2 * NC);
    bar_sync(B_V, 2 * NC);
    bar_sync(B_A, 3 * NC);
    if (valid) {
      const T divu = xb[DIVU * NC + cell], SS = xb[SSQ * NC + cell], j2 = xb[J2 * NC + cell];
      A.out[LNRHO][idx] = rk3<STEP>(pl, lrv, cont - divu, P.dt);
      // exp(lnT) = exp(lnT0) * exp(arg): the reference evaluates a third exp (rounding-level difference)
      const T inv_pT = T(1.0) / (rho * (P.elnT0 * earg));
      const T RHS = P.eta * P.mu0 * j2 + T(2.0) * rho * P.nu * SS + P.zeta * rho * divu * divu;
      const T chi = T(0.001) / (rho * P.cp);
      const T ent = entadv + inv_pT * RHS + P.cp * chi * heat_in;
      A.out[ENTROPY][idx] = rk3<STEP>(ps, sv, ent, P.dt);
    }
  }
}

// ---------------------------------------------------------------------------------------------- team kernel, TMA-fed ring
// The same two teams, but the ring is filled by the copy engine: one thread issues ONE cp.async.bulk.tensor per field and
// plane (a 24 x (TY+6) box of the halo'd tile, 3.4 KiB) instead of every thread issuing 16 eight-byte cp.async with their
// address arithmetic -- ncu on the cp.async version: 2.8 "MIO throttle" stalls per issued instruction, caused by the
// 192 LDGSTS per plane (8 cycles of the MIO / LSU path each) that all warps fire at the top of a plane, and a 289-instruction
// loop head per warp.  Completion is an mbarrier per ring slot (complete_tx::bytes); cells outside the allocation are
// zero-filled by the TMA unit, so partial tiles need no clamping.  FP64 only: the box's inner extent and every global
// stride must be multiples of 16 bytes (262 doubles per row are, 262 floats are not), and a box must START on a 16-byte
// address (measured in round 1), so the box begins at the even element at or before x0 - 3 and is 24 wide.
struct AcMaps {
  alignas(64) unsigned long long m[kAcFields][16]; // CUtensorMap x 8
};

__device__ __forceinline__ unsigned ac_smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ac_mbar_init(unsigned long long *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(ac_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void ac_mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(ac_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ac_mbar_wait(unsigned long long *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "AC_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra AC_DONE_%=;\n"
      "bra AC_WAIT_%=;\n"
      "AC_DONE_%=:\n"
      "}\n" ::"r"(ac_smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void ac_tma_load_3d(void *smem, const void *map, unsigned long long *bar, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(
                   ac_smem_u32(smem)),
               "l"(map), "r"(ac_smem_u32(bar)), "r"(x), "r"(y), "r"(z)
               : "memory");
}

template <int STEP, int TX, int TY, int NTEAM, bool PACED>
__global__ void __launch_bounds__(NTEAM *TX *TY, 1) ac_team_tma_kernel(const __grid_constant__ AcArgs<double> A, const __grid_constant__ AcMaps maps, int xshift) {
  using T = double;
  constexpr int NSLOT = 8, W = TX + 8, H = TY + 6, PL = W * H, NC = TX * TY;
  static_assert((PL * sizeof(T)) % 128 == 0, "every ring plane starts on a 128-byte boundary (TMA destination)");
  extern __shared__ __align__(1024) unsigned char ac_smem[];
  T *ring = reinterpret_cast<T *>(ac_smem);                                          // [field][slot][H][W]
  constexpr int NXB = NTEAM == 2 ? 4 : 14;
  T *xb = ring + kAcFields * NSLOT * PL;                                             // [NXB][NC]
  unsigned long long *bars = reinterpret_cast<unsigned long long *>(xb + NXB * NC); // [NSLOT]

  const int tid = threadIdx.x;
  const int team = tid / NC; // 2 teams: 0 = U, 1 = A; 3 teams: 0 = T, 1 = V, 2 = A
  const int cell = tid - team * NC;
  const int tx = cell % TX, ty = cell / TX;
  const int x0 = A.lo[0] + blockIdx.x * TX, y0 = A.lo[1] + blockIdx.y * TY;
  const int z0 = A.lo[2] + blockIdx.z * A.zchunk;
  const int z1 = min(z0 + A.zchunk, A.hi[2]);
  // tensor coordinate of allocation element x is x + xshift (the map's base is the allocation rounded down to 16 bytes);
  // the box starts at the even coordinate at or below that of x0 - 3
  const int bxs = (x0 - 3 + xshift) & ~1;
  const int dx0 = (x0 - 3 + xshift) - bxs; // 0 or 1: where allocation element x0 - 3 sits inside the box

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NSLOT; ++i) ac_mbar_init(&bars[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue_plane = [&](int p, int slot) { // one thread
    ac_mbar_expect_tx(&bars[slot], unsigned(kAcFields * PL * sizeof(T)));
#pragma unroll
    for (int f = 0; f < kAcFields; ++f) ac_tma_load_3d(ring + (f * NSLOT + slot) * PL, &maps.m[f][0], &bars[slot], bxs, y0 - 3, p);
  };
  if (tid == 0)
    for (int k = 0; k < 7; ++k) issue_plane(z0 - 3 + k, k);
  for (int k = 0; k < 7; ++k) ac_mbar_wait(&bars[k], 0);

  const bool valid = (x0 + tx < A.hi[0]) && (y0 + ty < A.hi[1]);
  const int o0 = (ty + 3) * W + tx + 3 + dx0;
  long long idx = (long long)z0 * A.mxy + (long long)(y0 + ty) * A.mx + (x0 + tx);
  for (int z = z0; z < z1; ++z, idx += A.mxy) {
    const int zi = z - z0;
    const bool more = z + 1 < z1;
    if (more && tid == 0) issue_plane(z + 4, (zi + 7) % NSLOT); // that slot held plane z - 4: nobody reads it any more
    if (NTEAM == 2) team_plane<STEP, T, W, PL, NSLOT, NC, PACED>(A, ring, xb, zi, o0, cell, team == 1, valid, idx);
    else team3_plane<STEP, T, W, PL, NSLOT, NC, PACED>(A, ring, xb, zi, o0, cell, team, valid, idx);
    if (more) ac_mbar_wait(&bars[(zi + 7) % NSLOT], unsigned((zi + 7) / NSLOT) & 1u);
    __syncthreads(); // everyone is done with plane z - 3 (and with xb) before the next iteration overwrites them
  }
}

template <int STEP, typename T, int TX, int TY> int launch_team(AcArgs<T> &A, cudaStream_t stream) {
  constexpr int NSLOT = 8;
  constexpr size_t smem = (size_t(kAcFields) * NSLOT * (TX + 6) * (TY + 6) + 4 * TX * TY) * sizeof(T);
  static unsigned long long configured = 0;
  static const bool paced = env_int("SB_AC_PACE", 1) != 0;
  auto kern = paced ? ac_team_kernel<STEP, T, TX, TY, NSLOT, true> : ac_team_kernel<STEP, T, TX, TY, NSLOT, false>;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  if (!(configured >> (dev & 63) & 1)) {
    if (cudaFuncSetAttribute(ac_team_kernel<STEP, T, TX, TY, NSLOT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) return -1;
    if (cudaFuncSetAttribute(ac_team_kernel<STEP, T, TX, TY, NSLOT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) return -1;
    configured |= 1ull << (dev & 63);
  }
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int ex = A.hi[0] - A.lo[0], ey = A.hi[1] - A.lo[1], ez = A.hi[2] - A.lo[2];
  const int gx = (ex + TX - 1) / TX, gy = (ey + TY - 1) / TY;
  int best_len = ez;
  long long best_cost = -1;
  for (int n = 1; n <= ez && n <= 64; ++n) { // see launch_tile
    const int len = (ez + n - 1) / n;
    const long long ctas = (long long)gx * gy * ((ez + len - 1) / len);
    const long long cost = ((ctas + sms - 1) / sms) * (len + 4);
    if (best_cost < 0 || cost < best_cost) best_cost = cost, best_len = len;
  }
  const int forced = env_int("SB_AC_ZCHUNK", 0);
  A.zchunk = forced > 0 ? (forced < ez ? forced : ez) : best_len;
  dim3 grid(gx, gy, (ez + A.zchunk - 1) / A.zchunk);
  kern<<<grid, 2 * TX * TY, smem, stream>>>(A);
  return 1;
}

int env_int(const char *name, int dflt) {
  const char *s = getenv(name);
  return (s && *s) ? atoi(s) : dflt;
}

template <int STEP, typename T, int TX, int TY, int NSLOT> int launch_tile(AcArgs<T> &A, cudaStream_t stream) {
  constexpr size_t smem = size_t(kAcFields) * NSLOT * (TX + 6) * (TY + 6) * sizeof(T);
  static unsigned long long configured = 0; // bit per device: the opt-in is per function and per context
  auto kern = ac_tile_kernel<STEP, T, TX, TY, NSLOT>;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  if (!(configured >> (dev & 63) & 1)) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) return -1;
    configured |= 1ull << (dev & 63);
  }
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int ex = A.hi[0] - A.lo[0], ey = A.hi[1] - A.lo[1], ez = A.hi[2] - A.lo[2];
  const int gx = (ex + TX - 1) / TX, gy = (ey + TY - 1) / TY;
  // z chunks: a chunk of `len` planes costs len + 7 plane times (ring warm-up); one CTA per SM, so pick the chunk
  // count that minimises (waves of CTAs) x (chunk cost) on this GPU
  int best_len = ez;
  long long best_cost = -1;
  for (int n = 1; n <= ez && n <= 64; ++n) {
    const int len = (ez + n - 1) / n;
    const long long ctas = (long long)gx * gy * ((ez + len - 1) / len);
    const long long cost = ((ctas + sms - 1) / sms) * (len + 7);
    if (best_cost < 0 || cost < best_cost) best_cost = cost, best_len = len;
  }
  const int forced = env_int("SB_AC_ZCHUNK", 0);
  A.zchunk = forced > 0 ? (forced < ez ? forced : ez) : best_len;
  dim3 grid(gx, gy, (ez + A.zchunk - 1) / A.zchunk);
  kern<<<grid, TX * TY, smem, stream>>>(A);
  return 1;
}

// tensor maps of the 8 input fields (cuTensorMapEncodeTiled through the runtime's driver entry point), cached by pointer:
// the driver alternates between two sets of buffers
typedef CUresult (*AcEncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static bool ac_field_map(const void *field, long long mx, long long my, long long mz, int bw, int bh, unsigned long long out[16]) {
  static AcEncodeTiledFn fn = []() -> AcEncodeTiledFn {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
      cudaGetLastError();
      return nullptr;
    }
    return reinterpret_cast<AcEncodeTiledFn>(p);
  }();
  if (!fn) return false;
  struct Key {
    const void *p;
    long long mx, my, mz;
    int bw, bh;
    bool operator<(const Key &o) const { return std::tie(p, mx, my, mz, bw, bh) < std::tie(o.p, o.mx, o.my, o.mz, o.bw, o.bh); }
  };
  static std::mutex mu;
  static std::map<Key, std::array<unsigned long long, 16>> cache;
  std::lock_guard<std::mutex> lk(mu);
  const Key key{field, mx, my, mz, bw, bh};
  auto it = cache.find(key);
  if (it == cache.end()) {
    const uintptr_t addr = reinterpret_cast<uintptr_t>(field);
    const unsigned shift = unsigned(addr & 15u) / 8u; // elements between the 16-byte aligned base and the allocation
    CUtensorMap m;
    const cuuint64_t dims[3] = {cuuint64_t(mx) + shift, cuuint64_t(my), cuuint64_t(mz)};
    const cuuint64_t strides[2] = {cuuint64_t(mx) * 8u, cuuint64_t(mx) * cuuint64_t(my) * 8u};
    const cuuint32_t box[3] = {cuuint32_t(bw), cuuint32_t(bh), 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    if (fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, reinterpret_cast<void *>(addr & ~uintptr_t(15)), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
    std::array<unsigned long long, 16> a;
    static_assert(sizeof(CUtensorMap) == 128, "CUtensorMap is 128 bytes");
    std::memcpy(a.data(), &m, 128);
    if (cache.size() > 256) cache.clear();
    it = cache.emplace(key, a).first;
  }
  std::memcpy(out, it->second.data(), 128);
  return true;
}

// returns 0 if the TMA-fed kernel does not apply to these buffers (the caller falls back to the cp.async-fed one)
template <int STEP, int TX, int TY, int NTEAM> int launch_team_tma(AcArgs<double> &A, long long mz, cudaStream_t stream) {
  constexpr int W = TX + 8, H = TY + 6;
  constexpr size_t smem = (size_t(kAcFields) * 8 * W * H + (NTEAM == 2 ? 4 : 14) * TX * TY) * sizeof(double) + 8 * sizeof(unsigned long long);
  if (A.mx % 2 != 0) return 0; // row stride must be a multiple of 16 bytes
  const unsigned phase = unsigned(reinterpret_cast<uintptr_t>(A.in[0]) & 15u);
  if (phase % 8 != 0) return 0;
  AcMaps maps;
  for (int f = 0; f < kAcFields; ++f) {
    if ((reinterpret_cast<uintptr_t>(A.in[f]) & 15u) != phase) return 0; // one box origin for all fields
    if (!ac_field_map(A.in[f], A.mx, A.my, mz, W, H, maps.m[f])) return 0;
  }
  static const bool paced = env_int("SB_AC_PACE", 1) != 0;
  auto kern = paced ? ac_team_tma_kernel<STEP, TX, TY, NTEAM, true> : ac_team_tma_kernel<STEP, TX, TY, NTEAM, false>;
  static unsigned long long configured = 0;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  if (!(configured >> (dev & 63) & 1)) {
    if (cudaFuncSetAttribute(ac_team_tma_kernel<STEP, TX, TY, NTEAM, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) return 0;
    if (cudaFuncSetAttribute(ac_team_tma_kernel<STEP, TX, TY, NTEAM, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)) != cudaSuccess) return 0;
    configured |= 1ull << (dev & 63);
  }
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int ex = A.hi[0] - A.lo[0], ey = A.hi[1] - A.lo[1], ez = A.hi[2] - A.lo[2];
  const int gx = (ex + TX - 1) / TX, gy = (ey + TY - 1) / TY;
  int best_len = ez;
  long long best_cost = -1;
  for (int n = 1; n <= ez && n <= 64; ++n) { // see launch_tile
    const int len = (ez + n - 1) / n;
    const long long ctas = (long long)gx * gy * ((ez + len - 1) / len);
    const long long cost = ((ctas + sms - 1) / sms) * (len + 3);
    if (best_cost < 0 || cost < best_cost) best_cost = cost, best_len = len;
  }
  const int forced = env_int("SB_AC_ZCHUNK", 0);
  A.zchunk = forced > 0 ? (forced < ez ? forced : ez) : best_len;
  dim3 grid(gx, gy, (ez + A.zchunk - 1) / A.zchunk);
  kern<<<grid, NTEAM * TX * TY, smem, stream>>>(A, maps, int(phase / 8));
  return 1;
}

template <int STEP, typename T> int launch_cell(AcArgs<T> &A, cudaStream_t stream) {
  const int ex = A.hi[0] - A.lo[0], ey = A.hi[1] - A.lo[1], ez = A.hi[2] - A.lo[2];
  int lgx = 0, lgy = 0;
  while ((1 << lgx) < ex && lgx < 5) ++lgx; // up to 32 lanes along x
  while ((1 << lgy) < ey && lgx + lgy < 7) ++lgy;
  if ((1 << (lgx + lgy)) < 128 && ez == 1) { /* flat box: waste is unavoidable */ }
  const int bz = 128 >> (lgx + lgy);
  dim3 grid((ex + (1 << lgx) - 1) >> lgx, (ey + (1 << lgy) - 1) >> lgy, (ez + bz - 1) / bz);
  ac_cell_kernel<STEP, T><<<grid, 128, 0, stream>>>(A, lgx, lgy);
  return 1;
}

template <int STEP, typename T> int launch_step(AcArgs<T> &A, long long mz, int variant, cudaStream_t stream) {
  const int ex = A.hi[0] - A.lo[0], ey = A.hi[1] - A.lo[1], ez = A.hi[2] - A.lo[2];
  // thick boxes: FP64 -> the TMA-fed two-team kernel, FP32 -> the tile kernel (the faster of the variants where they were
  // tuned, on a B200; not re-timed on the H100); thin boxes (exterior slabs) -> one thread per cell
  if (variant == AC_AUTO) variant = (ex >= 8 && ey >= 8 && ez >= 8) ? (sizeof(T) == 8 ? AC_TEAM : AC_TILE) : AC_CELL;
  if (variant == AC_CELL) return launch_cell<STEP>(A, stream);
  if (variant == AC_TEAM || variant == AC_TEAM_TMA || variant == AC_TEAM3_TMA) {
    if constexpr (sizeof(T) == 8) {
      if (variant != AC_TEAM || env_int("SB_AC_TMA", 1) != 0) {
        // two teams by default; SB_AC_TEAMS=3 or variant 5 = three teams
        const bool three = variant == AC_TEAM3_TMA || (variant == AC_TEAM && env_int("SB_AC_TEAMS", 2) == 3);
        const int n = three ? launch_team_tma<STEP, 16, 10, 3>(A, mz, stream) : launch_team_tma<STEP, 16, 12, 2>(A, mz, stream);
        if (n > 0) return n;
        if (variant != AC_TEAM) return -4; // asked for explicitly and not applicable
      }
      return launch_team<STEP, T, 16, 12>(A, stream);
    } else {
      if (variant != AC_TEAM) return -4;
      return launch_team<STEP, T, 32, 8>(A, stream);
    }
  }
  const int shape = env_int("SB_AC_SHAPE", 0);
  if constexpr (sizeof(T) == 8) {
    if (shape == 1) return launch_tile<STEP, T, 16, 16, 7>(A, stream);
    return launch_tile<STEP, T, 16, 14, 8>(A, stream);
  } else {
    // 32x8 tiles (256 threads) by default, SB_AC_SHAPE=1 for 32x16 (512 threads)
    if (shape == 1) return launch_tile<STEP, T, 32, 16, 8>(A, stream);
    return launch_tile<STEP, T, 32, 8, 8>(A, stream);
  }
}

template <typename T>
int launch_typed(int step, const AcFields &f, long long mx, long long my, long long mz, const int lo[3], const int hi[3], const AcParams &p,
                 int variant, cudaStream_t stream) {
  AcArgs<T> A;
  for (int i = 0; i < kAcFields; ++i) {
    A.in[i] = static_cast<const T *>(f.in[i]);
    A.out[i] = static_cast<T *>(f.out[i]);
  }
  A.mx = int(mx), A.my = int(my), A.mxy = mx * my;
  for (int k = 0; k < 3; ++k) A.lo[k] = lo[k], A.hi[k] = hi[k];
  A.zchunk = hi[2] - lo[2];
  A.P = make_const<T>(p);
  switch (step) {
  case 0: return launch_step<0>(A, mz, variant, stream);
  case 1: return launch_step<1>(A, mz, variant, stream);
  case 2: return launch_step<2>(A, mz, variant, stream);
  default: return -1;
  }
}

} // namespace

int launch_astaroth_substep(int step, const AcFields &f, int dtype_size, long long mx, long long my, long long mz, const int lo[3],
                            const int hi[3], const AcParams &p, int variant, cudaStream_t stream) {
  for (int k = 0; k < 3; ++k) {
    if (hi[k] <= lo[k]) return 0;
  }
  const long long m[3] = {mx, my, mz};
  for (int k = 0; k < 3; ++k) {
    if (lo[k] < 3 || hi[k] > m[k] - 3) return -2; // every cell needs three allocated neighbours on each side
  }
  if (mx * my >= (1ll << 31)) return -3; // in-plane offsets are 32-bit
  if (dtype_size == 8) return launch_typed<double>(step, f, mx, my, mz, lo, hi, p, variant, stream);
  if (dtype_size == 4) return launch_typed<float>(step, f, mx, my, mz, lo, hi, p, variant, stream);
  return -1;
}

} // namespace sb
