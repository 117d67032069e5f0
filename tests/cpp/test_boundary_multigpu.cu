// C++ API check of boundary conditions on non-periodic grids, on ALL visible GPUs -- 1 process x N GPUs, or one rank per
// GPU under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs than ranks; the verdict is all-reduced).
//  1. exchange: walls on some axes, a BC per quantity and wall face; after every exchange the WHOLE allocation of every
//     quantity must equal what the analytic field gives through the per-cell rule of include/stencil_b200.h.
//  2. FusedJacobi3d on a walled domain with ODD(0.25) must match, bit for bit, the same steps done by hand
//     (dd.exchange() then sb_jacobi3d over each compute region): the domain's BCs make it take the reference schedule.
// Build: make bin/test_boundary_multigpu      Run: bin/test_boundary_multigpu
#include <cstdio>
#include <cstring>
#include <vector>

#include "stencil/jacobi3d.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::BC;
using B = Topology::Boundary;

template <typename T> __host__ __device__ T field(int q, int64_t x, int64_t y, int64_t z, int rep) {
  return T((x * 7 + y * 131 + z * 1009 + q * 3 + rep * 17) % 8191);
}

template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, int q, int rep) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x) acc[Dim3(x, y, z)] = field<T>(q, x, y, z, rep);
}

struct Case {
  B bound[3];
  BC bc[3][6]; // per quantity (float, double, char) and face
};

static Dim3 g_grid; // compute size of the whole grid of the running case

// The expected value of allocation cell p (local coordinates) of quantity q; false if no rule fills it.
template <typename T>
static bool want(const Case &c, int q, const Dim3 &size, const Dim3 &org, const Radius &r, const Dim3 &p, int rep, T *out) {
  const int64_t gm[3] = {int64_t(r.x(-1)), int64_t(r.y(-1)), int64_t(r.z(-1))};
  const int64_t szv[3] = {size.x, size.y, size.z}, pv[3] = {p.x, p.y, p.z}, ov[3] = {org.x, org.y, org.z};
  int d[3];
  for (int a = 0; a < 3; ++a) d[a] = pv[a] < gm[a] ? -1 : (pv[a] >= gm[a] + szv[a] ? 1 : 0);
  if (!d[0] && !d[1] && !d[2]) {
    *out = field<T>(q, ov[0] + pv[0] - gm[0], ov[1] + pv[1] - gm[1], ov[2] + pv[2] - gm[2], rep);
    return true;
  }
  if (0 == r.dir(d[0], d[1], d[2])) return false;
  const int64_t grid[3] = {g_grid.x, g_grid.y, g_grid.z};
  int64_t g[3];
  bool wall[3], A[3], anyA = false, bare = false;
  for (int a = 0; a < 3; ++a) {
    g[a] = ov[a] + pv[a] - gm[a];
    wall[a] = d[a] && c.bound[a] == B::FIXED && (g[a] < 0 || g[a] >= grid[a]);
    A[a] = wall[a] && c.bc[q][2 * a + (d[a] > 0)].kind != BC::Kind::NONE;
    anyA = anyA || A[a];
    bare = bare || (wall[a] && !A[a]);
  }
  if (!anyA) {
    if (bare) {
      *out = T(0); // a wall ghost cell without a BC keeps what was there (zeroed before every round)
      return true;
    }
    for (int a = 0; a < 3; ++a) g[a] = ((g[a] % grid[a]) + grid[a]) % grid[a];
    *out = field<T>(q, g[0], g[1], g[2], rep);
    return true;
  }
  int64_t s[3];
  for (int a = 0; a < 3; ++a) s[a] = !A[a] ? pv[a] : (d[a] < 0 ? 2 * gm[a] - 1 - pv[a] : 2 * (gm[a] + szv[a]) - 1 - pv[a]);
  T v;
  if (!want<T>(c, q, size, org, r, Dim3(s[0], s[1], s[2]), rep, &v)) return false;
  for (int a = 0; a < 3; ++a) {
    if (!A[a]) continue;
    const BC &bc = c.bc[q][2 * a + (d[a] > 0)];
    if (bc.kind == BC::Kind::VALUE) v = T(bc.value);
    if (bc.kind == BC::Kind::ODD) v = T(T(2) * T(bc.value)) - v;
  }
  *out = v;
  return true;
}

template <typename T> static long check_quantity(const Case &c, LocalDomain &d, size_t q, const Radius &radius, int rep) {
  const std::vector<unsigned char> raw = d.quantity_to_host(q);
  const Dim3 rs = d.raw_size();
  const T *v = reinterpret_cast<const T *>(raw.data());
  long bad = 0;
  for (int64_t z = 0; z < rs.z; ++z)
    for (int64_t y = 0; y < rs.y; ++y)
      for (int64_t x = 0; x < rs.x; ++x) {
        T w;
        if (!want<T>(c, int(q), d.size(), d.origin(), radius, Dim3(x, y, z), rep, &w)) continue;
        const T got = v[(z * rs.y + y) * rs.x + x];
        if (std::memcmp(&got, &w, sizeof(T)) != 0) {
          if (bad < 5)
            std::fprintf(stderr, "MISMATCH gpu%d q%zu at alloc(%ld,%ld,%ld): got %g want %g\n", d.gpu(), q, long(x), long(y), long(z), double(got), double(w));
          ++bad;
        }
      }
  return bad;
}

static long run_case(size_t X, size_t Y, size_t Z, const Radius &radius, const Case &c, const char *name) {
  DistributedDomain dd(X, Y, Z);
  g_grid = Dim3(X, Y, Z);
  dd.set_radius(radius);
  dd.set_boundary(c.bound[0], c.bound[1], c.bound[2]);
  auto h0 = dd.add_data<float>("f");
  auto h1 = dd.add_data<double>("d");
  auto h2 = dd.add_data<char>("c");
  for (int f = 0; f < 6; ++f) {
    const Dim3 face(f / 2 == 0 ? (f % 2 ? 1 : -1) : 0, f / 2 == 1 ? (f % 2 ? 1 : -1) : 0, f / 2 == 2 ? (f % 2 ? 1 : -1) : 0);
    if (c.bound[f / 2] != B::FIXED) continue;
    dd.set_boundary_condition(h0, face, c.bc[0][f]);
    dd.set_boundary_condition(h1, face, c.bc[1][f]);
    dd.set_boundary_condition(h2, face, c.bc[2][f]);
  }
  dd.realize();
  long bad = 0;
  for (int rep = 0; rep < 3; ++rep) {
    for (auto &d : dd.domains()) {
      d.set_device();
      const Dim3 rs = d.raw_size();
      for (size_t q = 0; q < 3; ++q) CUDA_RUNTIME(cudaMemset(d.curr_data(q).ptr, 0, size_t(rs.x * rs.y * rs.z) * d.elem_size(q)));
      const Rect3 reg = d.get_compute_region();
      fill<float><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h0), reg, 0, rep);
      fill<double><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h1), reg, 1, rep);
      fill<char><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h2), reg, 2, rep);
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
    MPI_Barrier(MPI_COMM_WORLD);
    dd.exchange();
    for (auto &d : dd.domains()) {
      bad += check_quantity<float>(c, d, 0, radius, rep);
      bad += check_quantity<double>(c, d, 1, radius, rep);
      bad += check_quantity<char>(c, d, 2, radius, rep);
    }
    MPI_Barrier(MPI_COMM_WORLD);
    dd.swap();
  }
  long long all = bad;
  MPI_Allreduce(MPI_IN_PLACE, &all, 1, MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
  if (0 == mpi::world_rank())
    std::printf("%-36s %zux%zux%zu on %d rank(s) x %zu subdomain(s): %s (%lld mismatches)\n", name, X, Y, Z, mpi::world_size(), dd.domains().size(),
                all ? "FAIL" : "ok", all);
  return long(all);
}

// FusedJacobi3d (which must fall back to the reference schedule) against dd.exchange() + sb_jacobi3d by hand
static long run_jacobi(size_t n) {
  auto make = [&](DistributedDomain &dd) {
    dd.set_radius(Radius::face_edge_corner(1, 0, 0));
    dd.set_boundary(B::FIXED);
    auto h = dd.add_data<double>("d");
    for (const Dim3 &f : {Dim3(-1, 0, 0), Dim3(1, 0, 0), Dim3(0, -1, 0), Dim3(0, 1, 0), Dim3(0, 0, -1), Dim3(0, 0, 1)})
      dd.set_boundary_condition(h, f, BC::ODD(0.25));
    dd.realize();
    return h;
  };
  DistributedDomain a(n, n, n), b(n, n, n);
  make(a);
  auto hb = make(b);
  stencil::FusedJacobi3d jac(a, DataHandle<double>(0));
  jac.init(0.5);
  const Rect3 whole = b.get_compute_region();
  int64_t clo[3] = {whole.lo.x, whole.lo.y, whole.lo.z}, chi[3] = {whole.hi.x, whole.hi.y, whole.hi.z};
  for (auto &d : b.domains()) {
    const Rect3 cr = d.get_compute_region();
    const Dim3 ao = d.origin() - Dim3(1, 1, 1);
    int64_t acc[3] = {ao.x, ao.y, ao.z}, lo[3] = {cr.lo.x, cr.lo.y, cr.lo.z}, hi[3] = {cr.hi.x, cr.hi.y, cr.hi.z};
    const cudaPitchedPtr p = d.curr_data(hb.id());
    if (SB_OK != sb_fill(sb_pitched{p.ptr, int64_t(p.pitch), int64_t(p.ysize)}, 8, acc, lo, hi, 0.5, nullptr)) LOG_FATAL(sb_last_error());
  }
  for (auto &d : b.domains()) {
    d.set_device();
    CUDA_RUNTIME(cudaDeviceSynchronize());
  }
  for (int it = 0; it < 5; ++it) {
    jac.step();
    b.exchange();
    for (auto &d : b.domains()) {
      const Rect3 cr = d.get_compute_region();
      const Dim3 ao = d.origin() - Dim3(1, 1, 1);
      int64_t acc[3] = {ao.x, ao.y, ao.z}, lo[3] = {cr.lo.x, cr.lo.y, cr.lo.z}, hi[3] = {cr.hi.x, cr.hi.y, cr.hi.z};
      const cudaPitchedPtr s = d.curr_data(hb.id()), t = d.next_data(hb.id());
      if (SB_OK != sb_jacobi3d(sb_pitched{t.ptr, int64_t(t.pitch), int64_t(t.ysize)}, sb_pitched{s.ptr, int64_t(s.pitch), int64_t(s.ysize)}, 8, acc, lo, hi, clo,
                               chi, nullptr))
        LOG_FATAL(sb_last_error());
    }
    for (auto &d : b.domains()) {
      d.set_device();
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
    MPI_Barrier(MPI_COMM_WORLD);
    b.swap();
  }
  jac.synchronize();
  MPI_Barrier(MPI_COMM_WORLD);
  long bad = 0;
  if (jac.fused()) { // a domain with BCs must not run the fused kernel
    std::fprintf(stderr, "rank %d: FusedJacobi3d chose the fused kernel on a domain with boundary conditions\n", mpi::world_rank());
    ++bad;
  }
  for (size_t di = 0; di < a.domains().size(); ++di) {
    const std::vector<unsigned char> x = a.domains()[di].interior_to_host(0), y = b.domains()[di].interior_to_host(0);
    const double *xv = reinterpret_cast<const double *>(x.data()), *yv = reinterpret_cast<const double *>(y.data());
    const Dim3 sz = a.domains()[di].size();
    size_t diff = 0;
    double lo = 1e9, hi = -1e9;
    for (size_t i = 0; i < x.size() / 8; ++i) {
      if (std::memcmp(xv + i, yv + i, 8) != 0 && diff++ == 0)
        std::fprintf(stderr, "rank %d domain %zu: first difference at compute cell (%ld,%ld,%ld): %.17g vs %.17g by hand\n", mpi::world_rank(), di,
                     long(i % sz.x), long((i / sz.x) % sz.y), long(i / (sz.x * sz.y)), xv[i], yv[i]);
      lo = xv[i] < lo ? xv[i] : lo;
      hi = xv[i] > hi ? xv[i] : hi;
    }
    if (diff) std::fprintf(stderr, "rank %d domain %zu: %zu of %zu cells differ\n", mpi::world_rank(), di, diff, x.size() / 8);
    bad += diff ? 1 : 0;
    if (!(hi > lo)) ++bad; // the field must have evolved
  }
  long long all = bad;
  MPI_Allreduce(MPI_IN_PLACE, &all, 1, MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
  if (0 == mpi::world_rank())
    std::printf("%-36s %zu^3 on %d rank(s): %s\n", "FusedJacobi3d walls ODD(0.25) x5", n, mpi::world_size(), all ? "FAIL" : "ok");
  return long(all);
}

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  long bad = 0;
  Case all{};
  for (int a = 0; a < 3; ++a) all.bound[a] = B::FIXED;
  const BC kinds[5] = {BC::VALUE(1.5), BC::EVEN(), BC::ODD(0.5), BC::NONE(), BC::ODD(-2.25)};
  for (int f = 0; f < 6; ++f) {
    all.bc[0][f] = kinds[f % 5];
    all.bc[1][f] = kinds[(f + 2) % 5];
    all.bc[2][f] = (f % 3) ? BC::EVEN() : BC::NONE();
  }
  Case channel = all;
  channel.bound[0] = channel.bound[1] = B::PERIODIC;
  Case xwalls = all;
  xwalls.bound[1] = xwalls.bound[2] = B::PERIODIC;
  bad += run_case(40, 36, 44, Radius::constant(2), all, "walls on x, y, z; r=2");
  bad += run_case(37, 29, 41, Radius::face_edge_corner(2, 1, 0), channel, "channel (walls on z); faces 2, edges 1");
  bad += run_case(48, 40, 32, Radius::constant(1), xwalls, "walls on x; r=1");
  bad += run_jacobi(64); // on 2 or 4 ranks the subdomains are 32 cells wide: less than one 64-cell FP64 strip

  if (0 == mpi::world_rank()) std::printf(bad ? "FAILED\n" : "ALL OK\n");
  MPI_Finalize();
  return bad ? 1 : 0;
}
