// C++ API check of the multigrid transfers (DistributedDomain::restrict_to / prolong_from) inside V(2,2) cycles -- one
// process with N subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are
// fewer GPUs than ranks).
//   bin/test_mg_multigpu --single N OUT      one process, N subdomains: the bits must equal a one-subdomain run's, and are
//                                           written to OUT
//   bin/sb_mpirun -n N bin/test_mg_multigpu --expect OUT
//                                           one subdomain per rank: every rank's bits must equal OUT's
// Runs, in double and float, three V(2,2) cycles over 4 levels (32^3 .. 4^3) of -lap u = f with ODD(0) walls: red-black
// Gauss-Seidel (LinearStencil::relax(1) in coloured applies), the residual as one apply, restriction into the coarser f,
// u = 0 * f there, 30 sweeps on the coarsest level, and the in-place correction u <- u + P e.  Every step is
// partition-independent, so the bits after every cycle are the same for every partition and rank count; the residual
// must also fall by 10^2 over the three cycles.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <vector>

#include "stencil/linear_stencil.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::LinearStencil;
using stencil::Source;

// a right-hand side in [-4, 4)
template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, bool zero) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x)
        acc[Dim3(x, y, z)] = zero ? T(0) : T(double((x * 7 + y * 131 + z * 1009) % 8191) * 0.0009765625 - 4.0);
}

template <typename T> struct Level {
  std::unique_ptr<DistributedDomain> dd;
  DataHandle<T> u{0}, f{1}, r{2};
  LinearStencil gs, res, zero;

  Level(int64_t n, double h, const std::vector<int> &gpus) : dd(new DistributedDomain(n, n, n)) {
    dd->set_gpus(gpus);
    dd->set_radius(Radius::constant(1));
    u = dd->add_data<T>("u");
    f = dd->add_data<T>("f");
    r = dd->add_data<T>("r");
    dd->set_boundary(Topology::Boundary::FIXED);
    for (int a = 0; a < 3; ++a)
      for (int s = -1; s <= 1; s += 2) dd->set_boundary_condition(u, Dim3(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0), stencil::BC::ODD(0.0));
    dd->realize();
    // A = -lap; the Gauss-Seidel update, the residual f - A u and u = 0 * f
    const LinearStencil lap = LinearStencil::laplacian(2, h, h, h);
    LinearStencil A;
    for (const sb_stencil_term &t : lap.terms()) A.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight);
    gs = A.relax(1.0);
    res.add(Source::aux, 0, 0, 0, 1.0);
    for (const sb_stencil_term &t : A.terms()) res.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight);
    zero.add(Source::src, 0, 0, 0, 0.0);
  }
  void smooth(int sweeps) {
    for (int k = 0; k < sweeps; ++k)
      for (int c = 0; c < 2; ++c) dd->apply(gs, stencil::curr(u), u, stencil::curr(f), stencil::Colour{2, c});
  }
  double residual_norm() {
    dd->apply(res, stencil::curr(r), u, stencil::curr(f));
    return std::sqrt(dd->reduce(r, stencil::Which::curr, stencil::Sum::exact).sumsq);
  }
};

template <typename T> void vcycle(std::vector<std::unique_ptr<Level<T>>> &lv, size_t l) {
  Level<T> &L = *lv[l];
  if (l + 1 == lv.size()) {
    L.smooth(30);
    return;
  }
  L.smooth(2);
  L.dd->apply(L.res, stencil::curr(L.r), L.u, stencil::curr(L.f));
  Level<T> &C = *lv[l + 1];
  L.dd->restrict_to(*C.dd, stencil::curr(C.f), stencil::curr(L.r));
  C.dd->apply(C.zero, stencil::curr(C.u), C.f, false);
  vcycle(lv, l + 1);
  L.dd->prolong_from(*C.dd, stencil::curr(L.u), stencil::curr(C.u), stencil::curr(L.u));
  L.smooth(2);
}

template <typename T> std::vector<T> gather(DistributedDomain &dd, size_t q, int64_t n) {
  std::vector<T> out(size_t(n * n * n), T(0));
  for (LocalDomain &d : dd.domains()) {
    const Dim3 rs = d.raw_size(), sz = d.size(), o = d.origin();
    std::vector<T> a(size_t(rs.x * rs.y * rs.z));
    d.set_device();
    CUDA_RUNTIME(cudaMemcpy(a.data(), d.curr_data(q).ptr, a.size() * sizeof(T), cudaMemcpyDeviceToHost));
    for (int64_t z = 0; z < sz.z; ++z)
      for (int64_t y = 0; y < sz.y; ++y)
        for (int64_t x = 0; x < sz.x; ++x) out[size_t(((o.z + z) * n + o.y + y) * n + o.x + x)] = a[size_t(((z + 1) * rs.y + y + 1) * rs.x + x + 1)];
  }
  // every rank contributes its subdomains; the cells are disjoint, so a sum of zero-initialised 8-byte words merges them
  if (mpi::world_size() > 1) {
    std::vector<T> all(out.size());
    MPI_Allreduce(out.data(), all.data(), int(out.size() * sizeof(T) / 8), MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
    out.swap(all);
  }
  return out;
}

template <typename T> static std::string hexsum(const std::vector<T> &v) {
  uint64_t h = 1469598103934665603ull; // FNV-1a of the bits
  const unsigned char *b = reinterpret_cast<const unsigned char *>(v.data());
  for (size_t i = 0; i < v.size() * sizeof(T); ++i) h = (h ^ b[i]) * 1099511628211ull;
  char buf[32];
  std::snprintf(buf, sizeof(buf), "%016llx", (unsigned long long)h);
  return buf;
}

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits) {
  const int64_t n = 32;
  std::vector<std::unique_ptr<Level<T>>> lv;
  for (int l = 0; l < 4; ++l) lv.emplace_back(new Level<T>(n >> l, double(1 << l) / double(n), gpus));
  for (auto &L : lv)
    for (auto &d : L->dd->domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(L->u), d.get_compute_region(), true);
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(L->f), d.get_compute_region(), L.get() != lv[0].get());
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
  long bad = 0;
  const double r0 = lv[0]->residual_norm();
  for (int cyc = 0; cyc < 3; ++cyc) {
    vcycle(lv, 0);
    bits.push_back(hexsum(gather<T>(*lv[0]->dd, lv[0]->u.id(), n)));
  }
  const double r3 = lv[0]->residual_norm();
  if (!(r3 < 1e-2 * r0)) {
    if (0 == mpi::world_rank()) std::fprintf(stderr, "%zu-byte elements: residual %g -> %g after 3 cycles\n", sizeof(T), r0, r3);
    ++bad;
  }
  return bad;
}

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s --single N OUT | --expect OUT\n", argv[0]);
    return 2;
  }
  const bool single = std::string(argv[1]) == "--single";
  int ndev = 0;
  CUDA_RUNTIME(cudaGetDeviceCount(&ndev));
  std::vector<int> gpus = single ? std::vector<int>(size_t(std::atoi(argv[2])), 0) : std::vector<int>{mpi::world_rank() % ndev};
  const size_t nsub = single ? gpus.size() : size_t(mpi::world_size());
  std::vector<std::string> bits;
  long bad = run<double>(gpus, bits) + run<float>(gpus, bits);
  if (single) {
    std::vector<std::string> one;
    bad += run<double>({0}, one) + run<float>({0}, one);
    if (one != bits) {
      std::fprintf(stderr, "%zu subdomains: result bits differ from the one-subdomain run\n", nsub);
      ++bad;
    }
    std::ofstream f(argv[3]);
    for (const std::string &b : bits) f << b << "\n";
  } else {
    std::ifstream f(argv[2]);
    std::vector<std::string> want;
    for (std::string line; std::getline(f, line);) want.push_back(line);
    if (want != bits) {
      std::fprintf(stderr, "rank %d: result bits differ from the one-process run of the same partition\n", mpi::world_rank());
      ++bad;
    }
  }
  long long all = bad;
  MPI_Allreduce(MPI_IN_PLACE, &all, 1, MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
  if (0 == mpi::world_rank()) {
    std::printf("multigrid V-cycles through DistributedDomain::restrict_to / prolong_from, %zu subdomain(s) on %d rank(s): %s\n", nsub,
                mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
