// C++ API check of stencil::Multigrid<T> (include/stencil/multigrid.hpp) -- one process with N subdomains on GPU 0, or
// one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs than ranks).
//   bin/test_multigrid_multigpu --single N OUT      one process, N subdomains: the bits must equal a one-subdomain
//                                                  run's, and are written to OUT
//   bin/sb_mpirun -n N bin/test_multigrid_multigpu --expect OUT
//                                                  one subdomain per rank: every rank's bits must equal OUT's
//   bin/test_multigrid_multigpu --time N C         one GPU: C queued V(2,2) cycles of N^3 FP64 ODD(c) Poisson down to
//                                                  4^3 (30 coarsest sweeps) after a warm-up cycle; one JSON line with
//                                                  the wall time of each cycle and the residual after it
// Runs, in double and float, three queued V(2,2) cycles over 4 levels (32^3 .. 4^3) of -lap u = f with ODD(c) walls (a
// different c on each face), and checks, in the one-process mode, that the queued cycle gives the bits of the same
// cycle built from the public synchronising calls (restrict_to with the residual op, a cleared coarse u,
// prolong_from).  The residual must fall by 10^2 over the three cycles.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <vector>

#include "stencil/linear_stencil.hpp"
#include "stencil/multigrid.hpp"
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

const double WALL[6] = {0.0, 0.25, -0.5, 1.0, 0.125, -1.0};

LinearStencil A_at(int l, int64_t n) {
  const double h = double(1 << l) / double(n);
  const LinearStencil lap = LinearStencil::laplacian(2, h, h, h);
  LinearStencil A;
  for (const sb_stencil_term &t : lap.terms()) A.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight);
  return A;
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

template <typename T> struct Problem {
  std::unique_ptr<DistributedDomain> dd;
  DataHandle<T> u{0}, f{1}, r{2};
  std::unique_ptr<stencil::Multigrid<T>> mg;
  Problem(int64_t n, const std::vector<int> &gpus, int levels = 4) : dd(new DistributedDomain(n, n, n)) {
    dd->set_gpus(gpus);
    dd->set_radius(Radius::constant(1));
    u = dd->add_data<T>("u");
    f = dd->add_data<T>("f");
    r = dd->add_data<T>("r");
    dd->set_boundary(Topology::Boundary::FIXED);
    for (int a = 0, k = 0; a < 3; ++a)
      for (int s = -1; s <= 1; s += 2, ++k)
        dd->set_boundary_condition(u, Dim3(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0), stencil::BC::ODD(WALL[k]));
    dd->realize();
    for (auto &d : dd->domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(u), d.get_compute_region(), true);
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(f), d.get_compute_region(), false);
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
    mg.reset(new stencil::Multigrid<T>(*dd, u, f, r, [n](int l) { return A_at(l, n); }, 2, 2, 30, levels));
  }
  ~Problem() {
    mg.reset();
    dd.reset();
  }
};

// the same cycle from public synchronising calls, on a second problem's domains (levels built by hand)
template <typename T> struct Manual {
  struct Level {
    std::unique_ptr<DistributedDomain> dd;
    DataHandle<T> u{0}, f{1};
    LinearStencil gs, res;
  };
  Problem<T> &P;
  std::vector<Level> lv;
  Manual(Problem<T> &p, int64_t n, const std::vector<int> &gpus) : P(p) {
    for (int l = 1; l < 4; ++l) {
      Level L;
      const int64_t m = n >> l;
      L.dd.reset(new DistributedDomain(m, m, m));
      L.dd->set_gpus(gpus);
      L.dd->set_radius(Radius::constant(1));
      L.u = L.dd->template add_data<T>("u");
      L.f = L.dd->template add_data<T>("f");
      L.dd->set_boundary(Topology::Boundary::FIXED);
      for (int a = 0; a < 3; ++a)
        for (int s = -1; s <= 1; s += 2) L.dd->set_boundary_condition(L.u, Dim3(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0), stencil::BC::ODD(0.0));
      L.dd->realize();
      lv.push_back(std::move(L));
    }
  }
  LinearStencil gs(int l, int64_t n) { return A_at(l, n).relax(1.0); }
  LinearStencil res(int l, int64_t n) {
    const LinearStencil A = A_at(l, n);
    LinearStencil r;
    r.add(Source::aux, 0, 0, 0, 1.0);
    for (const sb_stencil_term &t : A.terms()) r.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight);
    return r;
  }
  void smooth(DistributedDomain &dd, DataHandle<T> u, DataHandle<T> f, const LinearStencil &g, int k) {
    for (int i = 0; i < k; ++i)
      for (int c = 0; c < 2; ++c) dd.apply(g, stencil::curr(u), u, stencil::curr(f), stencil::Colour{2, c});
  }
  void cycle(int l, int64_t n) {
    DistributedDomain &dd = l == 0 ? *P.dd : *lv[size_t(l - 1)].dd;
    const DataHandle<T> u = l == 0 ? P.u : lv[size_t(l - 1)].u, f = l == 0 ? P.f : lv[size_t(l - 1)].f;
    if (l == 3) {
      smooth(dd, u, f, gs(l, n), 30);
      return;
    }
    smooth(dd, u, f, gs(l, n), 2);
    Level &C = lv[size_t(l)];
    dd.restrict_to(*C.dd, stencil::curr(C.f), res(l, n), u, stencil::curr(f));
    for (auto &d : C.dd->domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(C.u), d.get_compute_region(), true);
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
    cycle(l + 1, n);
    dd.prolong_from(*C.dd, stencil::curr(u), stencil::curr(C.u), stencil::curr(u));
    smooth(dd, u, f, gs(l, n), 2);
  }
};

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits, bool manual) {
  const int64_t n = 32;
  long bad = 0;
  Problem<T> P(n, gpus);
  if (P.mg->num_levels() != 4 || P.mg->colours() != 2) {
    std::fprintf(stderr, "%zu levels, %d colours\n", P.mg->num_levels(), P.mg->colours());
    ++bad;
  }
  std::unique_ptr<Problem<T>> Q;
  std::unique_ptr<Manual<T>> M;
  if (manual) {
    Q.reset(new Problem<T>(n, gpus));
    M.reset(new Manual<T>(*Q, n, gpus));
  }
  const double r0 = P.mg->residual_norm();
  for (int cyc = 0; cyc < 3; ++cyc) {
    P.mg->cycle();
    const std::vector<T> got = gather<T>(*P.dd, P.u.id(), n);
    bits.push_back(hexsum(got));
    if (manual) {
      M->cycle(0, n);
      if (hexsum(gather<T>(*Q->dd, Q->u.id(), n)) != bits.back()) {
        std::fprintf(stderr, "%zu-byte elements, cycle %d: the queued cycle differs from the public calls\n", sizeof(T), cyc);
        ++bad;
      }
    }
  }
  const double r3 = P.mg->residual_norm();
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
  if (std::string(argv[1]) == "--time" && argc >= 4) {
    const int64_t n = std::atoll(argv[2]);
    const int cycles = std::atoi(argv[3]);
    Problem<double> P(n, {0}, int(std::log2(double(n))) - 1);
    P.mg->cycle(); // warm-up: plans, events, first launches
    for (auto &d : P.dd->domains()) {
      d.set_device();
      fill<double><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(P.u), d.get_compute_region(), true);
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
    std::printf("{\"workload\": \"%lld^3 FP64 ODD(c) Poisson, V(2,2) to 4^3, 30 coarsest sweeps: stencil::Multigrid<double>::cycle()\", \"ms_per_cycle\": [",
                (long long)n);
    std::vector<double> res;
    for (int k = 0; k < cycles; ++k) {
      const auto t0 = std::chrono::steady_clock::now();
      P.mg->cycle();
      const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      std::printf("%s%.2f", k ? ", " : "", ms);
      res.push_back(P.mg->residual_norm());
    }
    std::printf("], \"residual\": [");
    for (size_t k = 0; k < res.size(); ++k) std::printf("%s%.4g", k ? ", " : "", res[k]);
    std::printf("]}\n");
    MPI_Finalize();
    return 0;
  }
  const bool single = std::string(argv[1]) == "--single";
  int ndev = 0;
  CUDA_RUNTIME(cudaGetDeviceCount(&ndev));
  std::vector<int> gpus = single ? std::vector<int>(size_t(std::atoi(argv[2])), 0) : std::vector<int>{mpi::world_rank() % ndev};
  const size_t nsub = single ? gpus.size() : size_t(mpi::world_size());
  std::vector<std::string> bits;
  long bad = run<double>(gpus, bits, single) + run<float>(gpus, bits, single);
  if (single) {
    std::vector<std::string> one;
    bad += run<double>({0}, one, false) + run<float>({0}, one, false);
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
    std::printf("stencil::Multigrid queued V-cycles, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
