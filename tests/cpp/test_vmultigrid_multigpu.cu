// C++ API check of stencil::Multigrid<T> with coefficient fields (include/stencil/multigrid.hpp, DESIGN.md section
// 2.12) -- one process with N subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs
// when there are fewer GPUs than ranks).
//   bin/test_vmultigrid_multigpu --single N OUT     one process, N subdomains: the bits must equal a one-subdomain
//                                                  run's, and are written to OUT
//   bin/sb_mpirun -n N bin/test_vmultigrid_multigpu --expect OUT
//                                                  one subdomain per rank: every rank's bits must equal OUT's
//   bin/test_vmultigrid_multigpu --time N C         one GPU: C queued V(2,2) cycles of N^3 FP64 -div(kappa grad u) = f
//                                                  (smooth kappa, ODD(0) walls) down to 4^3 after a warm-up cycle, then
//                                                  as many constant-coefficient -lap u = f cycles; one JSON line each
// Runs, in double and float, three queued V(2,2) cycles over 4 levels (32^3 .. 4^3) of -div(kappa grad u) + sigma u = f,
// kappa smooth on faces (EVEN walls), sigma a cell field (VALUE walls), u with ODD(c) walls (a different c on each
// face), then update_coefficients() after kappa is scaled and solve().  In the one-process mode it checks that the
// queued cycle gives the bits of the same cycle built from the public synchronising calls (relax, restrict_to with the
// coefficient residual, a cleared coarse u, prolong_from; the coarse fields by the public face and cell restrictions).
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

// what: 0 zero, 1 a right-hand side in [-4, 4), 2 sigma in [0.5, 2), 3 + a kappa on the faces normal to axis a, times s
template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, int what, double n, double s) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x) {
        double v = 0.0;
        if (what == 1) v = double((x * 7 + y * 131 + z * 1009) % 8191) * 0.0009765625 - 4.0;
        if (what == 2) v = 0.5 + double((x * 13 + y * 29 + z * 71) % 97) / 64.0;
        if (what >= 3) {
          const int a = what - 3;
          const double p[3] = {(double(x) + (a == 0 ? 0.0 : 0.5)) / n, (double(y) + (a == 1 ? 0.0 : 0.5)) / n, (double(z) + (a == 2 ? 0.0 : 0.5)) / n};
          v = s * std::exp(0.5 * std::sin(6.283185307179586 * p[0]) * std::sin(6.283185307179586 * p[1]) * std::sin(6.283185307179586 * p[2]));
        }
        acc[Dim3(x, y, z)] = T(v);
      }
}

const double WALL[6] = {0.0, 0.25, -0.5, 1.0, 0.125, -1.0};
const std::vector<std::string> KINDS = {"x", "y", "z", "cell"};

// -div(kappa grad u) (+ sigma u, field 3)
LinearStencil A_at(int l, int64_t n, bool sigma) {
  const double h = double(1 << l) / double(n);
  LinearStencil A = LinearStencil::div_grad(h, h, h).scaled(-1.0);
  if (sigma) A.add(Source::src, 0, 0, 0, 1.0, 3, 0, 0, 0);
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
  if (mpi::world_size() > 1) { // disjoint cells: a sum of zero-initialised 8-byte words merges them
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

template <typename T> void fill_q(DistributedDomain &dd, DataHandle<T> q, int what, int64_t n, double s = 1.0) {
  for (auto &d : dd.domains()) {
    d.set_device();
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(q), d.get_compute_region(), what, double(n), s);
    CUDA_RUNTIME(cudaDeviceSynchronize());
  }
}

template <typename T> struct Problem {
  std::unique_ptr<DistributedDomain> dd;
  DataHandle<T> u{0}, f{1}, r{2};
  std::vector<DataHandle<T>> k;
  std::unique_ptr<stencil::Multigrid<T>> mg;
  // sigma: the cell field and ODD(c) walls; without: -div(kappa grad u) with ODD(0) walls
  Problem(int64_t n, const std::vector<int> &gpus, int levels = 4, bool sigma = true, bool coefs = true) : dd(new DistributedDomain(n, n, n)) {
    dd->set_gpus(gpus);
    dd->set_radius(Radius::constant(1));
    u = dd->add_data<T>("u");
    f = dd->add_data<T>("f");
    r = dd->add_data<T>("r");
    const int nk = coefs ? (sigma ? 4 : 3) : 0;
    for (int i = 0; i < nk; ++i) k.push_back(dd->add_data<T>("k" + std::to_string(i)));
    dd->set_boundary(Topology::Boundary::FIXED);
    for (int a = 0, j = 0; a < 3; ++a)
      for (int s = -1; s <= 1; s += 2, ++j) {
        const Dim3 dir(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0);
        dd->set_boundary_condition(u, dir, stencil::BC::ODD(sigma ? WALL[j] : 0.0));
        for (int i = 0; i < nk; ++i) dd->set_boundary_condition(k[size_t(i)], dir, i == 3 ? stencil::BC::VALUE(2.0) : stencil::BC::EVEN());
      }
    dd->realize();
    fill_q(*dd, u, 0, n);
    fill_q(*dd, f, 1, n);
    for (int i = 0; i < nk; ++i) fill_q(*dd, k[size_t(i)], i == 3 ? 2 : 3 + i, n);
    if (coefs)
      mg.reset(new stencil::Multigrid<T>(*dd, u, f, r, [n, sigma](int l) { return A_at(l, n, sigma); }, k,
                                         std::vector<std::string>(KINDS.begin(), KINDS.begin() + nk), 2, 2, 30, levels));
    else
      mg.reset(new stencil::Multigrid<T>(*dd, u, f, r, [n](int l) {
        const double h = double(1 << l) / double(n);
        return LinearStencil::laplacian(2, h, h, h).scaled(-1.0);
      }, 2, 2, 30, levels));
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
    std::vector<DataHandle<T>> k;
  };
  Problem<T> &P;
  int64_t n;
  std::vector<Level> lv;
  Manual(Problem<T> &p, int64_t n_, const std::vector<int> &gpus) : P(p), n(n_) {
    for (int l = 1; l < 4; ++l) {
      Level L;
      const int64_t m = n >> l;
      L.dd.reset(new DistributedDomain(m, m, m));
      L.dd->set_gpus(gpus);
      L.dd->set_radius(Radius::constant(1));
      L.u = L.dd->template add_data<T>("u");
      L.f = L.dd->template add_data<T>("f");
      for (int i = 0; i < 4; ++i) L.k.push_back(L.dd->template add_data<T>("k" + std::to_string(i)));
      L.dd->set_boundary(Topology::Boundary::FIXED);
      for (int a = 0; a < 3; ++a)
        for (int s = -1; s <= 1; s += 2) {
          const Dim3 dir(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0);
          L.dd->set_boundary_condition(L.u, dir, stencil::BC::ODD(0.0));
          for (int i = 0; i < 4; ++i) L.dd->set_boundary_condition(L.k[size_t(i)], dir, i == 3 ? stencil::BC::VALUE(2.0) : stencil::BC::EVEN());
        }
      L.dd->realize();
      lv.push_back(std::move(L));
    }
  }
  DistributedDomain &dd(int l) { return l == 0 ? *P.dd : *lv[size_t(l - 1)].dd; }
  std::vector<DataHandle<T>> k(int l) { return l == 0 ? P.k : lv[size_t(l - 1)].k; }
  void update() {
    for (int l = 0; l < 3; ++l)
      for (int i = 0; i < 4; ++i) {
        if (i < 3)
          dd(l).restrict_to(dd(l + 1), stencil::curr(k(l + 1)[size_t(i)]), stencil::curr(k(l)[size_t(i)]), i);
        else
          dd(l).restrict_to(dd(l + 1), stencil::curr(k(l + 1)[size_t(i)]), stencil::curr(k(l)[size_t(i)]));
      }
  }
  LinearStencil res(int l) {
    LinearStencil r;
    r.add(Source::aux, 0, 0, 0, 1.0);
    const LinearStencil A = A_at(l, n, true); // named: a range-for over a temporary's vterms() would dangle
    for (const sb_stencil_vterm &t : A.vterms())
      r.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight, t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2]);
    return r;
  }
  void smooth(int l, DataHandle<T> u, DataHandle<T> f, int sweeps) {
    for (int i = 0; i < sweeps; ++i)
      for (int c = 0; c < 2; ++c) dd(l).relax(A_at(l, n, true), stencil::curr(u), u, stencil::curr(f), k(l), stencil::Colour{2, c});
  }
  void cycle(int l) {
    const DataHandle<T> u = l == 0 ? P.u : lv[size_t(l - 1)].u, f = l == 0 ? P.f : lv[size_t(l - 1)].f;
    if (l == 3) {
      smooth(l, u, f, 30);
      return;
    }
    smooth(l, u, f, 2);
    Level &C = lv[size_t(l)];
    dd(l).restrict_to(*C.dd, stencil::curr(C.f), res(l), u, stencil::curr(f), k(l));
    fill_q(*C.dd, C.u, 0, n);
    cycle(l + 1);
    dd(l).prolong_from(*C.dd, stencil::curr(u), stencil::curr(C.u), stencil::curr(u));
    smooth(l, u, f, 2);
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
    M->update();
  }
  const double r0 = P.mg->residual_norm();
  for (int cyc = 0; cyc < 3; ++cyc) {
    P.mg->cycle();
    bits.push_back(hexsum(gather<T>(*P.dd, P.u.id(), n)));
    if (manual) {
      M->cycle(0);
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
  // kappa scaled by 1.5: re-coarsen, then solve
  for (int i = 0; i < 3; ++i) fill_q(*P.dd, P.k[size_t(i)], 3 + i, n, 1.5);
  P.mg->update_coefficients();
  const double rtol = sizeof(T) == 8 ? 1e-6 : 1e-3;
  const std::vector<double> hist = P.mg->solve(rtol, 25);
  const double fn = std::sqrt(P.dd->reduce(P.f, stencil::Which::curr, stencil::Sum::exact).sumsq);
  if (!(hist.back() <= rtol * fn)) {
    if (0 == mpi::world_rank()) std::fprintf(stderr, "%zu-byte elements: solve() stopped at %g > %g after %zu cycles\n", sizeof(T), hist.back(), rtol * fn, hist.size() - 1);
    ++bad;
  }
  bits.push_back(hexsum(gather<T>(*P.dd, P.u.id(), n)) + " " + std::to_string(hist.size()));
  return bad;
}

template <typename T> static void time_cycles(Problem<T> &P, int64_t n, int cycles, const char *what) {
  P.mg->cycle(); // warm-up: plans, events, first launches
  fill_q(*P.dd, P.u, 0, n);
  std::printf("{\"workload\": \"%lld^3 FP64 %s, ODD(0) walls, V(2,2) to 4^3, 30 coarsest sweeps: stencil::Multigrid<double>::cycle()\", \"ms_per_cycle\": [",
              (long long)n, what);
  std::vector<double> res, ms;
  for (int k = 0; k < cycles; ++k) {
    const auto t0 = std::chrono::steady_clock::now();
    P.mg->cycle();
    ms.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
    std::printf("%s%.2f", k ? ", " : "", ms.back());
    res.push_back(P.mg->residual_norm());
  }
  std::printf("], \"residual\": [");
  for (size_t k = 0; k < res.size(); ++k) std::printf("%s%.4g", k ? ", " : "", res[k]);
  std::printf("]}\n");
  std::fflush(stdout);
}

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s --single N OUT | --expect OUT | --time N C\n", argv[0]);
    return 2;
  }
  if (std::string(argv[1]) == "--time" && argc >= 4) {
    const int64_t n = std::atoll(argv[2]);
    const int cycles = std::atoi(argv[3]), levels = int(std::log2(double(n))) - 1;
    {
      Problem<double> P(n, {0}, levels, false, true);
      time_cycles(P, n, cycles, "-div(kappa grad u) = f, smooth kappa");
    }
    {
      Problem<double> P(n, {0}, levels, false, false);
      time_cycles(P, n, cycles, "-lap u = f");
    }
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
    std::printf("stencil::Multigrid with coefficient fields, queued V-cycles, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(),
                all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
