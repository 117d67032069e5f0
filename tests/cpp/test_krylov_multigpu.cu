// C++ API check of stencil::PCG<T> (include/stencil/krylov.hpp, DESIGN.md section 2.13) and DistributedDomain::dot --
// one process with N subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when
// there are fewer GPUs than ranks).
//   bin/test_krylov_multigpu --single N OUT     one process, N subdomains: the bits must equal a one-subdomain run's,
//                                              and are written to OUT
//   bin/sb_mpirun -n N bin/test_krylov_multigpu --expect OUT
//                                              one subdomain per rank: every rank's bits must equal OUT's
//   bin/test_krylov_multigpu --time N C        one GPU, N^3 FP64: C PCG iterations of -lap x = f (ODD(0) walls) against C
//                                              V(2,2) cycles of its preconditioner; then -div(kappa grad x) = f with a
//                                              10^3 jump in kappa solved to 1e-8 ||f|| by PCG, and Multigrid cycles for
//                                              the same wall time; one JSON line each
// Runs, in double and float, 1, 2 and 3 iterations of multigrid-preconditioned CG over 4 levels (32^3 .. 4^3) of
// -div(kappa grad x) + sigma x = f, kappa smooth on faces (EVEN walls), sigma a cell field (VALUE walls), x with ODD(c)
// walls (a different c on each face), then a solve(); and <f, f>, <x, f> by dot().  In the one-process mode it checks
// that the solver gives the bits of the same iterations written from public calls: Multigrid::cycle, apply, dot and the
// sb_krylov_plan_* passes.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <vector>

#include "stencil/krylov.hpp"
#include "stencil/linear_stencil.hpp"
#include "stencil/multigrid.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::LinearStencil;
using stencil::Source;

// what: 0 zero, 1 a right-hand side in [-4, 4), 2 sigma in [0.5, 2), 3 + a smooth kappa on the faces normal to axis a,
// 6 + a kappa with a 10^3 jump in the cube [1/4, 3/4)^3 on those faces
template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, int what, double n) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x) {
        double v = 0.0;
        if (what == 1) v = double((x * 7 + y * 131 + z * 1009) % 8191) * 0.0009765625 - 4.0;
        if (what == 2) v = 0.5 + double((x * 13 + y * 29 + z * 71) % 97) / 64.0;
        if (what >= 3) {
          const int a = (what - 3) % 3;
          const double p[3] = {(double(x) + (a == 0 ? 0.0 : 0.5)) / n, (double(y) + (a == 1 ? 0.0 : 0.5)) / n, (double(z) + (a == 2 ? 0.0 : 0.5)) / n};
          if (what < 6) {
            v = std::exp(0.5 * std::sin(6.283185307179586 * p[0]) * std::sin(6.283185307179586 * p[1]) * std::sin(6.283185307179586 * p[2]));
          } else {
            bool in = true;
            for (int b = 0; b < 3; ++b) in = in && (b == a ? (p[b] > 0.25 && p[b] < 0.75) : (p[b] >= 0.25 && p[b] < 0.75));
            v = in ? 1000.0 : 1.0;
          }
        }
        acc[Dim3(x, y, z)] = T(v);
      }
}

const double WALL[6] = {0.0, 0.25, -0.5, 1.0, 0.125, -1.0};
const std::vector<std::string> KINDS = {"x", "y", "z", "cell"};

// -div(kappa grad x) (+ sigma x, field 3), or -lap x with plain terms
LinearStencil A_at(int l, int64_t n, int ncoef) {
  const double h = double(1 << l) / double(n);
  if (ncoef == 0) return LinearStencil::laplacian(2, h, h, h).scaled(-1.0);
  LinearStencil A = LinearStencil::div_grad(h, h, h).scaled(-1.0);
  if (ncoef == 4) A.add(Source::src, 0, 0, 0, 1.0, 3, 0, 0, 0);
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

static std::string hexd(const std::vector<double> &v) { return hexsum(v); }

template <typename T> void fill_q(DistributedDomain &dd, DataHandle<T> q, int what, int64_t n) {
  for (auto &d : dd.domains()) {
    d.set_device();
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(q), d.get_compute_region(), what, double(n));
    CUDA_RUNTIME(cudaDeviceSynchronize());
  }
}

template <typename T> struct Problem {
  std::unique_ptr<DistributedDomain> dd;
  DataHandle<T> x{0}, f{1}, r{2}, z{3}, p{4}, q{5};
  std::vector<DataHandle<T>> k;
  int64_t n;
  int ncoef;
  std::unique_ptr<stencil::PCG<T>> cg;
  // ncoef 4: ODD(c) walls on x, smooth kappa and sigma; 3: ODD(0) walls, kappa smooth (kfill 3) or with a jump (kfill 6);
  // 0: -lap x = f on ODD(0) walls
  Problem(int64_t n_, const std::vector<int> &gpus, int levels, int ncoef_, int kfill = 3, bool solver = true)
      : dd(new DistributedDomain(n_, n_, n_)), n(n_), ncoef(ncoef_) {
    dd->set_gpus(gpus);
    dd->set_radius(Radius::constant(1));
    x = dd->add_data<T>("x");
    f = dd->add_data<T>("f");
    r = dd->add_data<T>("r");
    z = dd->add_data<T>("z");
    p = dd->add_data<T>("p");
    q = dd->add_data<T>("q");
    for (int i = 0; i < ncoef; ++i) k.push_back(dd->add_data<T>("k" + std::to_string(i)));
    dd->set_boundary(Topology::Boundary::FIXED);
    for (int a = 0, j = 0; a < 3; ++a)
      for (int s = -1; s <= 1; s += 2, ++j) {
        const Dim3 dir(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0);
        dd->set_boundary_condition(x, dir, stencil::BC::ODD(ncoef == 4 ? WALL[j] : 0.0));
        dd->set_boundary_condition(p, dir, stencil::BC::ODD(0.0));
        dd->set_boundary_condition(z, dir, stencil::BC::ODD(0.0));
        for (int i = 0; i < ncoef; ++i) dd->set_boundary_condition(k[size_t(i)], dir, i == 3 ? stencil::BC::VALUE(2.0) : stencil::BC::EVEN());
      }
    dd->realize();
    fill_q(*dd, x, 0, n);
    fill_q(*dd, f, 1, n);
    for (int i = 0; i < ncoef; ++i) fill_q(*dd, k[size_t(i)], i == 3 ? 2 : kfill + i, n);
    if (!solver) return;
    const int nc = ncoef;
    const int64_t nn = n;
    auto op = [nn, nc](int l) { return A_at(l, nn, nc); };
    if (ncoef)
      cg.reset(new stencil::PCG<T>(*dd, x, f, r, z, p, q, op, k, std::vector<std::string>(KINDS.begin(), KINDS.begin() + ncoef), true, 2, 2, 30, levels));
    else
      cg.reset(new stencil::PCG<T>(*dd, x, f, r, z, p, q, op, true, 2, 2, 30, levels));
  }
  ~Problem() {
    cg.reset();
    dd.reset();
  }
};

// one sb_krylov_plan pass per local subdomain over its compute region (the public C ABI), synchronously
template <typename T> void krylov_pass(DistributedDomain &dd, int mode, const std::vector<size_t> &qs, double s) {
  for (LocalDomain &d : dd.domains()) {
    d.set_device();
    const Rect3 cr = d.get_compute_region();
    const Dim3 ao = d.origin() - Dim3(1, 1, 1);
    std::vector<sb_pitched> bufs;
    for (size_t q : qs) {
      const cudaPitchedPtr pp = d.curr_data(q);
      bufs.push_back(sb_pitched{pp.ptr, int64_t(pp.pitch), int64_t(pp.ysize)});
    }
    const int64_t acc[3] = {ao.x, ao.y, ao.z}, lo[3] = {cr.lo.x, cr.lo.y, cr.lo.z}, hi[3] = {cr.hi.x, cr.hi.y, cr.hi.z};
    sb_krylov_plan *plan = nullptr;
    if (SB_OK != sb_krylov_plan_create(&plan, d.gpu(), mode, stencil::bc_dtype<T>(), bufs.data(), int(bufs.size()), acc, lo, hi)) LOG_FATAL(sb_last_error());
    sb_reduce_exact_part *parts = nullptr;
    CUDA_RUNTIME(cudaMalloc(&parts, 2 * sizeof(sb_reduce_exact_part)));
    if (SB_OK != sb_krylov_plan_launch(plan, s, parts, nullptr)) LOG_FATAL(sb_last_error());
    CUDA_RUNTIME(cudaDeviceSynchronize());
    sb_krylov_plan_destroy(plan);
    CUDA_RUNTIME(cudaFree(parts));
  }
}

// the same iterations from public calls, on a second problem's domain with its own Multigrid over (z, r, q)
template <typename T> std::vector<double> manual(Problem<T> &Q, int iters) {
  const int64_t n = Q.n;
  const int nc = Q.ncoef;
  stencil::Multigrid<T> mg(*Q.dd, Q.z, Q.r, Q.q, [n, nc](int l) { return A_at(l, n, nc); }, Q.k,
                           std::vector<std::string>(KINDS.begin(), KINDS.begin() + nc), 2, 2, 30, 4);
  const LinearStencil A = A_at(0, n, nc);
  LinearStencil res;
  res.add(Source::aux, 0, 0, 0, 1.0);
  for (const sb_stencil_vterm &t : A.vterms())
    res.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight, t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2]);
  DistributedDomain &dd = *Q.dd;
  dd.apply(res, stencil::curr(Q.r), Q.x, stencil::curr(Q.f), Q.k);
  std::vector<double> hist{std::sqrt(dd.dot(Q.r, Q.r))};
  double eta = 0;
  for (int k = 0; k < iters; ++k) {
    fill_q(dd, Q.z, 0, n);
    mg.cycle();
    const double gamma = dd.dot(Q.z, Q.r), delta = k ? dd.dot(Q.z, Q.q) : 0.0;
    krylov_pass<T>(dd, SB_KRYLOV_XPBY, {Q.p.id(), Q.z.id()}, k ? -delta / eta : 0.0);
    dd.apply(A, stencil::curr(Q.q), Q.p, Q.k);
    eta = dd.dot(Q.p, Q.q);
    krylov_pass<T>(dd, SB_KRYLOV_UPDATE, {Q.x.id(), Q.p.id(), Q.r.id(), Q.q.id()}, gamma / eta);
    hist.push_back(std::sqrt(dd.dot(Q.r, Q.r)));
  }
  return hist;
}

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits, bool check_manual) {
  const int64_t n = 32;
  long bad = 0;
  Problem<T> P(n, gpus, 4, 4);
  if (!P.cg->preconditioner() || P.cg->preconditioner()->num_levels() != 4) {
    std::fprintf(stderr, "the preconditioner has no 4 levels\n");
    ++bad;
  }
  std::vector<double> hist3;
  for (int it = 1; it <= 3; ++it) {
    fill_q(*P.dd, P.x, 0, n);
    const std::vector<double> hist = P.cg->solve(0.0, it);
    if (P.cg->breakdown() != -1 || int(hist.size()) != it + 1) {
      std::fprintf(stderr, "%zu-byte elements: %d iteration(s) gave %zu norms, breakdown %d\n", sizeof(T), it, hist.size(), P.cg->breakdown());
      ++bad;
    }
    bits.push_back(hexsum(gather<T>(*P.dd, P.x.id(), n)) + " " + hexd(hist));
    hist3 = hist;
  }
  if (check_manual) {
    Problem<T> Q(n, gpus, 4, 4, 3, false);
    const std::vector<double> hist = manual(Q, 3);
    if (hist != hist3 || hexsum(gather<T>(*Q.dd, Q.x.id(), n)) + " " + hexd(hist) != bits.back()) {
      std::fprintf(stderr, "%zu-byte elements: PCG differs from the same iterations written from public calls\n", sizeof(T));
      ++bad;
    }
  }
  bits.push_back(hexd({P.dd->dot(P.f, P.f), P.dd->dot(P.x, P.f)}));
  fill_q(*P.dd, P.x, 0, n);
  const double rtol = sizeof(T) == 8 ? 1e-8 : 1e-4;
  const std::vector<double> hist = P.cg->solve(rtol, 30);
  const double fn = std::sqrt(P.dd->dot(P.f, P.f)), tn = P.cg->residual_norm();
  if (!(hist.back() <= rtol * fn) || !(tn <= 10 * rtol * fn)) {
    if (0 == mpi::world_rank())
      std::fprintf(stderr, "%zu-byte elements: solve() stopped at %g (true %g) > %g after %zu iterations\n", sizeof(T), hist.back(), tn, rtol * fn, hist.size() - 1);
    ++bad;
  }
  bits.push_back(hexsum(gather<T>(*P.dd, P.x.id(), n)) + " " + std::to_string(hist.size()));
  return bad;
}

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static void timing(int64_t n, int iters) {
  const int levels = int(std::log2(double(n))) - 1;
  {
    Problem<double> P(n, {0}, levels, 0);
    P.cg->solve(0.0, 1); // warm-up: plans, events, first launches
    fill_q(*P.dd, P.x, 0, n);
    double t0 = now_ms();
    P.cg->solve(0.0, 0);
    const double t_start = now_ms() - t0;
    fill_q(*P.dd, P.x, 0, n);
    t0 = now_ms();
    const std::vector<double> hist = P.cg->solve(0.0, iters);
    const double t_pcg = (now_ms() - t0 - t_start) / iters;
    t0 = now_ms();
    for (int k = 0; k < iters; ++k) P.cg->preconditioner()->cycle();
    const double t_cyc = (now_ms() - t0) / iters;
    std::printf("{\"workload\": \"%lld^3 FP64 -lap x = f, ODD(0) walls, V(2,2) to 4^3: stencil::PCG<double> iteration vs its preconditioner's cycle()\", "
                "\"ms_per_iteration\": %.3f, \"ms_per_vcycle\": %.3f, \"ratio\": %.3f, \"factor_per_iteration\": %.4g}\n",
                (long long)n, t_pcg, t_cyc, t_pcg / t_cyc, std::pow(hist.back() / hist.front(), 1.0 / iters));
    std::fflush(stdout);
  }
  {
    Problem<double> P(n, {0}, levels, 3, 6);
    P.cg->solve(0.0, 1);
    fill_q(*P.dd, P.x, 0, n);
    double t0 = now_ms();
    const std::vector<double> hist = P.cg->solve(1e-8, 60);
    const double t_pcg = now_ms() - t0;
    // Multigrid alone on the same problem (x from 0, its residual in r) for the same wall time
    fill_q(*P.dd, P.x, 0, n);
    stencil::Multigrid<double> mg(*P.dd, P.x, P.f, P.r, [n](int l) { return A_at(l, n, 3); }, P.k, {"x", "y", "z"}, 2, 2, 30, levels);
    const double r0 = mg.residual_norm();
    mg.cycle();
    fill_q(*P.dd, P.x, 0, n);
    int cycles = 0;
    double t_mg = 0;
    while (t_mg < t_pcg) {
      t0 = now_ms();
      mg.cycle();
      t_mg += now_ms() - t0;
      ++cycles;
    }
    std::printf("{\"workload\": \"%lld^3 FP64 -div(kappa grad x) = f, 10^3 jump in kappa, ODD(0) walls: PCG to 1e-8 ||f|| vs Multigrid cycles for the same "
                "time\", \"pcg_iterations\": %zu, \"pcg_ms\": %.1f, \"pcg_final\": %.3g, \"mg_cycles\": %d, \"mg_ms\": %.1f, \"mg_final\": %.3g}\n",
                (long long)n, hist.size() - 1, t_pcg, hist.back() / hist.front(), cycles, t_mg, mg.residual_norm() / r0);
    std::fflush(stdout);
  }
}

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s --single N OUT | --expect OUT | --time N C\n", argv[0]);
    return 2;
  }
  if (std::string(argv[1]) == "--time" && argc >= 4) {
    timing(std::atoll(argv[2]), std::atoi(argv[3]));
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
    std::printf("stencil::PCG, multigrid-preconditioned CG, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
