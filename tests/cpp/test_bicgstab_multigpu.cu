// C++ API check of stencil::BiCGStab<T> (include/stencil/bicgstab.hpp, DESIGN.md section 2.14) -- one process with N
// subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs
// than ranks).
//   bin/test_bicgstab_multigpu --single N OUT   one process, N subdomains: the bits must equal a one-subdomain run's,
//                                              and are written to OUT
//   bin/sb_mpirun -n N bin/test_bicgstab_multigpu --expect OUT
//                                              one subdomain per rank: every rank's bits must equal OUT's
//   bin/test_bicgstab_multigpu --time N C      one GPU, N^3 FP64 -div(kappa grad x) + b . grad x = f with a 10^3 jump in
//                                              kappa, ODD(0) walls: C BiCGStab iterations against 2C V(2,2) cycles of its
//                                              preconditioner; then BiCGStab to 1e-8 ||f||, and Multigrid cycles and PCG
//                                              iterations for the same wall time; one JSON line each
// Runs, in double and float, 1, 2 and 3 iterations of multigrid-preconditioned BiCGStab over 4 levels (32^3 .. 4^3) of
// -div(kappa grad x) + b . grad x + sigma x = f, kappa smooth on faces (EVEN walls), sigma a cell field (VALUE walls),
// b = (4, 2.4, 1.2), x with ODD(c) walls (a different c on each face), then a solve().  In the one-process mode it
// checks that the solver gives the bits of the same iterations written from public calls: Multigrid::cycle on both
// pairs, apply, dot and the sb_krylov_plan_* passes.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <memory>
#include <string>
#include <vector>

#include "stencil/bicgstab.hpp"
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
const double B[3] = {4.0, 2.4, 1.2};
const std::vector<std::string> KINDS = {"x", "y", "z", "cell"};

// -div(kappa grad x) + b . grad x (+ sigma x, field 3): central differences of the convection
LinearStencil A_at(int l, int64_t n, int ncoef) {
  const double h = double(1 << l) / double(n);
  LinearStencil A = LinearStencil::div_grad(h, h, h).scaled(-1.0);
  if (ncoef == 4) A.add(Source::src, 0, 0, 0, 1.0, 3, 0, 0, 0);
  for (int a = 0; a < 3; ++a)
    for (int s = -1; s <= 1; s += 2) A.add(Source::src, a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0, s * B[a] / (2 * h));
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
  DataHandle<T> x{0}, f{1}, r{2}, r0{3}, p{4}, v{5}, ph{6}, sh{7}, t{8};
  std::vector<DataHandle<T>> k;
  int64_t n;
  int ncoef;
  std::unique_ptr<stencil::BiCGStab<T>> bi;
  // ncoef 4: ODD(c) walls on x, smooth kappa and sigma; 3: ODD(0) walls, kappa smooth (kfill 3) or with a jump (kfill 6)
  Problem(int64_t n_, const std::vector<int> &gpus, int levels, int ncoef_, int kfill = 3, bool solver = true)
      : dd(new DistributedDomain(n_, n_, n_)), n(n_), ncoef(ncoef_) {
    dd->set_gpus(gpus);
    dd->set_radius(Radius::constant(1));
    DataHandle<T> *vecs[9] = {&x, &f, &r, &r0, &p, &v, &ph, &sh, &t};
    const char *names[9] = {"x", "f", "r", "r0", "p", "v", "phat", "shat", "t"};
    for (int i = 0; i < 9; ++i) *vecs[i] = dd->add_data<T>(names[i]);
    for (int i = 0; i < ncoef; ++i) k.push_back(dd->add_data<T>("k" + std::to_string(i)));
    dd->set_boundary(Topology::Boundary::FIXED);
    for (int a = 0, j = 0; a < 3; ++a)
      for (int s = -1; s <= 1; s += 2, ++j) {
        const Dim3 dir(a == 0 ? s : 0, a == 1 ? s : 0, a == 2 ? s : 0);
        dd->set_boundary_condition(x, dir, stencil::BC::ODD(ncoef == 4 ? WALL[j] : 0.0));
        dd->set_boundary_condition(ph, dir, stencil::BC::ODD(0.0));
        dd->set_boundary_condition(sh, dir, stencil::BC::ODD(0.0));
        for (int i = 0; i < ncoef; ++i) dd->set_boundary_condition(k[size_t(i)], dir, i == 3 ? stencil::BC::VALUE(2.0) : stencil::BC::EVEN());
      }
    dd->realize();
    fill_q(*dd, x, 0, n);
    fill_q(*dd, f, 1, n);
    for (int i = 0; i < ncoef; ++i) fill_q(*dd, k[size_t(i)], i == 3 ? 2 : kfill + i, n);
    if (!solver) return;
    const int nc = ncoef;
    const int64_t nn = n;
    bi.reset(new stencil::BiCGStab<T>(*dd, x, f, r, r0, p, v, ph, sh, t, [nn, nc](int l) { return A_at(l, nn, nc); }, k,
                                      std::vector<std::string>(KINDS.begin(), KINDS.begin() + ncoef), 2, 2, 30, levels));
  }
  ~Problem() {
    bi.reset();
    dd.reset();
  }
};

// one sb_krylov_plan pass per local subdomain over its compute region (the public C ABI, two scalars), synchronously
template <typename T> void krylov_pass(DistributedDomain &dd, int mode, const std::vector<size_t> &qs, double s, double t = 0.0) {
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
    if (SB_OK != sb_krylov_plan_launch2(plan, s, t, parts, nullptr)) LOG_FATAL(sb_last_error());
    CUDA_RUNTIME(cudaDeviceSynchronize());
    sb_krylov_plan_destroy(plan);
    CUDA_RUNTIME(cudaFree(parts));
  }
}

// the same iterations from public calls, on a second problem's domain with its own Multigrid over (phat, p, v)
template <typename T> std::vector<double> manual(Problem<T> &Q, int iters) {
  const int64_t n = Q.n;
  const int nc = Q.ncoef;
  stencil::Multigrid<T> mg(*Q.dd, Q.ph, Q.p, Q.v, [n, nc](int l) { return A_at(l, n, nc); }, Q.k,
                           std::vector<std::string>(KINDS.begin(), KINDS.begin() + nc), 2, 2, 30, 4);
  const LinearStencil A = A_at(0, n, nc);
  LinearStencil res;
  res.add(Source::aux, 0, 0, 0, 1.0);
  for (const sb_stencil_vterm &t : A.vterms())
    res.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight, t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2]);
  DistributedDomain &dd = *Q.dd;
  dd.apply(res, stencil::curr(Q.r), Q.x, stencil::curr(Q.f), Q.k);
  krylov_pass<T>(dd, SB_KRYLOV_XPBY, {Q.r0.id(), Q.r.id()}, 0.0);
  double rho = dd.dot(Q.r0, Q.r), rho_prev = 0, alpha = 0, omega = 0;
  std::vector<double> hist{std::sqrt(rho)};
  for (int k = 0; k < iters; ++k) {
    if (k == 0)
      krylov_pass<T>(dd, SB_KRYLOV_XPBY, {Q.p.id(), Q.r.id()}, 0.0);
    else
      krylov_pass<T>(dd, SB_KRYLOV_BICG_P, {Q.p.id(), Q.r.id(), Q.v.id()}, (rho / rho_prev) * (alpha / omega), omega);
    fill_q(dd, Q.ph, 0, n);
    mg.cycle();
    dd.apply(A, stencil::curr(Q.v), Q.ph, Q.k);
    alpha = rho / dd.dot(Q.r0, Q.v);
    krylov_pass<T>(dd, SB_KRYLOV_UPDATE, {Q.x.id(), Q.ph.id(), Q.r.id(), Q.v.id()}, alpha);
    fill_q(dd, Q.sh, 0, n);
    mg.cycle(Q.sh, Q.r);
    dd.apply(A, stencil::curr(Q.t), Q.sh, Q.k);
    omega = dd.dot(Q.t, Q.r) / dd.dot(Q.t, Q.t);
    krylov_pass<T>(dd, SB_KRYLOV_UPDATE, {Q.x.id(), Q.sh.id(), Q.r.id(), Q.t.id()}, omega);
    rho_prev = rho;
    rho = dd.dot(Q.r0, Q.r);
    hist.push_back(std::sqrt(dd.dot(Q.r, Q.r)));
  }
  return hist;
}

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits, bool check_manual) {
  const int64_t n = 32;
  long bad = 0;
  Problem<T> P(n, gpus, 4, 4);
  if (P.bi->preconditioner()->num_levels() != 4) {
    std::fprintf(stderr, "the preconditioner has no 4 levels\n");
    ++bad;
  }
  std::vector<double> hist3;
  for (int it = 1; it <= 3; ++it) {
    fill_q(*P.dd, P.x, 0, n);
    const std::vector<double> hist = P.bi->solve(0.0, it);
    if (P.bi->breakdown() != -1 || int(hist.size()) != it + 1) {
      std::fprintf(stderr, "%zu-byte elements: %d iteration(s) gave %zu norms, breakdown %d\n", sizeof(T), it, hist.size(), P.bi->breakdown());
      ++bad;
    }
    bits.push_back(hexsum(gather<T>(*P.dd, P.x.id(), n)) + " " + hexd(hist));
    hist3 = hist;
  }
  if (check_manual) {
    Problem<T> Q(n, gpus, 4, 4, 3, false);
    const std::vector<double> hist = manual(Q, 3);
    if (hist != hist3 || hexsum(gather<T>(*Q.dd, Q.x.id(), n)) + " " + hexd(hist) != bits.back()) {
      std::fprintf(stderr, "%zu-byte elements: BiCGStab differs from the same iterations written from public calls\n", sizeof(T));
      ++bad;
    }
  }
  fill_q(*P.dd, P.x, 0, n);
  const double rtol = sizeof(T) == 8 ? 1e-8 : 1e-4;
  const std::vector<double> hist = P.bi->solve(rtol, 30);
  const double fn = std::sqrt(P.dd->dot(P.f, P.f)), tn = P.bi->residual_norm();
  if (P.bi->breakdown() != -1 || !(hist.back() <= rtol * fn) || !(tn <= 10 * rtol * fn)) {
    if (0 == mpi::world_rank())
      std::fprintf(stderr, "%zu-byte elements: solve() stopped at %g (true %g) > %g after %zu iterations, breakdown %d\n", sizeof(T), hist.back(), tn, rtol * fn,
                   hist.size() - 1, P.bi->breakdown());
    ++bad;
  }
  bits.push_back(hexsum(gather<T>(*P.dd, P.x.id(), n)) + " " + std::to_string(hist.size()));
  return bad;
}

static double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

static void timing(int64_t n, int iters) {
  const int levels = int(std::log2(double(n))) - 1;
  Problem<double> P(n, {0}, levels, 3, 6);
  P.bi->solve(0.0, 1); // warm-up: plans, events, first launches
  fill_q(*P.dd, P.x, 0, n);
  double t0 = now_ms();
  P.bi->solve(0.0, 0);
  const double t_start = now_ms() - t0;
  fill_q(*P.dd, P.x, 0, n);
  t0 = now_ms();
  P.bi->solve(0.0, iters);
  const double t_it = (now_ms() - t0 - t_start) / iters;
  t0 = now_ms();
  for (int k = 0; k < 2 * iters; ++k) P.bi->preconditioner()->cycle();
  const double t_cyc = (now_ms() - t0) / (2 * iters);
  std::printf("{\"workload\": \"%lld^3 FP64 jump kappa + convection, V(2,2) to 4^3: stencil::BiCGStab<double> iteration vs two cycle()s of its "
              "preconditioner\", \"ms_per_iteration\": %.3f, \"ms_per_vcycle\": %.3f, \"ratio_to_two_cycles\": %.3f}\n",
              (long long)n, t_it, t_cyc, t_it / (2 * t_cyc));
  std::fflush(stdout);
  // BiCGStab to 1e-8 ||f||
  fill_q(*P.dd, P.x, 0, n);
  t0 = now_ms();
  const std::vector<double> hist = P.bi->solve(1e-8, 60);
  const double t_bi = now_ms() - t0;
  const double fn = std::sqrt(P.dd->dot(P.f, P.f));
  const double bi_true = P.bi->residual_norm() / fn;
  const int bi_breakdown = P.bi->breakdown();
  P.bi.reset();
  // Multigrid alone on the same problem (x from 0, its residual in r) for the same wall time
  stencil::Multigrid<double> mg(*P.dd, P.x, P.f, P.r, [n](int l) { return A_at(l, n, 3); }, P.k, {"x", "y", "z"}, 2, 2, 30, levels);
  mg.cycle();
  fill_q(*P.dd, P.x, 0, n);
  int cycles = 0;
  double t_mg = 0;
  while (t_mg < t_bi) {
    t0 = now_ms();
    mg.cycle();
    t_mg += now_ms() - t0;
    ++cycles;
  }
  const double mg_true = mg.residual_norm() / fn;
  // PCG on the same non-symmetric op (p, z carry ODD(0): the solver's phat and shat), iterations for the same wall time
  stencil::PCG<double> cg(*P.dd, P.x, P.f, P.r, P.sh, P.ph, P.t, [n](int l) { return A_at(l, n, 3); }, P.k, {"x", "y", "z"}, true, 2, 2, 30, levels);
  cg.solve(0.0, 1);
  int its = 1;
  double t_cg = 0;
  for (;; ++its) {
    fill_q(*P.dd, P.x, 0, n);
    t0 = now_ms();
    cg.solve(0.0, its);
    t_cg = now_ms() - t0;
    if (t_cg >= t_bi || cg.breakdown() != -1) break;
  }
  const double cg_true = cg.residual_norm() / fn;
  std::printf("{\"workload\": \"%lld^3 FP64 -div(kappa grad x) + b . grad x = f, 10^3 jump in kappa, b = (4, 2.4, 1.2), ODD(0) walls, V(2,2) to 4^3: "
              "BiCGStab to 1e-8 ||f|| vs Multigrid cycles and PCG iterations for the same time (true residuals / ||f||)\", \"bicgstab_iterations\": %zu, "
              "\"bicgstab_ms\": %.1f, \"bicgstab_final\": %.3g, \"bicgstab_breakdown\": %d, \"mg_cycles\": %d, \"mg_ms\": %.1f, \"mg_final\": %.3g, "
              "\"pcg_iterations\": %d, \"pcg_ms\": %.1f, \"pcg_final\": %.3g, \"pcg_breakdown\": %d}\n",
              (long long)n, hist.size() - 1, t_bi, bi_true, bi_breakdown, cycles, t_mg, mg_true, its, t_cg, cg_true, cg.breakdown());
  std::fflush(stdout);
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
    std::printf("stencil::BiCGStab, multigrid-preconditioned BiCGStab, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
