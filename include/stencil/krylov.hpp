// Multigrid-preconditioned conjugate gradients for A x = f on a DistributedDomain (DESIGN.md section 2.13), the C++ twin
// of stencil_b200.PCG: flexible CG (the Polak-Ribiere form, which tolerates the V-cycle's slight asymmetry) with one
// V-cycle of stencil::Multigrid as the preconditioner, the vector algebra in the fused Krylov kernels (sb_krylov_plan_*)
// and every inner product exact, so the iterates are the same bits on every partition and rank count.
//
//     stencil::PCG<double> cg(dd, x, f, r, z, p, q, [&](int l) { return A(l); }, {kx, ky, kz}, {"x", "y", "z"});
//     std::vector<double> history = cg.solve(1e-8, 50);                          // sqrt(<r, r>) per iteration
//
// x, f, r, z, p and q are distinct quantities of the realized domain dd: x the solution (its value the first guess), f
// the right-hand side, r the residual, z the preconditioned residual, p the search direction and q = A p.  p and z must
// carry the homogeneous counterpart of x's BC on every FIXED face (ODD(c) -> ODD(0), EVEN -> EVEN, VALUE(c) ->
// VALUE(0)); x keeps its own, which enters through the first residual.  With precond = true an internal
// Multigrid<T>(dd, z, r, q, op_at, ...) is the preconditioner (its u is z, its f is r; q is only the scratch of its
// residual_norm, never called); with precond = false z is not used (z is r) and only op_at(0) is.  Refusals (LOG_FATAL)
// come before any domain is built.  Each iteration queues the V-cycle, a DOT, XPBY, the apply, a DOT and UPDATE on the
// apply streams and waits on the host three times, for beta, alpha and the stopping test (in float, where gamma and
// delta come from two one-pair DOTs, the first wait takes two gathers).  Every pass looks its buffers up for the
// current swap parity, so dd.swap() may be called between solves.  A breakdown (a non-positive or
// non-finite <p, A p>, or a non-finite <z, r>) is not fatal: solve() returns the history so far and breakdown() names
// the iteration.  Building, solve(), residual_norm() and update_coefficients() are collective under MPI.
#pragma once

#include <cmath>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "stencil/multigrid.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

namespace stencil {

template <typename T> class PCG {
public:
  PCG(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> z, DataHandle<T> p, DataHandle<T> q,
      const std::function<LinearStencil(int)> &op_at, bool precond = true, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : dd_(dd), x_(x), f_(f), r_(r), z_(precond ? z : r), p_(p), q_(q) {
    init(op_at, precond, {}, {}, nu1, nu2, coarse_sweeps, levels);
  }
  PCG(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> z, DataHandle<T> p, DataHandle<T> q,
      const std::function<LinearStencil(int)> &op_at, const std::vector<DataHandle<T>> &coefs, const std::vector<std::string> &coef_kinds,
      bool precond = true, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : dd_(dd), x_(x), f_(f), r_(r), z_(precond ? z : r), p_(p), q_(q) {
    init(op_at, precond, coefs, coef_kinds, nu1, nu2, coarse_sweeps, levels);
  }

  // the iteration at which the last solve() broke down, or -1
  int breakdown() const { return breakdown_; }
  Multigrid<T> *preconditioner() { return mg_.get(); }

  // iterations from the current x until sqrt(<r, r>) <= rtol ||f||_2 (||f||_2 exact) or max_iters; sqrt(<r, r>) before
  // the first iteration and after each (r the recursive residual)
  std::vector<double> solve(double rtol, int max_iters) {
    const double target = rtol * std::sqrt(dd_.reduce(f_, Which::curr, Sum::exact).sumsq);
    breakdown_ = -1;
    std::vector<double> hist{std::sqrt(start())};
    for (int k = 0; hist.back() > target && k < max_iters; ++k) {
      double rho;
      if (!iterate(k, rho)) break;
      hist.push_back(std::sqrt(rho));
    }
    finish();
    return hist;
  }

  // the true ||f - A x||_2 (the residual into r, then an exact dot)
  double residual_norm() {
    if (coefs_.empty())
      dd_.apply(res_, curr(r_), x_, curr(f_));
    else
      dd_.apply(res_, curr(r_), x_, curr(f_), coefs_);
    return std::sqrt(dd_.dot(r_, r_));
  }

  // re-coarsen the preconditioner's coefficient fields after they change (A on the fine level reads them directly)
  void update_coefficients() {
    if (mg_) mg_->update_coefficients();
  }

private:
  DistributedDomain &dd_;
  DataHandle<T> x_, f_, r_, z_, p_, q_;
  std::vector<DataHandle<T>> coefs_;
  LinearStencil A_, res_;
  std::unique_ptr<Multigrid<T>> mg_;
  int breakdown_ = -1;
  double eta_ = 0;

  static BC homogeneous(const BC &bc) {
    return bc.kind == BC::Kind::ODD ? BC::ODD(0.0) : bc.kind == BC::Kind::EVEN ? BC::EVEN() : BC::VALUE(0.0);
  }

  void init(const std::function<LinearStencil(int)> &op_at, bool precond, const std::vector<DataHandle<T>> &coefs,
            const std::vector<std::string> &coef_kinds, int nu1, int nu2, int coarse_sweeps, int levels) {
    const int dtype = bc_dtype<T>();
    if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL("PCG: the quantities must be float or double");
    if (dd_.domains_.empty()) LOG_FATAL("PCG: dd must be realized");
    std::vector<std::pair<const char *, size_t>> named{{"x", x_.id()}, {"f", f_.id()}, {"r", r_.id()}, {"p", p_.id()}, {"q", q_.id()}};
    if (precond) named.push_back({"z", z_.id()});
    for (size_t i = 0; i < named.size(); ++i)
      for (size_t j = 0; j < i; ++j)
        if (named[i].second == named[j].second) LOG_FATAL("PCG: " << named[i].first << " and " << named[j].first << " must be different quantities");
    for (size_t k = 0; k < coefs.size(); ++k)
      for (const auto &n : named)
        if (coefs[k].id() == n.second) LOG_FATAL("PCG: coefficient " << k << " must be a quantity other than x, f, r, z, p and q");
    static const char *const kFace[6] = {"-x", "+x", "-y", "+y", "-z", "+z"};
    for (int fc = 0; fc < 6; ++fc) {
      if (dd_.boundary_[fc / 2] != Topology::Boundary::FIXED) continue;
      auto bx = dd_.bcs_.find(std::make_pair(x_.id(), fc));
      if (bx == dd_.bcs_.end() || bx->second.kind == BC::Kind::NONE)
        LOG_FATAL("PCG: x needs a boundary condition (ODD, EVEN or VALUE) on every FIXED face (face " << kFace[fc] << ")");
      const BC want = homogeneous(bx->second);
      std::vector<std::pair<const char *, size_t>> vecs{{"p", p_.id()}};
      if (precond) vecs.push_back({"z", z_.id()});
      for (const auto &v : vecs) {
        auto it = dd_.bcs_.find(std::make_pair(v.second, fc));
        const BC got = it == dd_.bcs_.end() ? BC::NONE() : it->second;
        if (got.kind != want.kind || got.value != want.value)
          LOG_FATAL("PCG: " << v.first << " needs the homogeneous counterpart of x's BC on face " << kFace[fc] << " (kind " << int(want.kind)
                            << ", value 0), not kind " << int(got.kind) << ", value " << got.value);
      }
    }
    A_ = op_at(0);
    if (A_.has_aux()) LOG_FATAL("PCG: op_at(0) has an aux term; A reads x only");
    if (size_t(A_.ncoef()) != coefs.size())
      LOG_FATAL("PCG: op_at(0) reads " << A_.ncoef() << " coefficient fields, but " << coefs.size() << " were given");
    res_ = Multigrid<T>::residual(A_);
    coefs_ = coefs;
    dd_.create_apply_streams();
    if (precond) {
      if (coefs.empty())
        mg_.reset(new Multigrid<T>(dd_, z_, r_, q_, op_at, nu1, nu2, coarse_sweeps, levels));
      else
        mg_.reset(new Multigrid<T>(dd_, z_, r_, q_, op_at, coefs, coef_kinds, nu1, nu2, coarse_sweeps, levels));
    }
  }

  void queued(bool on) {
    dd_.queued_ = on;
    if (mg_)
      for (auto &L : mg_->levels_) L.dd->queued_ = on;
  }

  // r = f - A x (x's own BC through the exchange); returns <r, r>
  double start() {
    queued(true);
    if (coefs_.empty())
      dd_.apply(res_, curr(r_), x_, curr(f_));
    else
      dd_.apply(res_, curr(r_), x_, curr(f_), coefs_);
    DistributedDomain::KrylovCache &c = dd_.krylov_plans(SB_KRYLOV_DOT, {r_.id(), r_.id()});
    dd_.krylov_launch(c, 0.0, true);
    return dd_.krylov_sums(c, true)[0];
  }

  bool iterate(int k, double &rho) {
    if (mg_) { // z = M r from z = +0 (a memset of the curr allocation; the cycle's exchanges refill the ghost cells)
      dd_.queue_after_exterior();
      for (size_t di = 0; di < dd_.domains_.size(); ++di) {
        LocalDomain &d = dd_.domains_[di];
        d.set_device();
        const cudaPitchedPtr pp = d.curr_data(z_.id());
        CUDA_RUNTIME(cudaMemsetAsync(pp.ptr, 0, pp.pitch * pp.ysize * size_t(d.raw_size().z), dd_.applyStreams_[2 * di]));
      }
      mg_->vcycle(0);
    }
    // <z, r> and <z, q>: one two-pair DOT in double (3 reads instead of 4); in float the two-pair kernel is bound by its
    // per-cell work and two one-pair launches are faster (DESIGN.md section 2.13).  The sums are exact either way.
    double gamma, delta = 0.0;
    if (k == 0 || sizeof(T) == 4) {
      DistributedDomain::KrylovCache &zr = dd_.krylov_plans(SB_KRYLOV_DOT, {z_.id(), r_.id()});
      dd_.krylov_launch(zr, 0.0, true);
      if (k > 0) {
        DistributedDomain::KrylovCache &zq = dd_.krylov_plans(SB_KRYLOV_DOT, {z_.id(), q_.id()});
        dd_.krylov_launch(zq, 0.0, true);
        delta = dd_.krylov_sums(zq, true)[0];
      }
      gamma = dd_.krylov_sums(zr, true)[0];
    } else {
      DistributedDomain::KrylovCache &zrq = dd_.krylov_plans(SB_KRYLOV_DOT, {z_.id(), r_.id(), q_.id()});
      dd_.krylov_launch(zrq, 0.0, true);
      const std::vector<double> gd = dd_.krylov_sums(zrq, true);
      gamma = gd[0];
      delta = gd[1];
    }
    if (!std::isfinite(gamma)) {
      breakdown_ = k;
      return false;
    }
    dd_.krylov_launch(dd_.krylov_plans(SB_KRYLOV_XPBY, {p_.id(), z_.id()}), k == 0 ? 0.0 : -delta / eta_, true);
    if (coefs_.empty())
      dd_.apply(A_, curr(q_), p_);
    else
      dd_.apply(A_, curr(q_), p_, coefs_);
    DistributedDomain::KrylovCache &pq = dd_.krylov_plans(SB_KRYLOV_DOT, {p_.id(), q_.id()});
    dd_.krylov_launch(pq, 0.0, true);
    const double eta = dd_.krylov_sums(pq, true)[0];
    if (!(std::isfinite(eta) && eta > 0.0)) {
      breakdown_ = k;
      return false;
    }
    eta_ = eta;
    DistributedDomain::KrylovCache &up = dd_.krylov_plans(SB_KRYLOV_UPDATE, {x_.id(), p_.id(), r_.id(), q_.id()});
    dd_.krylov_launch(up, gamma / eta, true);
    rho = dd_.krylov_sums(up, true)[0];
    return true;
  }

  // the end of a queued solve: every apply stream and exchange complete
  void finish() {
    queued(false);
    for (size_t i = 0; i < dd_.applyStreams_.size(); ++i) {
      CUDA_RUNTIME(cudaSetDevice(dd_.domains_[i / 2].gpu()));
      CUDA_RUNTIME(cudaStreamSynchronize(dd_.applyStreams_[i]));
    }
    dd_.exchange_wait();
    if (mg_)
      for (auto &L : mg_->levels_) L.dd->exchange_wait();
  }
};

} // namespace stencil
