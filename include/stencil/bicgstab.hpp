// Multigrid-preconditioned BiCGStab for A x = f on a DistributedDomain (DESIGN.md section 2.14), the C++ twin of
// stencil_b200.BiCGStab: right-preconditioned BiCGStab for non-symmetric operators such as advection-diffusion, with one
// V-cycle of stencil::Multigrid from zero as M, the vector algebra in the fused Krylov kernels (SB_KRYLOV_BICG_P and
// SB_KRYLOV_UPDATE with c among them) and every inner product exact, so the iterates are the same bits on every
// partition and rank count.
//
//     stencil::BiCGStab<double> bi(dd, x, f, r, r0, p, v, phat, shat, t, [&](int l) { return A(l); }, {kx, ky, kz}, {"x", "y", "z"});
//     std::vector<double> history = bi.solve(1e-8, 50);                        // sqrt(<r, r>) per iteration
//
// x, f, r, r0, p, v, phat, shat and t are nine distinct quantities of the realized domain dd: x the solution (its value
// the first guess), f the right-hand side, r the residual (s from the half step on), r0 the shadow residual, p the
// direction, v = A phat, phat = M p, shat = M s, t = A shat.  phat and shat carry the homogeneous counterpart of x's BC
// on every FIXED face; x keeps its own.  The internal Multigrid<T>(dd, phat, p, v, op_at, ...) is M, run on (phat, p)
// and, by its pair form, on (shat, r); v is only the scratch of its residual_norm, never called.  Refusals (LOG_FATAL)
// come before any domain is built.  Each iteration waits on the host three times (for sigma, for <s, s>, <t, r>, <t, t>
// and for <r, r>, <r0, r>), each wait gathering every sum it needs in one exchange; every pass looks its buffers up for
// the current swap parity.  A breakdown (<r0, v> zero or not finite, <t, t> zero, omega zero or not finite, a new
// <r0, r> zero or not finite) is not fatal: solve() returns the history so far and breakdown() names the iteration.
// Building, solve(), residual_norm() and update_coefficients() are collective under MPI.  The refusals, the
// preconditioner and the queued passes are detail::KrylovSolver's (krylov.hpp), shared with PCG.
#pragma once

#include <cmath>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "stencil/krylov.hpp"
#include "stencil/multigrid.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

namespace stencil {

template <typename T> class BiCGStab : public detail::KrylovSolver<T> {
  using B = detail::KrylovSolver<T>;
  using typename B::Cache;
  using B::dd_;
  using B::x_;
  using B::f_;
  using B::r_;
  using B::breakdown_;
  using B::plans;
  using B::queue;
  using B::combine;
  using B::queue_residual;
  using B::apply_A;
  using B::precondition;
  using B::finish;

public:
  BiCGStab(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> r0, DataHandle<T> p, DataHandle<T> v,
           DataHandle<T> phat, DataHandle<T> shat, DataHandle<T> t, const std::function<LinearStencil(int)> &op_at, int nu1 = 2, int nu2 = 2,
           int coarse_sweeps = 30, int levels = 0)
      : BiCGStab(dd, x, f, r, r0, p, v, phat, shat, t, op_at, {}, {}, nu1, nu2, coarse_sweeps, levels) {}
  BiCGStab(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> r0, DataHandle<T> p, DataHandle<T> v,
           DataHandle<T> phat, DataHandle<T> shat, DataHandle<T> t, const std::function<LinearStencil(int)> &op_at, const std::vector<DataHandle<T>> &coefs,
           const std::vector<std::string> &coef_kinds, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : B(dd, x, f, r), r0_(r0), p_(p), v_(v), phat_(phat), shat_(shat), t_(t) {
    this->init("BiCGStab",
               {{"x", x.id()}, {"f", f.id()}, {"r", r.id()}, {"r0", r0.id()}, {"p", p.id()}, {"v", v.id()}, {"phat", phat.id()}, {"shat", shat.id()}, {"t", t.id()}},
               {{"phat", phat.id()}, {"shat", shat.id()}}, op_at, coefs, coef_kinds, {{phat, p}, {shat, r}}, v, nu1, nu2, coarse_sweeps, levels);
  }

  // iterations from the current x until sqrt(<r, r>) <= rtol ||f||_2 (||f||_2 exact) or max_iters; sqrt(<r, r>) before
  // the first iteration and after each, the last entry that of the x left behind (the half-step iterate after a
  // half-step stop or an omega breakdown)
  std::vector<double> solve(double rtol, int max_iters) {
    const double target = rtol * std::sqrt(dd_.reduce(f_, Which::curr, Sum::exact).sumsq);
    breakdown_ = -1;
    rho_ = start();
    std::vector<double> hist{std::sqrt(rho_)};
    for (int k = 0; hist.back() > target && k < max_iters; ++k)
      if (!iterate(k, target, hist)) break;
    finish();
    return hist;
  }

private:
  DataHandle<T> r0_, p_, v_, phat_, shat_, t_;
  double rho_ = 0, rho_prev_ = 0, alpha_ = 0, omega_ = 0;

  // r = f - A x (x's own BC through the exchange), r0 = r; returns <r0, r>
  double start() {
    queue_residual();
    queue(plans(SB_KRYLOV_XPBY, {r0_.id(), r_.id()}));
    Cache &c = plans(SB_KRYLOV_DOT, {r0_.id(), r_.id()});
    queue(c);
    return combine({&c})[0];
  }

  bool iterate(int k, double target, std::vector<double> &hist) {
    if (k == 0)
      queue(plans(SB_KRYLOV_XPBY, {p_.id(), r_.id()}));
    else
      queue(plans(SB_KRYLOV_BICG_P, {p_.id(), r_.id(), v_.id()}), (rho_ / rho_prev_) * (alpha_ / omega_), omega_);
    precondition(phat_, p_);
    apply_A(v_, phat_);
    Cache &rv = plans(SB_KRYLOV_DOT, {r0_.id(), v_.id()});
    queue(rv);
    const double sigma = combine({&rv})[0];
    if (sigma == 0.0 || !std::isfinite(sigma)) {
      breakdown_ = k;
      return false;
    }
    const double alpha = rho_ / sigma;
    Cache &half = plans(SB_KRYLOV_UPDATE, {x_.id(), phat_.id(), r_.id(), v_.id()});
    queue(half, alpha);
    precondition(shat_, r_);
    apply_A(t_, shat_);
    // <t, r> and <t, t>: one two-pair DOT in double, two one-pair DOTs in float (DESIGN.md section 2.13); exact either way.
    // One wait gathers them with <s, s> from the half step.
    std::vector<double> s;
    if (sizeof(T) == 4) {
      Cache &tr = plans(SB_KRYLOV_DOT, {t_.id(), r_.id()}), &tt = plans(SB_KRYLOV_DOT, {t_.id(), t_.id()});
      queue(tr);
      queue(tt);
      s = combine({&half, &tr, &tt});
    } else {
      Cache &trt = plans(SB_KRYLOV_DOT, {t_.id(), r_.id(), t_.id()});
      queue(trt);
      s = combine({&half, &trt});
    }
    const double t_r = s[1], t_t = s[2];
    hist.push_back(std::sqrt(s[0]));
    if (hist.back() <= target) return false;
    const double omega = t_t != 0.0 ? t_r / t_t : 0.0;
    if (t_t == 0.0 || omega == 0.0 || !std::isfinite(omega)) {
      breakdown_ = k;
      return false;
    }
    Cache &full = plans(SB_KRYLOV_UPDATE, {x_.id(), shat_.id(), r_.id(), t_.id(), r0_.id()});
    queue(full, omega);
    const std::vector<double> rr = combine({&full});
    hist.back() = std::sqrt(rr[0]);
    rho_prev_ = rho_;
    rho_ = rr[1];
    alpha_ = alpha;
    omega_ = omega;
    if (hist.back() <= target) return false;
    if (rho_ == 0.0 || !std::isfinite(rho_)) {
      breakdown_ = k;
      return false;
    }
    return true;
  }
};

} // namespace stencil
