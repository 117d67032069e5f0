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
// and for <r, r>, <r0, r>); every pass looks its buffers up for the current swap parity.  A breakdown (<r0, v> zero or
// not finite, <t, t> zero, omega zero or not finite, a new <r0, r> zero or not finite) is not fatal: solve() returns the
// history so far and breakdown() names the iteration.  Building, solve(), residual_norm() and update_coefficients() are
// collective under MPI.
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

template <typename T> class BiCGStab {
public:
  BiCGStab(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> r0, DataHandle<T> p, DataHandle<T> v,
           DataHandle<T> phat, DataHandle<T> shat, DataHandle<T> t, const std::function<LinearStencil(int)> &op_at, int nu1 = 2, int nu2 = 2,
           int coarse_sweeps = 30, int levels = 0)
      : dd_(dd), x_(x), f_(f), r_(r), r0_(r0), p_(p), v_(v), phat_(phat), shat_(shat), t_(t) {
    init(op_at, {}, {}, nu1, nu2, coarse_sweeps, levels);
  }
  BiCGStab(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> r0, DataHandle<T> p, DataHandle<T> v,
           DataHandle<T> phat, DataHandle<T> shat, DataHandle<T> t, const std::function<LinearStencil(int)> &op_at, const std::vector<DataHandle<T>> &coefs,
           const std::vector<std::string> &coef_kinds, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : dd_(dd), x_(x), f_(f), r_(r), r0_(r0), p_(p), v_(v), phat_(phat), shat_(shat), t_(t) {
    init(op_at, coefs, coef_kinds, nu1, nu2, coarse_sweeps, levels);
  }

  // the iteration at which the last solve() broke down, or -1
  int breakdown() const { return breakdown_; }
  Multigrid<T> *preconditioner() { return mg_.get(); }

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

  // the true ||f - A x||_2 (the residual into r, then an exact dot)
  double residual_norm() {
    if (coefs_.empty())
      dd_.apply(res_, curr(r_), x_, curr(f_));
    else
      dd_.apply(res_, curr(r_), x_, curr(f_), coefs_);
    return std::sqrt(dd_.dot(r_, r_));
  }

  // re-coarsen the preconditioner's coefficient fields after they change (A on the fine level reads them directly)
  void update_coefficients() { mg_->update_coefficients(); }

private:
  DistributedDomain &dd_;
  DataHandle<T> x_, f_, r_, r0_, p_, v_, phat_, shat_, t_;
  std::vector<DataHandle<T>> coefs_;
  LinearStencil A_, res_;
  std::unique_ptr<Multigrid<T>> mg_;
  int breakdown_ = -1;
  double rho_ = 0, rho_prev_ = 0, alpha_ = 0, omega_ = 0;

  static BC homogeneous(const BC &bc) {
    return bc.kind == BC::Kind::ODD ? BC::ODD(0.0) : bc.kind == BC::Kind::EVEN ? BC::EVEN() : BC::VALUE(0.0);
  }

  void init(const std::function<LinearStencil(int)> &op_at, const std::vector<DataHandle<T>> &coefs, const std::vector<std::string> &coef_kinds, int nu1,
            int nu2, int coarse_sweeps, int levels) {
    const int dtype = bc_dtype<T>();
    if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL("BiCGStab: the quantities must be float or double");
    if (dd_.domains_.empty()) LOG_FATAL("BiCGStab: dd must be realized");
    const std::vector<std::pair<const char *, size_t>> named{{"x", x_.id()},       {"f", f_.id()},       {"r", r_.id()}, {"r0", r0_.id()}, {"p", p_.id()},
                                                             {"v", v_.id()},       {"phat", phat_.id()}, {"shat", shat_.id()}, {"t", t_.id()}};
    for (size_t i = 0; i < named.size(); ++i)
      for (size_t j = 0; j < i; ++j)
        if (named[i].second == named[j].second) LOG_FATAL("BiCGStab: " << named[i].first << " and " << named[j].first << " must be different quantities");
    for (size_t k = 0; k < coefs.size(); ++k)
      for (const auto &n : named)
        if (coefs[k].id() == n.second) LOG_FATAL("BiCGStab: coefficient " << k << " must be a quantity other than the nine vectors");
    static const char *const kFace[6] = {"-x", "+x", "-y", "+y", "-z", "+z"};
    for (int fc = 0; fc < 6; ++fc) {
      if (dd_.boundary_[fc / 2] != Topology::Boundary::FIXED) continue;
      auto bx = dd_.bcs_.find(std::make_pair(x_.id(), fc));
      if (bx == dd_.bcs_.end() || bx->second.kind == BC::Kind::NONE)
        LOG_FATAL("BiCGStab: x needs a boundary condition (ODD, EVEN or VALUE) on every FIXED face (face " << kFace[fc] << ")");
      const BC want = homogeneous(bx->second);
      for (const auto &w : {std::make_pair("phat", phat_.id()), std::make_pair("shat", shat_.id())}) {
        auto it = dd_.bcs_.find(std::make_pair(w.second, fc));
        const BC got = it == dd_.bcs_.end() ? BC::NONE() : it->second;
        if (got.kind != want.kind || got.value != want.value)
          LOG_FATAL("BiCGStab: " << w.first << " needs the homogeneous counterpart of x's BC on face " << kFace[fc] << " (kind " << int(want.kind)
                                 << ", value 0), not kind " << int(got.kind) << ", value " << got.value);
      }
    }
    A_ = op_at(0);
    if (A_.has_aux()) LOG_FATAL("BiCGStab: op_at(0) has an aux term; A reads x only");
    if (size_t(A_.ncoef()) != coefs.size())
      LOG_FATAL("BiCGStab: op_at(0) reads " << A_.ncoef() << " coefficient fields, but " << coefs.size() << " were given");
    res_ = Multigrid<T>::residual(A_);
    coefs_ = coefs;
    dd_.create_apply_streams();
    if (coefs.empty())
      mg_.reset(new Multigrid<T>(dd_, phat_, p_, v_, op_at, nu1, nu2, coarse_sweeps, levels));
    else
      mg_.reset(new Multigrid<T>(dd_, phat_, p_, v_, op_at, coefs, coef_kinds, nu1, nu2, coarse_sweeps, levels));
    mg_->pair_level(shat_, r_); // the second pair's checks, now rather than at the first solve
  }

  void queued(bool on) {
    dd_.queued_ = on;
    for (auto &L : mg_->levels_) L.dd->queued_ = on;
  }

  void apply_A(DataHandle<T> out, DataHandle<T> src) {
    if (coefs_.empty())
      dd_.apply(A_, curr(out), src);
    else
      dd_.apply(A_, curr(out), src, coefs_);
  }

  // u = M f: u set to +0 (a memset of the curr allocation; the cycle's exchanges refill the ghost cells), then one
  // queued cycle on the pair (u, f)
  void precondition(DataHandle<T> u, DataHandle<T> f) {
    dd_.queue_after_exterior();
    for (size_t di = 0; di < dd_.domains_.size(); ++di) {
      LocalDomain &d = dd_.domains_[di];
      d.set_device();
      const cudaPitchedPtr pp = d.curr_data(u.id());
      CUDA_RUNTIME(cudaMemsetAsync(pp.ptr, 0, pp.pitch * pp.ysize * size_t(d.raw_size().z), dd_.applyStreams_[2 * di]));
    }
    mg_->vcycle(0, &mg_->pair_level(u, f));
  }

  // r = f - A x (x's own BC through the exchange), r0 = r; returns <r0, r>
  double start() {
    queued(true);
    if (coefs_.empty())
      dd_.apply(res_, curr(r_), x_, curr(f_));
    else
      dd_.apply(res_, curr(r_), x_, curr(f_), coefs_);
    dd_.krylov_launch(dd_.krylov_plans(SB_KRYLOV_XPBY, {r0_.id(), r_.id()}), 0.0, true);
    DistributedDomain::KrylovCache &c = dd_.krylov_plans(SB_KRYLOV_DOT, {r0_.id(), r_.id()});
    dd_.krylov_launch(c, 0.0, true);
    return dd_.krylov_sums(c, true)[0];
  }

  bool iterate(int k, double target, std::vector<double> &hist) {
    if (k == 0)
      dd_.krylov_launch(dd_.krylov_plans(SB_KRYLOV_XPBY, {p_.id(), r_.id()}), 0.0, true);
    else
      dd_.krylov_launch(dd_.krylov_plans(SB_KRYLOV_BICG_P, {p_.id(), r_.id(), v_.id()}), (rho_ / rho_prev_) * (alpha_ / omega_), omega_, true);
    precondition(phat_, p_);
    apply_A(v_, phat_);
    DistributedDomain::KrylovCache &rv = dd_.krylov_plans(SB_KRYLOV_DOT, {r0_.id(), v_.id()});
    dd_.krylov_launch(rv, 0.0, true);
    const double sigma = dd_.krylov_sums(rv, true)[0];
    if (sigma == 0.0 || !std::isfinite(sigma)) {
      breakdown_ = k;
      return false;
    }
    const double alpha = rho_ / sigma;
    DistributedDomain::KrylovCache &half = dd_.krylov_plans(SB_KRYLOV_UPDATE, {x_.id(), phat_.id(), r_.id(), v_.id()});
    dd_.krylov_launch(half, alpha, true);
    precondition(shat_, r_);
    apply_A(t_, shat_);
    // <t, r> and <t, t>: one two-pair DOT in double, two one-pair DOTs in float (DESIGN.md section 2.13); exact either way
    double t_r, t_t;
    if (sizeof(T) == 4) {
      DistributedDomain::KrylovCache &tr = dd_.krylov_plans(SB_KRYLOV_DOT, {t_.id(), r_.id()});
      DistributedDomain::KrylovCache &tt = dd_.krylov_plans(SB_KRYLOV_DOT, {t_.id(), t_.id()});
      dd_.krylov_launch(tr, 0.0, true);
      dd_.krylov_launch(tt, 0.0, true);
      t_r = dd_.krylov_sums(tr, true)[0];
      t_t = dd_.krylov_sums(tt, true)[0];
    } else {
      DistributedDomain::KrylovCache &trt = dd_.krylov_plans(SB_KRYLOV_DOT, {t_.id(), r_.id(), t_.id()});
      dd_.krylov_launch(trt, 0.0, true);
      const std::vector<double> s = dd_.krylov_sums(trt, true);
      t_r = s[0];
      t_t = s[1];
    }
    hist.push_back(std::sqrt(dd_.krylov_sums(half, true)[0]));
    if (hist.back() <= target) return false;
    const double omega = t_t != 0.0 ? t_r / t_t : 0.0;
    if (t_t == 0.0 || omega == 0.0 || !std::isfinite(omega)) {
      breakdown_ = k;
      return false;
    }
    DistributedDomain::KrylovCache &full = dd_.krylov_plans(SB_KRYLOV_UPDATE, {x_.id(), shat_.id(), r_.id(), t_.id(), r0_.id()});
    dd_.krylov_launch(full, omega, true);
    const std::vector<double> rr = dd_.krylov_sums(full, true);
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

  // the end of a queued solve: every apply stream and exchange complete
  void finish() {
    queued(false);
    for (size_t i = 0; i < dd_.applyStreams_.size(); ++i) {
      CUDA_RUNTIME(cudaSetDevice(dd_.domains_[i / 2].gpu()));
      CUDA_RUNTIME(cudaStreamSynchronize(dd_.applyStreams_[i]));
    }
    dd_.exchange_wait();
    for (auto &L : mg_->levels_) L.dd->exchange_wait();
  }
};

} // namespace stencil
