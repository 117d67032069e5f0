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
// apply streams and waits on the host three times, for beta, alpha and the stopping test; each wait gathers every sum
// it needs in one exchange (in float, where gamma and delta come from two one-pair DOTs, both DOTs' parts).  Every pass
// looks its buffers up for the current swap parity, so dd.swap() may be called between solves.  A breakdown (a
// non-positive or non-finite <p, A p>, or a non-finite <z, r>) is not fatal: solve() returns the history so far and
// breakdown() names the iteration.  Building, solve(), residual_norm() and update_coefficients() are collective under
// MPI.
//
// detail::KrylovSolver holds what PCG and BiCGStab (bicgstab.hpp) share: the refusals, A and its residual, the
// Multigrid preconditioner, and the queued passes with their host waits.
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
namespace detail {

template <typename T> class KrylovSolver {
public:
  // the iteration at which the last solve() broke down, or -1
  int breakdown() const { return breakdown_; }
  Multigrid<T> *preconditioner() { return mg_.get(); }

  // the true ||f - A x||_2 (the residual into r, then an exact dot)
  double residual_norm() {
    dd_.apply(res_, curr(r_), x_, curr(f_), coefs_);
    return std::sqrt(dd_.dot(r_, r_));
  }

  // re-coarsen the preconditioner's coefficient fields after they change (A on the fine level reads them directly)
  void update_coefficients() {
    if (mg_) mg_->update_coefficients();
  }

protected:
  using Named = std::vector<std::pair<const char *, size_t>>;
  using Pairs = std::vector<std::pair<DataHandle<T>, DataHandle<T>>>;
  using Cache = DistributedDomain::KrylovCache;

  KrylovSolver(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r) : dd_(dd), x_(x), f_(f), r_(r) {}

  DistributedDomain &dd_;
  DataHandle<T> x_, f_, r_;
  std::vector<DataHandle<T>> coefs_;
  LinearStencil A_, res_;
  std::unique_ptr<Multigrid<T>> mg_;
  int breakdown_ = -1;

  // The refusals of solver `who` (LOG_FATAL, before any domain is built), then the preconditioner.  named: every vector
  // by name; applied: those A is applied to, which carry the homogeneous counterpart of x's BC on every FIXED face.
  // pairs: the (u, f) pairs M runs on, none without a preconditioner; the Multigrid is built on the first with the
  // scratch r, and the others are checked now rather than at the first solve.
  void init(const char *who, const Named &named, const Named &applied, const std::function<LinearStencil(int)> &op_at,
            const std::vector<DataHandle<T>> &coefs, const std::vector<std::string> &coef_kinds, const Pairs &pairs, DataHandle<T> scratch, int nu1,
            int nu2, int coarse_sweeps, int levels) {
    const int dtype = bc_dtype<T>();
    if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL(who << ": the quantities must be float or double");
    if (dd_.domains_.empty()) LOG_FATAL(who << ": dd must be realized");
    std::string names;
    for (size_t i = 0; i < named.size(); ++i) {
      for (size_t j = 0; j < i; ++j)
        if (named[i].second == named[j].second) LOG_FATAL(who << ": " << named[i].first << " and " << named[j].first << " must be different quantities");
      names += (i ? ", " : "") + std::string(named[i].first);
    }
    for (size_t k = 0; k < coefs.size(); ++k)
      for (const auto &n : named)
        if (coefs[k].id() == n.second) LOG_FATAL(who << ": coefficient " << k << " must be a quantity other than " << names);
    static const char *const kFace[6] = {"-x", "+x", "-y", "+y", "-z", "+z"};
    for (int fc = 0; fc < 6; ++fc) {
      if (dd_.boundary_[fc / 2] != Topology::Boundary::FIXED) continue;
      auto bx = dd_.bcs_.find(std::make_pair(x_.id(), fc));
      if (bx == dd_.bcs_.end() || bx->second.kind == BC::Kind::NONE)
        LOG_FATAL(who << ": x needs a boundary condition (ODD, EVEN or VALUE) on every FIXED face (face " << kFace[fc] << ")");
      const BC want = bx->second.kind == BC::Kind::ODD ? BC::ODD(0.0) : bx->second.kind == BC::Kind::EVEN ? BC::EVEN() : BC::VALUE(0.0);
      for (const auto &v : applied) {
        auto it = dd_.bcs_.find(std::make_pair(v.second, fc));
        const BC got = it == dd_.bcs_.end() ? BC::NONE() : it->second;
        if (got.kind != want.kind || got.value != want.value)
          LOG_FATAL(who << ": " << v.first << " needs the homogeneous counterpart of x's BC on face " << kFace[fc] << " (kind " << int(want.kind)
                        << ", value 0), not kind " << int(got.kind) << ", value " << got.value);
      }
    }
    A_ = op_at(0);
    if (A_.has_aux()) LOG_FATAL(who << ": op_at(0) has an aux term; A reads x only");
    if (size_t(A_.ncoef()) != coefs.size())
      LOG_FATAL(who << ": op_at(0) reads " << A_.ncoef() << " coefficient fields, but " << coefs.size() << " were given");
    res_ = Multigrid<T>::residual(A_);
    coefs_ = coefs;
    dd_.create_apply_streams();
    if (pairs.empty()) return;
    mg_.reset(new Multigrid<T>(dd_, pairs[0].first, pairs[0].second, scratch, op_at, coefs, coef_kinds, nu1, nu2, coarse_sweeps, levels));
    for (size_t i = 1; i < pairs.size(); ++i) mg_->pair_level(pairs[i].first, pairs[i].second);
  }

  // the queued passes: plans of dd's cache for the current swap parity, one launch per local domain on its interior
  // apply stream, and the host wait that gathers the sums of several launched caches in one exchange
  Cache &plans(int mode, const std::vector<size_t> &qs) { return dd_.krylov_plans(mode, qs); }
  void queue(Cache &c, double s = 0.0, double t = 0.0) { dd_.krylov_launch(c, s, t, true); }
  std::vector<double> combine(const std::vector<Cache *> &cs) { return dd_.krylov_sums(cs, true); }

  // dd and, with a preconditioner, its coarse levels queue their work (or stop queueing it)
  void queued(bool on) {
    if (mg_)
      mg_->set_queued(on);
    else
      dd_.queued_ = on;
  }

  // the start of a queued solve: the coefficient fields exchanged (once per solve: every later exchange moves only the
  // vector A reads, DESIGN.md section 2.15), then r = f - A x (x's own BC through the exchange)
  void queue_residual() {
    queued(true);
    if (!coefs_.empty()) dd_.queue_exchange(Multigrid<T>::set_of(coefs_));
    dd_.apply(res_, curr(r_), x_, curr(f_), coefs_, Multigrid<T>::only(x_));
  }

  void apply_A(DataHandle<T> out, DataHandle<T> src) { dd_.apply(A_, curr(out), src, coefs_, Multigrid<T>::only(src)); }

  // u = M f: u set to +0 (the cycle's exchanges refill the ghost cells), then one queued cycle on the pair (u, f)
  void precondition(DataHandle<T> u, DataHandle<T> f) {
    dd_.clear_queued(u.id());
    mg_->vcycle(0, &mg_->pair_level(u, f));
  }

  // the end of a queued solve: every apply stream and exchange complete (the preconditioner's finish covers dd, its
  // finest level)
  void finish() {
    if (mg_) {
      mg_->finish();
      return;
    }
    queued(false);
    DistributedDomain::wait_queued({&dd_});
  }
};

} // namespace detail

template <typename T> class PCG : public detail::KrylovSolver<T> {
  using B = detail::KrylovSolver<T>;
  using typename B::Cache;
  using B::dd_;
  using B::x_;
  using B::f_;
  using B::r_;
  using B::mg_;
  using B::breakdown_;
  using B::plans;
  using B::queue;
  using B::combine;
  using B::queue_residual;
  using B::apply_A;
  using B::precondition;
  using B::finish;

public:
  PCG(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> z, DataHandle<T> p, DataHandle<T> q,
      const std::function<LinearStencil(int)> &op_at, bool precond = true, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : PCG(dd, x, f, r, z, p, q, op_at, {}, {}, precond, nu1, nu2, coarse_sweeps, levels) {}
  PCG(DistributedDomain &dd, DataHandle<T> x, DataHandle<T> f, DataHandle<T> r, DataHandle<T> z, DataHandle<T> p, DataHandle<T> q,
      const std::function<LinearStencil(int)> &op_at, const std::vector<DataHandle<T>> &coefs, const std::vector<std::string> &coef_kinds,
      bool precond = true, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : B(dd, x, f, r), z_(precond ? z : r), p_(p), q_(q) {
    typename B::Named named{{"x", x.id()}, {"f", f.id()}, {"r", r.id()}, {"p", p.id()}, {"q", q.id()}}, applied{{"p", p.id()}};
    typename B::Pairs pairs;
    if (precond) {
      named.push_back({"z", z.id()});
      applied.push_back({"z", z.id()});
      pairs.push_back({z, r});
    }
    this->init("PCG", named, applied, op_at, coefs, coef_kinds, pairs, q, nu1, nu2, coarse_sweeps, levels);
  }

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

private:
  DataHandle<T> z_, p_, q_;
  double eta_ = 0;

  // r = f - A x; returns <r, r>
  double start() {
    queue_residual();
    Cache &c = plans(SB_KRYLOV_DOT, {r_.id(), r_.id()});
    queue(c);
    return combine({&c})[0];
  }

  bool iterate(int k, double &rho) {
    if (mg_) precondition(z_, r_);
    // <z, r> and <z, q>: one two-pair DOT in double (3 reads instead of 4); in float the two-pair kernel is bound by its
    // per-cell work and two one-pair launches are faster (DESIGN.md section 2.13).  The sums are exact either way.
    std::vector<double> gd;
    if (k == 0) {
      Cache &zr = plans(SB_KRYLOV_DOT, {z_.id(), r_.id()});
      queue(zr);
      gd = combine({&zr});
    } else if (sizeof(T) == 4) {
      Cache &zr = plans(SB_KRYLOV_DOT, {z_.id(), r_.id()});
      queue(zr);
      Cache &zq = plans(SB_KRYLOV_DOT, {z_.id(), q_.id()});
      queue(zq);
      gd = combine({&zr, &zq});
    } else {
      Cache &zrq = plans(SB_KRYLOV_DOT, {z_.id(), r_.id(), q_.id()});
      queue(zrq);
      gd = combine({&zrq});
    }
    const double gamma = gd[0];
    if (!std::isfinite(gamma)) {
      breakdown_ = k;
      return false;
    }
    queue(plans(SB_KRYLOV_XPBY, {p_.id(), z_.id()}), k == 0 ? 0.0 : -gd[1] / eta_);
    apply_A(q_, p_);
    Cache &pq = plans(SB_KRYLOV_DOT, {p_.id(), q_.id()});
    queue(pq);
    const double eta = combine({&pq})[0];
    if (!(std::isfinite(eta) && eta > 0.0)) {
      breakdown_ = k;
      return false;
    }
    eta_ = eta;
    Cache &up = plans(SB_KRYLOV_UPDATE, {x_.id(), p_.id(), r_.id(), q_.id()});
    queue(up, gamma / eta);
    rho = combine({&up})[0];
    return true;
  }
};

} // namespace stencil
