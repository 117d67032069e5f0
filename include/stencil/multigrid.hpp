// Geometric multigrid for A u = f on a DistributedDomain (DESIGN.md section 2.11), the C++ twin of
// stencil_b200.Multigrid: V(nu1, nu2) cycles over coarsenings by 2, built from the coloured sweeps (section 2.9), the
// fused residual-restriction and the prolongation, queued on CUDA events with one host wait per cycle.
//
//     stencil::Multigrid<double> mg(dd, u, f, r, [&](int l) { return A(l); });   // A on level l, l = 0 finest
//     std::vector<double> history = mg.solve(1e-8, 20);                          // ||f - A u||_2 per cycle
//
// u, f and r are quantities of the realized domain dd (r: scratch for the residual norm).  Each coarse level is a
// DistributedDomain of u and f on the same GPUs, placement and boundary kinds, with dd's radius raised to >= 1 in all 26
// directions; the grid is halved while every subdomain extent is even and its half >= 2, at most `levels` grids (0: no
// cap).  Coarse u takes ODD(0) where u has ODD(c) and EVEN where u has EVEN; VALUE, a FIXED face without a BC on u, a
// grid that cannot be coarsened once, an op with aux terms (or coefficient terms without coefs) or of reach > 1 are
// refused (LOG_FATAL) before
// any domain is built.  The smoother is red-black Gauss-Seidel if every level's A passes the red-black colour check,
// else 8-colour.  Building, cycle() and solve() are collective under MPI.  Periodic Poisson needs f of zero mean.
//
// Variable coefficients (DESIGN.md section 2.12): the constructor taking coefs and coef_kinds accepts ops with
// coefficient terms, such as -div(kappa grad u) with kappa on faces in three quantities.  Kind "x", "y" or "z" marks a
// face field (coarsened by the face restriction), "cell" a cell-centred one (the 8-cell restriction).  Each coarse level
// holds one quantity per field with the fine field's BC on every FIXED face (a field without one is refused).
// Coefficient ops are smoothed by the diagonal relaxation (DistributedDomain::relax, omega = 1) and their residual goes
// through the fused coefficient restriction; update_coefficients() re-coarsens every level from the fine fields.
//     stencil::Multigrid<double> mg(dd, u, f, r, [&](int l) { return A(l); }, {kx, ky, kz}, {"x", "y", "z"});
//
// cycle(u2, f2) runs the cycle on another fine-level pair through the same coarse levels and coarse coefficient fields
// (DESIGN.md section 2.14): u2 and f2 are two different quantities of dd of type T, not coefficient fields, and u2
// carries the constructor u's BC on every FIXED face (the coarse walls derive from it); the cycle is then the bits of one
// on a Multigrid built on (u2, f2).
#pragma once

#include <cmath>
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "stencil/linear_stencil.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

namespace stencil {

template <typename T> class Multigrid {
  friend class detail::KrylovSolver<T>; // queues this solver's cycles as the preconditioner of PCG and BiCGStab

public:
  Multigrid(DistributedDomain &dd, DataHandle<T> u, DataHandle<T> f, DataHandle<T> r, const std::function<LinearStencil(int)> &op_at, int nu1 = 2,
            int nu2 = 2, int coarse_sweeps = 30, int levels = 0)
      : nu1_(nu1), nu2_(nu2), coarse_sweeps_(coarse_sweeps), r_(r) {
    init(dd, u, f, op_at, levels, {}, {});
  }
  Multigrid(DistributedDomain &dd, DataHandle<T> u, DataHandle<T> f, DataHandle<T> r, const std::function<LinearStencil(int)> &op_at,
            const std::vector<DataHandle<T>> &coefs, const std::vector<std::string> &coef_kinds, int nu1 = 2, int nu2 = 2, int coarse_sweeps = 30,
            int levels = 0)
      : nu1_(nu1), nu2_(nu2), coarse_sweeps_(coarse_sweeps), r_(r) {
    init(dd, u, f, op_at, levels, coefs, coef_kinds);
  }

  size_t num_levels() const { return levels_.size(); }
  int colours() const { return colours_; }

  // One V(nu1, nu2) cycle, queued after the work on the legacy default stream; returns when it is complete.
  void cycle() {
    set_queued(true);
    fine_coefs_current();
    vcycle(0);
    finish();
  }

  // The same cycle on the fine-level pair (u, f) instead of the constructor's (see the header comment).
  void cycle(DataHandle<T> u, DataHandle<T> f) {
    Level &top = pair_level(u, f);
    set_queued(true);
    fine_coefs_current();
    vcycle(0, &top);
    finish();
  }

  // Re-coarsen every level's coefficient fields from the current fine ones, level by level, queued like a cycle with one
  // host wait.  The constructor calls it once; call it again whenever the fine fields change.  It then exchanges the
  // fields of every level: a cycle exchanges only the vector each call reads at an offset (DESIGN.md section 2.15), never
  // a coefficient field, so after a cycle the ghost cells of the other quantities are not refreshed as a side effect.
  void update_coefficients() {
    set_queued(true);
    for (size_t l = 0; l + 1 < levels_.size(); ++l)
      for (size_t k = 0; k < axes_.size(); ++k) {
        Level &F = levels_[l], &C = levels_[l + 1];
        if (axes_[k] >= 0)
          F.dd->restrict_to(*C.dd, curr(C.coefs[k]), curr(F.coefs[k]), axes_[k]);
        else
          F.dd->restrict_to(*C.dd, curr(C.coefs[k]), curr(F.coefs[k]));
      }
    for (Level &L : levels_)
      if (!L.coefs.empty()) L.dd->queue_exchange(set_of(L.coefs));
    coefParity_ = levels_[0].dd->parity_;
    finish();
  }

  // ||f - A u||_2: the residual into r and an exact reduction, the same on every rank and partition
  double residual_norm() {
    Level &L = levels_[0];
    L.dd->apply(L.res, curr(r_), L.u, curr(L.f), L.coefs);
    return std::sqrt(L.dd->reduce(r_, Which::curr, Sum::exact).sumsq);
  }

  // cycles until ||f - A u||_2 <= rtol ||f||_2 or max_cycles; the norm before the first cycle and after each
  std::vector<double> solve(double rtol, int max_cycles) {
    Level &L = levels_[0];
    const double target = rtol * std::sqrt(L.dd->reduce(L.f, Which::curr, Sum::exact).sumsq);
    std::vector<double> hist{residual_norm()};
    while (hist.back() > target && int(hist.size()) - 1 < max_cycles) {
      cycle();
      hist.push_back(residual_norm());
    }
    return hist;
  }

private:
  struct Level {
    DistributedDomain *dd;
    std::unique_ptr<DistributedDomain> owned; // the coarse levels
    DataHandle<T> u, f;
    LinearStencil A, gs, res; // gs: the SOR table of a plain op (a coefficient op is smoothed by relax)
    std::vector<DataHandle<T>> coefs;
  };
  int nu1_, nu2_, coarse_sweeps_, colours_ = 0;
  int coefParity_ = -1; // the fine swap parity the coefficient fields were last exchanged in
  DataHandle<T> r_;
  std::vector<Level> levels_;
  std::vector<int> axes_; // per coefficient field: the face axis, or -1 for a cell field
  std::vector<std::pair<int, BC>> ubcs_; // the constructor u's BC on every FIXED face
  std::vector<Level> pairs_;             // the fine levels of other pairs (cycle(u, f))

  // the fine level of the pair (u, f): the constructor's, or one sharing A, the coefficient fields and the coarse levels
  Level &pair_level(DataHandle<T> u, DataHandle<T> f) {
    Level &L0 = levels_[0];
    if (u.id() == L0.u.id() && f.id() == L0.f.id()) return L0;
    for (Level &P : pairs_)
      if (P.u.id() == u.id() && P.f.id() == f.id()) return P;
    DistributedDomain &dd = *L0.dd;
    if (u.id() == f.id()) LOG_FATAL("Multigrid::cycle: u and f must be two different quantities");
    for (size_t q : {u.id(), f.id()})
      if (q >= dd.dataDtype_.size() || dd.dataDtype_[q] != bc_dtype<T>()) LOG_FATAL("Multigrid::cycle: u and f must be quantities of dd of the constructor u's type");
    for (const DataHandle<T> &k : L0.coefs)
      if (k.id() == u.id() || k.id() == f.id()) LOG_FATAL("Multigrid::cycle: u and f must not be coefficient fields");
    for (const auto &w : ubcs_) {
      auto it = dd.bcs_.find(std::make_pair(u.id(), w.first));
      const BC got = it == dd.bcs_.end() ? BC::NONE() : it->second;
      if (got.kind != w.second.kind || got.value != w.second.value)
        LOG_FATAL("Multigrid::cycle: u needs the constructor u's BC on every FIXED face (face " << w.first << ": kind " << int(w.second.kind) << ", value "
                                                                                                << w.second.value << ", not kind " << int(got.kind) << ", value "
                                                                                                << got.value << ")");
    }
    pairs_.push_back(Level{&dd, nullptr, u, f, L0.A, L0.gs, L0.res, L0.coefs});
    return pairs_.back();
  }

  void init(DistributedDomain &dd, DataHandle<T> u, DataHandle<T> f, const std::function<LinearStencil(int)> &op_at, int levels,
            const std::vector<DataHandle<T>> &coefs, const std::vector<std::string> &coef_kinds) {
    const DataHandle<T> r = r_;
    const int nu1 = nu1_, nu2 = nu2_, coarse_sweeps = coarse_sweeps_;
    const int dtype = bc_dtype<T>();
    if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL("Multigrid: u, f and r must be float or double");
    if (dd.domains_.empty()) LOG_FATAL("Multigrid: dd must be realized");
    if (u.id() == f.id() || u.id() == r.id() || f.id() == r.id()) LOG_FATAL("Multigrid: u, f and r must be three different quantities");
    if (nu1 < 0 || nu2 < 0 || coarse_sweeps < 1) LOG_FATAL("Multigrid: nu1 and nu2 must be >= 0 and coarse_sweeps >= 1");
    if (levels == 1 || levels < 0) LOG_FATAL("Multigrid: levels must be >= 2 (or 0: no cap)");
    if (coefs.size() > 4) LOG_FATAL("Multigrid: at most 4 coefficient fields");
    if (coef_kinds.size() != coefs.size()) LOG_FATAL("Multigrid: coef_kinds must name one of x, y, z, cell per coefficient field");
    for (size_t k = 0; k < coefs.size(); ++k) {
      const std::string &kind = coef_kinds[k];
      if (kind != "x" && kind != "y" && kind != "z" && kind != "cell")
        LOG_FATAL("Multigrid: coef_kinds must name one of x, y, z, cell per coefficient field, not " << kind);
      axes_.push_back(kind == "cell" ? -1 : kind[0] - 'x');
      const size_t q = coefs[k].id();
      if (q == u.id() || q == f.id() || q == r.id()) LOG_FATAL("Multigrid: coefficient " << k << " must be a quantity other than u, f and r");
      for (size_t j = 0; j < k; ++j)
        if (coefs[j].id() == q) LOG_FATAL("Multigrid: the coefficient fields must be different quantities");
    }
    // the coarse BCs of u
    std::vector<std::pair<int, BC>> walls;
    for (int fc = 0; fc < 6; ++fc) {
      if (dd.boundary_[fc / 2] != Topology::Boundary::FIXED) continue;
      auto it = dd.bcs_.find(std::make_pair(u.id(), fc));
      const int kind = it == dd.bcs_.end() ? SB_BC_NONE : int(it->second.kind);
      if (kind == SB_BC_VALUE) LOG_FATAL("Multigrid: VALUE walls are not consistent across levels (DESIGN.md section 2.10); use ODD(c)");
      if (kind == SB_BC_NONE) LOG_FATAL("Multigrid: u needs a boundary condition (ODD or EVEN) on every FIXED face");
      walls.push_back(std::make_pair(fc, kind == SB_BC_ODD ? BC::ODD(0.0) : BC::EVEN()));
      ubcs_.push_back(std::make_pair(fc, it->second));
    }
    // every coefficient field's BCs, kept on every level
    std::vector<std::vector<std::pair<int, BC>>> coef_walls(coefs.size());
    for (int fc = 0; fc < 6; ++fc) {
      if (dd.boundary_[fc / 2] != Topology::Boundary::FIXED) continue;
      for (size_t k = 0; k < coefs.size(); ++k) {
        auto it = dd.bcs_.find(std::make_pair(coefs[k].id(), fc));
        if (it == dd.bcs_.end() || it->second.kind == BC::Kind::NONE)
          LOG_FATAL("Multigrid: coefficient " << k << " needs a boundary condition on every FIXED face");
        coef_walls[k].push_back(std::make_pair(fc, it->second));
      }
    }
    // the number of grids: every subdomain extent (global information, the same verdict on every rank)
    const Dim3 dim = dd.placement_->dim();
    int nlev = 1;
    for (int64_t step = 1; levels == 0 || nlev < levels; step *= 2, ++nlev) {
      bool ok = true;
      for (int64_t z = 0; z < dim.z && ok; ++z)
        for (int64_t y = 0; y < dim.y && ok; ++y)
          for (int64_t x = 0; x < dim.x && ok; ++x) {
            const Dim3 s = dd.placement_->subdomain_size(Dim3(x, y, z));
            for (int64_t v : {s.x, s.y, s.z}) ok = ok && v % (2 * step) == 0 && v / (2 * step) >= 2;
          }
      if (!ok) break;
    }
    if (nlev < 2) LOG_FATAL("Multigrid: the grid cannot be coarsened once: every subdomain extent must be even and >= 4");
    Radius cr = dd.radius_;
    for (int z = -1; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x)
          if (x || y || z) cr.dir(x, y, z) = std::max<size_t>(cr.dir(x, y, z), 1);
    std::vector<LinearStencil> ops;
    for (int l = 0; l < nlev; ++l) {
      ops.push_back(op_at(l));
      const LinearStencil &A = ops.back();
      if (A.has_aux() || (A.ncoef() > 0 && coefs.empty())) LOG_FATAL("Multigrid: op_at(" << l << ") has coefficient or aux terms");
      if (!coefs.empty() && size_t(A.ncoef()) != coefs.size())
        LOG_FATAL("Multigrid: op_at(" << l << ") reads " << A.ncoef() << " coefficient fields, but " << coefs.size() << " were given");
      bool centre = false;
      for (const sb_stencil_vterm &t : A.vterms()) {
        centre = centre || (!t.offset[0] && !t.offset[1] && !t.offset[2]);
        for (int a = 0; a < 3; ++a)
          if (t.offset[a] < -1 || t.offset[a] > 1) LOG_FATAL("Multigrid: op_at(" << l << ") reaches beyond 1 cell");
      }
      if (A.ncoef() > 0 && !centre) LOG_FATAL("Multigrid: op_at(" << l << ") has no term at offset (0, 0, 0)");
    }
    for (int m : {2, 8}) {
      bool ok = true;
      for (int l = 0; l < nlev && ok; ++l) {
        int64_t r27[27];
        const Radius &rad = l == 0 ? dd.radius_ : cr;
        for (int z = -1, i = 0; z <= 1; ++z)
          for (int y = -1; y <= 1; ++y)
            for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(rad.dir(x, y, z));
        ok = SB_OK == sb_stencil_ccheck(ops[l].vterms().data(), int(ops[l].vterms().size()), r27, m);
      }
      if (ok) {
        colours_ = m;
        break;
      }
    }
    if (!colours_) LOG_FATAL("Multigrid: no Gauss-Seidel colouring applies to A (or it leaves the radius)");
    dd.create_apply_streams();
    levels_.push_back(Level{&dd, nullptr, u, f, ops[0], smoother(ops[0]), residual(ops[0]), coefs});
    Dim3 size = dd.size_;
    for (int l = 1; l < nlev; ++l) {
      size = Dim3(size.x / 2, size.y / 2, size.z / 2);
      std::unique_ptr<DistributedDomain> cd(new DistributedDomain(size.x, size.y, size.z));
      if (!dd.gpus_.empty()) cd->set_gpus(dd.gpus_);
      cd->set_placement(dd.strategy_);
      cd->set_radius(cr);
      DataHandle<T> cu = cd->template add_data<T>("u"), cf = cd->template add_data<T>("f");
      std::vector<DataHandle<T>> ck;
      for (size_t k = 0; k < coefs.size(); ++k) ck.push_back(cd->template add_data<T>("coef" + std::to_string(k)));
      cd->set_boundary(dd.boundary_[0], dd.boundary_[1], dd.boundary_[2]);
      for (const auto &w : walls) cd->set_boundary_condition(cu, face_dir(w.first), w.second);
      for (size_t k = 0; k < coefs.size(); ++k)
        for (const auto &w : coef_walls[k]) cd->set_boundary_condition(ck[k], face_dir(w.first), w.second);
      cd->realize();
      // every level queues on dd's apply streams, so stream order alone orders consecutive levels
      cd->applyStreams_ = dd.applyStreams_;
      cd->sharedApplyStreams_ = true;
      levels_.push_back(Level{cd.get(), std::move(cd), cu, cf, ops[size_t(l)], smoother(ops[size_t(l)]), residual(ops[size_t(l)]), ck});
    }
    for (size_t l = 0; l + 1 < levels_.size(); ++l) levels_[l].dd->check_pairing(*levels_[l + 1].dd, true);
    if (!coefs.empty()) update_coefficients();
  }

  static Dim3 face_dir(int fc) {
    const int s = fc % 2 ? 1 : -1;
    return Dim3(fc / 2 == 0 ? s : 0, fc / 2 == 1 ? s : 0, fc / 2 == 2 ? s : 0);
  }

  static LinearStencil smoother(const LinearStencil &A) { return A.ncoef() > 0 ? LinearStencil() : A.relax(1.0); }

  // every level queues its work (or stops queueing it)
  void set_queued(bool on) {
    for (Level &L : levels_) L.dd->queued_ = on;
  }

  // the end of a queued cycle: every apply stream and exchange of every level complete
  void finish() {
    set_queued(false);
    std::vector<DistributedDomain *> doms;
    for (Level &L : levels_) doms.push_back(L.dd);
    DistributedDomain::wait_queued(doms);
  }

  // r = f - A u: (aux, 0, 1), then each term of A with its weight negated (a coefficient term keeps its field)
  static LinearStencil residual(const LinearStencil &A) {
    LinearStencil res;
    res.add(Source::aux, 0, 0, 0, 1.0);
    for (const sb_stencil_vterm &t : A.vterms())
      res.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight, t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2]);
    return res;
  }

  // the bit set of some quantities (Exchange::only): each exchange of a cycle moves the one vector its call reads at an
  // offset; the coefficient fields are exchanged by update_coefficients()
  static uint64_t set_of(const std::vector<DataHandle<T>> &hs) {
    uint64_t s = 0;
    for (const DataHandle<T> &h : hs) s |= uint64_t(1) << h.id();
    return s;
  }
  static Exchange only(DataHandle<T> h) { return Exchange::only(uint64_t(1) << h.id()); }

  // after dd.swap() the fine coefficient fields' curr buffers are the other allocation: exchange them once
  void fine_coefs_current() {
    Level &L = levels_[0];
    if (!L.coefs.empty() && coefParity_ != L.dd->parity_) {
      L.dd->queue_exchange(set_of(L.coefs));
      coefParity_ = L.dd->parity_;
    }
  }

  void smooth(Level &L, int sweeps) {
    for (int k = 0; k < sweeps; ++k)
      for (int c = 0; c < colours_; ++c) {
        if (L.coefs.empty())
          L.dd->apply(L.gs, curr(L.u), L.u, curr(L.f), Colour{colours_, c}, only(L.u));
        else
          L.dd->relax(L.A, curr(L.u), L.u, curr(L.f), L.coefs, Colour{colours_, c}, 1.0, only(L.u));
      }
  }

  // top: the fine level of another pair (pair_level), or nullptr for the constructor's
  void vcycle(size_t l, Level *top = nullptr) {
    Level &L = l == 0 && top ? *top : levels_[l];
    if (l + 1 == levels_.size()) {
      smooth(L, coarse_sweeps_);
      return;
    }
    smooth(L, nu1_);
    Level &C = levels_[l + 1];
    L.dd->restrict_to(*C.dd, curr(C.f), L.res, L.u, curr(L.f), L.coefs, only(L.u));
    C.dd->clear_queued(C.u.id()); // coarse u <- +0
    vcycle(l + 1);
    L.dd->prolong_from(*C.dd, curr(L.u), curr(C.u), curr(L.u), only(C.u));
    smooth(L, nu2_);
  }
};

} // namespace stencil
