#pragma once
// Linear stencil operators on a DistributedDomain, constant and variable coefficients (DESIGN.md section 2.7; the rule,
// the reach check and the Laplacian and div-grad tables are the C ABI's sb_stencil_* of include/stencil_b200.h).
//
//     stencil::LinearStencil lap = stencil::LinearStencil::laplacian(4, hx, hy, hz);
//     stencil::LinearStencil heat = lap.scaled(dt).add(stencil::Source::src, 0, 0, 0, 1.0);   // u + dt lap(u)
//     dd.apply(heat, stencil::next(h), h);                                                        // overlapped with exchange()
//     dd.swap();
//
//     // u + dt div(kappa grad u), kappa on the x / y / z faces in three quantities (their curr buffers)
//     stencil::LinearStencil kheat = stencil::LinearStencil::div_grad(hx, hy, hz).scaled(dt).add(stencil::Source::src, 0, 0, 0, 1.0);
//     dd.apply(kheat, stencil::next(h), h, {kx, ky, kz});
//
//     // Gauss-Seidel / SOR for A u = f (DESIGN.md section 2.9): one coloured apply per colour, in place, f on aux
//     stencil::LinearStencil sor = stencil::LinearStencil::laplacian(2, h, h, h).scaled(-1.0).relax(omega);
//     for (int c = 0; c < 2; ++c) dd.apply(sor, stencil::curr(u), u, stencil::curr(f), stencil::Colour{2, c});
#include <cstdint>
#include <vector>

#include "stencil/local_domain.cuh"
#include "stencil/logging.hpp"
#include "stencil/reduce.hpp"
#include "stencil_b200.h"

namespace stencil {

enum class Source { src = 0, aux = 1 };

// A colouring m (1, 2 or 8) and one of its colours c (0 .. m-1), from global coordinates: m = 2 is red-black,
// (x + y + z) mod 2; m = 8 is (x mod 2) + 2 (y mod 2) + 4 (z mod 2).  A coloured apply writes the cells of colour c only.
struct Colour {
  int m = 1, c = 0;
};

// What an operator call (apply, relax, restrict_to with an op, prolong_from) exchanges before it reads ghost cells
// (DESIGN.md section 2.15): true (the default) every quantity, false nothing (the caller guarantees the ghost cells),
// Exchange::reads() only the quantities the call reads at a non-zero offset (src, the coefficient fields a term reads
// at a non-zero coefficient offset, a system's inputs read at an offset; prolong_from: the coarse src), and
// Exchange::only(set) the quantities of a bit set (bit q: quantity q), as the solvers use it.
struct Exchange {
  enum Mode { kNone, kAll, kReads, kOnly };
  Mode mode;
  uint64_t quantities = 0;
  Exchange(bool all) : mode(all ? kAll : kNone) {} // NOLINT: a bool converts, as the parameter was a bool
  static Exchange reads() {
    Exchange e(true);
    e.mode = kReads;
    return e;
  }
  static Exchange only(uint64_t set) {
    Exchange e(true);
    e.mode = kOnly;
    e.quantities = set;
    return e;
  }
};

// An operator: terms (source, offset, weight) applied in list order, each of which may also read a coefficient field k at
// an offset of reach 1 (then it contributes (T(w) * C_k) * S).  Terms on aux have offset 0.
class LinearStencil {
  std::vector<sb_stencil_term> terms_;   // every term without its coefficient
  std::vector<sb_stencil_vterm> vterms_; // every term with its coefficient (coef = -1: none)

public:
  LinearStencil() = default;
  explicit LinearStencil(std::vector<sb_stencil_term> terms) : terms_(std::move(terms)) {
    for (const sb_stencil_term &t : terms_)
      vterms_.push_back(sb_stencil_vterm{t.source, {t.offset[0], t.offset[1], t.offset[2]}, -1, {0, 0, 0}, t.weight});
  }
  explicit LinearStencil(const std::vector<sb_stencil_vterm> &vterms) {
    for (const sb_stencil_vterm &t : vterms) add(Source(t.source), t.offset[0], t.offset[1], t.offset[2], t.weight, t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2]);
  }

  LinearStencil &add(Source s, int dx, int dy, int dz, double w) {
    terms_.push_back(sb_stencil_term{int32_t(s), {dx, dy, dz}, w});
    vterms_.push_back(sb_stencil_vterm{int32_t(s), {dx, dy, dz}, -1, {0, 0, 0}, w});
    return *this;
  }
  // a coefficient term: also reads coefficient field coef (-1: none) at (cx, cy, cz)
  LinearStencil &add(Source s, int dx, int dy, int dz, double w, int coef, int cx, int cy, int cz) {
    terms_.push_back(sb_stencil_term{int32_t(s), {dx, dy, dz}, w});
    vterms_.push_back(sb_stencil_vterm{int32_t(s), {dx, dy, dz}, coef, {cx, cy, cz}, w});
    return *this;
  }
  // every weight multiplied by f (in double)
  LinearStencil scaled(double f) const {
    LinearStencil out(*this);
    for (sb_stencil_term &t : out.terms_) t.weight *= f;
    for (sb_stencil_vterm &t : out.vterms_) t.weight *= f;
    return out;
  }
  // the conservative second-order div(kappa grad u) on a grid of spacing (hx, hy, hz): sb_stencil_div_grad.  Coefficient
  // field a holds kappa on the faces normal to axis a (C_a(p) on the face between p - e_a and p).
  static LinearStencil div_grad(double hx, double hy, double hz) {
    const double h[3] = {hx, hy, hz};
    const int n = sb_stencil_div_grad(h, nullptr, 0);
    if (n < 0) LOG_FATAL("LinearStencil::div_grad: " << sb_last_error());
    std::vector<sb_stencil_vterm> terms(static_cast<size_t>(n));
    sb_stencil_div_grad(h, terms.data(), n);
    return LinearStencil(terms);
  }
  // the SOR update of A u = f for this op A (constant coefficients, one centre term, no aux term), f on aux:
  // u + omega (f - A u) / a_c (sb_stencil_relax).  omega = 1 in a coloured sweep is Gauss-Seidel; omega outside (0, 2)
  // diverges for a symmetric positive definite A.
  LinearStencil relax(double omega) const {
    for (const sb_stencil_vterm &t : vterms_)
      if (t.coef >= 0) LOG_FATAL("LinearStencil::relax: the op has coefficient terms; the relaxation table takes constant coefficients");
    const int n = int(terms_.size());
    std::vector<sb_stencil_term> out(static_cast<size_t>(n + 1));
    const int m = sb_stencil_relax(terms_.data(), n, omega, out.data(), n + 1);
    if (m < 0) LOG_FATAL("LinearStencil::relax: " << sb_last_error());
    out.resize(static_cast<size_t>(m));
    return LinearStencil(std::move(out));
  }
  // the central-difference Laplacian of order 2, 4, 6 or 8 on a grid of spacing (hx, hy, hz): sb_stencil_laplacian
  static LinearStencil laplacian(int order, double hx, double hy, double hz) {
    const double h[3] = {hx, hy, hz};
    const int n = sb_stencil_laplacian(order, h, nullptr, 0);
    if (n < 0) LOG_FATAL("LinearStencil::laplacian: " << sb_last_error());
    std::vector<sb_stencil_term> terms(static_cast<size_t>(n));
    sb_stencil_laplacian(order, h, terms.data(), n);
    return LinearStencil(std::move(terms));
  }

  const std::vector<sb_stencil_term> &terms() const noexcept { return terms_; }
  const std::vector<sb_stencil_vterm> &vterms() const noexcept { return vterms_; }
  bool has_aux() const noexcept {
    for (const sb_stencil_term &t : terms_)
      if (t.source == 1) return true;
    return false;
  }
  // the number of coefficient fields DistributedDomain::apply takes: the highest field a term names, plus one
  int ncoef() const noexcept {
    int n = 0;
    for (const sb_stencil_vterm &t : vterms_) n = t.coef + 1 > n ? t.coef + 1 : n;
    return n;
  }
};

// A system (DESIGN.md section 2.8): terms (output, input, offset, weight), each of which may also read an input as its
// coefficient at an offset of reach 1, over nin() inputs and nout() outputs; each output sums its own terms in list order
// by the operator rule.  One launch per box computes every output.
//
//     // E = E + (dt / eps) curl- H in place: inputs Hx, Hy, Hz, Ex, Ey, Ez; outputs Ex, Ey, Ez
//     stencil::LinearSystem e = stencil::LinearSystem().add(0, 3, 0, 0, 0, 1.0).add(1, 4, 0, 0, 0, 1.0).add(2, 5, 0, 0, 0, 1.0) +
//                               stencil::LinearSystem::curl(-1, h, h, h).scaled(dt / eps);
//     dd.apply(e, {curr(ex), curr(ey), curr(ez)}, {curr(hx), curr(hy), curr(hz), curr(ex), curr(ey), curr(ez)});
class LinearSystem {
  std::vector<sb_stencil_sys_term> terms_;
  int nin_ = 0, nout_ = 0;

  template <typename Fn> static LinearSystem table(Fn fn, const char *name, int stagger, double hx, double hy, double hz) {
    const double h[3] = {hx, hy, hz};
    const int n = fn(stagger, h, nullptr, 0);
    if (n < 0) LOG_FATAL("LinearSystem::" << name << ": " << sb_last_error());
    std::vector<sb_stencil_sys_term> terms(static_cast<size_t>(n));
    fn(stagger, h, terms.data(), n);
    LinearSystem s;
    for (const sb_stencil_sys_term &t : terms) s.push(t);
    return s;
  }
  void push(const sb_stencil_sys_term &t) {
    terms_.push_back(t);
    nout_ = t.output + 1 > nout_ ? t.output + 1 : nout_;
    nin_ = t.input + 1 > nin_ ? t.input + 1 : nin_;
    nin_ = t.coef + 1 > nin_ ? t.coef + 1 : nin_;
  }

public:
  LinearSystem &add(int out, int in, int dx, int dy, int dz, double w) {
    push(sb_stencil_sys_term{out, in, {dx, dy, dz}, -1, {0, 0, 0}, w});
    return *this;
  }
  // a coefficient term: also reads input coef (-1: none) at (cx, cy, cz)
  LinearSystem &add(int out, int in, int dx, int dy, int dz, double w, int coef, int cx, int cy, int cz) {
    push(sb_stencil_sys_term{out, in, {dx, dy, dz}, coef, {cx, cy, cz}, w});
    return *this;
  }
  // every weight multiplied by f (in double)
  LinearSystem scaled(double f) const {
    LinearSystem out(*this);
    for (sb_stencil_sys_term &t : out.terms_) t.weight *= f;
    return out;
  }
  // the same system reading inputs input_base + i (coefficients included) and writing outputs output_base + j
  LinearSystem shifted(int input_base, int output_base) const {
    LinearSystem out;
    for (sb_stencil_sys_term t : terms_) {
      t.output += output_base;
      t.input += input_base;
      if (t.coef >= 0) t.coef += input_base;
      out.push(t);
    }
    out.nin_ = nin_ + input_base > out.nin_ ? nin_ + input_base : out.nin_;
    out.nout_ = nout_ + output_base > out.nout_ ? nout_ + output_base : out.nout_;
    return out;
  }
  // concatenation: this system's terms, then o's
  LinearSystem operator+(const LinearSystem &o) const {
    LinearSystem out(*this);
    for (const sb_stencil_sys_term &t : o.terms_) out.push(t);
    out.nin_ = o.nin_ > out.nin_ ? o.nin_ : out.nin_;
    out.nout_ = o.nout_ > out.nout_ ? o.nout_ : out.nout_;
    return out;
  }
  // difference tables (sb_stencil_grad / div / curl): stagger +1 forward, -1 backward, 0 central
  static LinearSystem grad(int stagger, double hx, double hy, double hz) { return table(sb_stencil_grad, "grad", stagger, hx, hy, hz); }
  static LinearSystem div(int stagger, double hx, double hy, double hz) { return table(sb_stencil_div, "div", stagger, hx, hy, hz); }
  static LinearSystem curl(int stagger, double hx, double hy, double hz) { return table(sb_stencil_curl, "curl", stagger, hx, hy, hz); }

  const std::vector<sb_stencil_sys_term> &terms() const noexcept { return terms_; }
  int nin() const noexcept { return nin_; }
  int nout() const noexcept { return nout_; }
};

// A buffer of a quantity for DistributedDomain::apply: its curr or next allocation.
template <typename T> struct Buffer {
  DataHandle<T> h;
  Which which;
};
template <typename T> Buffer<T> curr(const DataHandle<T> &h) { return Buffer<T>{h, Which::curr}; }
template <typename T> Buffer<T> next(const DataHandle<T> &h) { return Buffer<T>{h, Which::next}; }

} // namespace stencil
