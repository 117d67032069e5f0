#pragma once
// Constant-coefficient linear stencil operators on a DistributedDomain (DESIGN.md section 2.7; the rule, the reach check
// and the Laplacian table are the C ABI's sb_stencil_* of include/stencil_b200.h).
//
//     stencil::LinearStencil lap = stencil::LinearStencil::laplacian(4, hx, hy, hz);
//     stencil::LinearStencil heat = lap.scaled(dt).add(stencil::Source::src, 0, 0, 0, 1.0);   // u + dt lap(u)
//     dd.apply(heat, stencil::next(h), h);                                                        // overlapped with exchange()
//     dd.swap();
#include <cstdint>
#include <vector>

#include "stencil/local_domain.cuh"
#include "stencil/logging.hpp"
#include "stencil/reduce.hpp"
#include "stencil_b200.h"

namespace stencil {

enum class Source { src = 0, aux = 1 };

// An operator: terms (source, offset, weight) applied in list order.  Terms on aux have offset 0.
class LinearStencil {
  std::vector<sb_stencil_term> terms_;

public:
  LinearStencil() = default;
  explicit LinearStencil(std::vector<sb_stencil_term> terms) : terms_(std::move(terms)) {}

  LinearStencil &add(Source s, int dx, int dy, int dz, double w) {
    terms_.push_back(sb_stencil_term{int32_t(s), {dx, dy, dz}, w});
    return *this;
  }
  // every weight multiplied by f (in double)
  LinearStencil scaled(double f) const {
    LinearStencil out(*this);
    for (sb_stencil_term &t : out.terms_) t.weight *= f;
    return out;
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
  bool has_aux() const noexcept {
    for (const sb_stencil_term &t : terms_)
      if (t.source == 1) return true;
    return false;
  }
};

// A buffer of a quantity for DistributedDomain::apply: its curr or next allocation.
template <typename T> struct Buffer {
  DataHandle<T> h;
  Which which;
};
template <typename T> Buffer<T> curr(const DataHandle<T> &h) { return Buffer<T>{h, Which::curr}; }
template <typename T> Buffer<T> next(const DataHandle<T> &h) { return Buffer<T>{h, Which::next}; }

} // namespace stencil
