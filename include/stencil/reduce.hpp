#pragma once
// Deterministic reductions over a DistributedDomain (DESIGN.md section 2.6; the kernel and the merge rule are the C ABI's
// sb_reduce_* of include/stencil_b200.h).  Named Reduction, not Statistics: the reference's drivers define that name.
//
//     stencil::Reduction r = dd.reduce(h);                       // min, max, sum, sum of squares of curr
//     double res = dd.reduce_diff(h).l2();                       // ||curr - next||_2
//     double urms = dd.reduce_norm(hx, hy, hz).rms();            // sqrt(sum |u|^2 / N)
//     auto rs = dd.reduce_many({stencil::ReduceItem::scalar(h), stencil::ReduceItem::diff(h)});  // one launch per subdomain
//     double total = dd.reduce(h, stencil::Which::curr, stencil::Sum::exact).sum;  // correctly rounded, any partition
#include <cmath>
#include <cstddef>
#include <cstdint>

#include "stencil/local_domain.cuh"
#include "stencil_b200.h"

namespace stencil {

struct Reduction {
  double min, max; // of the per-cell value v (NaN if any v is NaN; +inf / -inf for an empty region)
  double sum;      // of v
  double sumsq;    // of the squared term q (v * v; for a norm the sum of the squared components)
  int64_t count;   // cells

  double mean() const { return count ? sum / double(count) : NAN; }
  double rms() const { return count ? std::sqrt(sumsq / double(count)) : NAN; }
  double l2() const { return std::sqrt(sumsq); }
};

enum class Which { curr, next };

// How sum and sumsq are formed.  ordered: the fixed trees of sb_reduce_plan_* (the faster path; the bits depend on the
// partition).  exact: sb_reduce_exact_plan_* -- the exact sums rounded once, the same bits for every partition and rank
// count (DESIGN.md section 2.6.1).  min, max and count are the same either way on one subdomain.
enum class Sum { ordered, exact };

// One item of DistributedDomain::reduce_many: a SCALAR (curr or next buffer), a DIFF (curr - next) or a NORM3
// (|(x, y, z)| of three quantities' curr buffers) over the whole compute region.
struct ReduceItem {
  sb_reduce_kind kind;
  size_t q[3];
  Which which;

  template <typename T> static ReduceItem scalar(const DataHandle<T> &h, Which w = Which::curr) {
    return ReduceItem{SB_REDUCE_SCALAR, {h.id(), h.id(), h.id()}, w};
  }
  template <typename T> static ReduceItem diff(const DataHandle<T> &h) { return ReduceItem{SB_REDUCE_DIFF, {h.id(), h.id(), h.id()}, Which::curr}; }
  template <typename T> static ReduceItem norm(const DataHandle<T> &x, const DataHandle<T> &y, const DataHandle<T> &z) {
    return ReduceItem{SB_REDUCE_NORM3, {x.id(), y.id(), z.id()}, Which::curr};
  }
};

} // namespace stencil
