#pragma once
// stencil::BC: the boundary condition of one quantity on one wall face of a non-periodic grid
// (DistributedDomain::set_boundary_condition).  Kinds and the per-cell rule are those of the C ABI
// (include/stencil_b200.h, sb_bc_regions):
//   BC::NONE()     the ghost cells are left alone (the default)
//   BC::VALUE(c)   ghost = c                              float / double quantities
//   BC::EVEN()     ghost = its mirror image about the face any quantity (a copy)
//   BC::ODD(c)     ghost = 2c - its mirror image          float / double; c is the value at the face
// Where walls meet, the faces apply in order x, y, z.

#include <type_traits>

namespace stencil {

struct BC {
  enum class Kind { NONE = 0, VALUE = 1, EVEN = 2, ODD = 3 }; // the values of sb_bc_kind
  Kind kind = Kind::NONE;
  double value = 0;

  static BC NONE() { return BC{}; }
  static BC VALUE(double c) { return BC{Kind::VALUE, c}; }
  static BC EVEN() { return BC{Kind::EVEN, 0}; }
  static BC ODD(double c = 0) { return BC{Kind::ODD, c}; }
};

// sb_dtype of an element type: float and double carry arithmetic, anything else is copied as raw bytes
template <typename T> constexpr int bc_dtype() {
  return std::is_same<T, float>::value ? 1 : std::is_same<T, double>::value ? 2 : 0;
}

} // namespace stencil
