#pragma once
// The grid of subdomains as a graph: Topology::get_neighbor(index, dir) answers "which subdomain lies one step in
// direction dir (each component -1, 0 or +1) from subdomain `index`?".  The reference only has periodic grids
// (topology.hpp:12-15: `enum Boundary { NONE, PERIODIC }`, boundary.hpp is a stub); FIXED is this library's addition, per
// axis: the grid ends at its faces along that axis, a step across one has no neighbour (OptionalNeighbor::exists ==
// false) and no message is planned for it.  The ghost cells behind such a wall face keep what the application put into
// them, unless a boundary condition is set for them (DistributedDomain::set_boundary_condition).

#include <cassert>

#include "stencil/dim3.hpp"
#include "stencil/logging.hpp"

class Topology {
public:
  enum class Boundary { NONE, PERIODIC, FIXED };

  struct OptionalNeighbor {
    Dim3 index;
    bool exists = false;
    explicit operator bool() const noexcept { return exists; }
  };

  Topology() : grid_(0, 0, 0), kind_{Boundary::NONE, Boundary::NONE, Boundary::NONE} {}
  Topology(const Dim3 &extent, const Boundary &boundary) : grid_(extent), kind_{boundary, boundary, boundary} {}
  Topology(const Dim3 &extent, Boundary x, Boundary y, Boundary z) : grid_(extent), kind_{x, y, z} {}

  OptionalNeighbor get_neighbor(const Dim3 &index, const Dim3 &dir) const noexcept;

  const Dim3 &extent() const noexcept { return grid_; }
  Boundary boundary(int axis) const noexcept { return kind_[axis]; }

private:
  Dim3 grid_;        // subdomains per axis
  Boundary kind_[3]; // how the grid closes at its faces, per axis
};
