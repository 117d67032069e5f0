#pragma once
// The grid of subdomains as a graph: Topology::get_neighbor(index, dir) answers "which subdomain lies one step in
// direction dir (each component -1, 0 or +1) from subdomain `index`?".  The reference only has periodic grids
// (topology.hpp:12-15: `enum Boundary { NONE, PERIODIC }`, boundary.hpp is a stub); FIXED is this library's addition, per
// axis: the grid ends at its faces along that axis, a step across one has no neighbour (OptionalNeighbor::exists ==
// false) and no message is planned for it.  The ghost cells behind such a wall face keep what the application put into
// them, unless a boundary condition is set for them (DistributedDomain::set_boundary_condition).

#include <cassert>
#include <cstdio>
#include <cstdlib>

#include "stencil/dim3.hpp"

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

  OptionalNeighbor get_neighbor(const Dim3 &index, const Dim3 &dir) const noexcept {
    assert(index.all_ge(0) && "subdomain indices are non-negative");
    assert(dir.all_gt(-2) && dir.all_lt(2) && "a direction has components in {-1, 0, +1}");
    OptionalNeighbor answer;
    Dim3 to = index + dir;
    answer.exists = true;
    for (int a = 0; a < 3; ++a) {
      switch (kind_[a]) {
      case Boundary::PERIODIC: // a periodic axis wraps: stepping off one face re-enters through the opposite one
        to[a] = ((to[a] % grid_[a]) + grid_[a]) % grid_[a];
        break;
      case Boundary::FIXED: // the grid ends at its faces along this axis: a step that leaves it has no neighbour
        if (to[a] < 0 || to[a] >= grid_[a]) answer.exists = false;
        break;
      default:
        std::fprintf(stderr, "Topology::get_neighbor: the topology has no boundary kind (default-constructed?)\n");
        std::exit(1);
      }
    }
    answer.index = answer.exists ? to : index;
    return answer;
  }

  const Dim3 &extent() const noexcept { return grid_; }
  Boundary boundary(int axis) const noexcept { return kind_[axis]; }

private:
  Dim3 grid_;        // subdomains per axis
  Boundary kind_[3]; // how the grid closes at its faces, per axis
};
