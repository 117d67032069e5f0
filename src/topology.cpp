#include "stencil/topology.hpp"

Topology::OptionalNeighbor Topology::get_neighbor(const Dim3 &index, const Dim3 &dir) const noexcept {
  assert(index.all_ge(0) && "subdomain indices are non-negative");
  assert(dir.all_gt(-2) && dir.all_lt(2) && "a direction has components in {-1, 0, +1}");
  OptionalNeighbor answer;
  Dim3 to = index + dir;
  answer.exists = true;
  for (int a = 0; a < 3; ++a) {
    int64_t &v = a == 0 ? to.x : a == 1 ? to.y : to.z;
    const int64_t n = a == 0 ? grid_.x : a == 1 ? grid_.y : grid_.z;
    switch (kind_[a]) {
    case Boundary::PERIODIC: // a periodic axis wraps: stepping off one face re-enters through the opposite one
      v = ((v % n) + n) % n;
      break;
    case Boundary::FIXED: // the grid ends at its faces along this axis: a step that leaves it has no neighbour
      if (v < 0 || v >= n) answer.exists = false;
      break;
    default:
      LOG_FATAL("Topology::get_neighbor: the topology has no boundary kind (default-constructed?)");
    }
  }
  answer.index = answer.exists ? to : index;
  return answer;
}
