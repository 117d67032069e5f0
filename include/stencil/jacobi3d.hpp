#pragma once
// stencil::FusedJacobi3d -- the H100 fast path for the loop of the reference's jacobi3d driver
// (bin/jacobi3d.cu:296-368), for C++ users of the DistributedDomain API.  NOT part of the reference's API: an
// unchanged bin/jacobi3d.cu keeps launching its own stencil_kernel (7 global loads per cell); a driver that wants
// the roofline kernel replaces its loop body by step():
//
//     DistributedDomain dd(x, y, z);  dd.set_radius(faces1);  auto h = dd.add_data<double>("d");  dd.realize();
//     stencil::FusedJacobi3d jac(dd, h);
//     jac.init(0.5);                        // init_kernel, bin/jacobi3d.cu:18-29
//     for (...) jac.step();                 // interior + exchange + exterior + swap of one iteration
//     jac.synchronize();
//
// step() launches ONE kernel per local subdomain (sb_jacobi3d_fused: the update of the whole compute region, with
// every face cell also stored into the ghost cell of the neighbour that reads it next iteration) and orders
// subdomains with CUDA events; it does not block the host.  Where the fused kernel does not apply (face radius
// other than 1, fewer than 16 cells along x) it runs the reference's schedule with this library's kernels:
// interior (sb_jacobi3d) || dd.exchange() -> exterior slabs in one launch (sb_jacobi3d_regions) -> sync -> swap.
// Results are bit-identical either way (IEEE division, the reference's summation order).
#include <vector>

#include "stencil/stencil.hpp"

namespace stencil {

class FusedJacobi3d {
public:
  // allowFused = false forces the reference's schedule (interior || exchange -> exterior) over this library's kernels
  template <typename T> FusedJacobi3d(DistributedDomain &dd, const DataHandle<T> &h, bool allowFused = true) : FusedJacobi3d(dd, h.id(), sizeof(T), allowFused) {}
  FusedJacobi3d(DistributedDomain &dd, size_t quantity, size_t elemSize, bool allowFused = true);
  ~FusedJacobi3d();
  FusedJacobi3d(const FusedJacobi3d &) = delete;
  FusedJacobi3d &operator=(const FusedJacobi3d &) = delete;

  void init(double value = 0.5); // compute region of curr := value
  void step();                   // one iteration, swap included
  void synchronize();            // wait for everything step() queued
  bool fused() const noexcept { return fused_; }

private:
  struct Call; // argument pack of one subdomain and swap parity
  DistributedDomain &dd_;
  size_t q_, es_;
  bool fused_, ghostsCurrent_;
  int parity_; // number of step() calls mod 2 relative to construction
  std::vector<RcStream> streams_;
  std::vector<cudaEvent_t> done_;            // one per local subdomain: its last kernel
  std::vector<std::vector<size_t>> nbrs_;    // local subdomains whose kernels a subdomain must wait for
  std::vector<Call> *calls_;                 // [parity * ndomains + domain]
  void step_reference_schedule();
};

} // namespace stencil
