// C++ API check of DistributedDomain::exchange(quantities) (DESIGN.md section 2.15), in one process or one rank per GPU
// under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs than ranks; every rank checks its own subdomains
// and the verdict is all-reduced).  Every allocation is poisoned (all bytes 0xff: NaN in float and double), the compute
// cells filled from the global coordinate; a full exchange gives the reference bytes.  Then, from the same poisoned
// state, an exchange of a subset must give each quantity of the subset the full exchange's bytes, ghost cells and wall
// BCs included, and leave every byte of the other quantities as it was: across ranks that runs the subset through the
// CUDA-IPC epoch handshake and the full layout's staging offsets on both ends.  Periodic and walled grids, radius 1, 2
// and face-edge-corner, several subsets, before and after swap().  (The C++ PCG and BiCGStab, which exchange subsets on
// their queued paths, are checked across ranks by test_krylov_multigpu and test_bicgstab_multigpu.)
// Build: make bin/test_exchange_subset_multigpu      Run: bin/sb_mpirun -n 4 bin/test_exchange_subset_multigpu
#include <cstdio>
#include <vector>

#include "stencil/stencil.hpp"

template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, int q, int seed) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x) acc[Dim3(x, y, z)] = T((x * 7 + y * 131 + z * 1009 + q * 3 + seed) % 101);
}

struct Handles {
  DataHandle<float> f0;
  DataHandle<char> c1;
  DataHandle<double> d2;
  DataHandle<float> f3;
};

static void load(DistributedDomain &dd, const Handles &h, int seed) {
  for (auto &d : dd.domains()) {
    d.set_device();
    for (size_t q = 0; q < 4; ++q) {
      const cudaPitchedPtr p = d.curr_data(q);
      CUDA_RUNTIME(cudaMemset(p.ptr, 0xff, p.pitch * p.ysize * size_t(d.raw_size().z)));
    }
    const Rect3 reg = d.get_compute_region();
    fill<float><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h.f0), reg, 0, seed);
    fill<char><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h.c1), reg, 1, seed);
    fill<double><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h.d2), reg, 2, seed);
    fill<float><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h.f3), reg, 3, seed);
    CUDA_RUNTIME(cudaDeviceSynchronize());
  }
}

// [local domain][quantity] -> the whole allocation's bytes
static std::vector<std::vector<std::vector<unsigned char>>> snapshot(DistributedDomain &dd) {
  std::vector<std::vector<std::vector<unsigned char>>> out;
  for (auto &d : dd.domains()) {
    out.emplace_back();
    for (size_t q = 0; q < 4; ++q) out.back().push_back(d.quantity_to_host(q));
  }
  return out;
}

static long check_subsets(DistributedDomain &dd, const Handles &h, int seed) {
  const std::vector<std::vector<size_t>> subsets = {{0}, {1}, {2}, {0, 2}, {3, 1}, {0, 1, 2, 3}};
  load(dd, h, seed);
  dd.exchange();
  const auto full = snapshot(dd);
  long bad = 0;
  for (const std::vector<size_t> &sub : subsets) {
    load(dd, h, seed);
    const auto before = snapshot(dd);
    dd.exchange(sub);
    const auto got = snapshot(dd);
    for (size_t di = 0; di < got.size(); ++di)
      for (size_t q = 0; q < 4; ++q) {
        bool in = false;
        for (size_t s : sub) in = in || s == q;
        if (got[di][q] != (in ? full[di][q] : before[di][q])) {
          if (bad < 5) std::fprintf(stderr, "MISMATCH subdomain %zu quantity %zu (%s the subset)\n", di, q, in ? "in" : "not in");
          ++bad;
        }
      }
  }
  return bad;
}

static long run_case(const Radius &radius, bool walls, const char *name) {
  DistributedDomain dd(24, 18, 20);
  dd.set_radius(radius);
  Handles h{dd.add_data<float>("f0"), dd.add_data<char>("c1"), dd.add_data<double>("d2"), dd.add_data<float>("f3")};
  if (walls) {
    dd.set_boundary(Topology::Boundary::FIXED, Topology::Boundary::PERIODIC, Topology::Boundary::FIXED);
    const Dim3 faces[4] = {Dim3(-1, 0, 0), Dim3(1, 0, 0), Dim3(0, 0, -1), Dim3(0, 0, 1)};
    for (int f = 0; f < 4; ++f) {
      dd.set_boundary_condition(h.f0, faces[f], f % 2 ? stencil::BC::ODD(0.25) : stencil::BC::EVEN());
      dd.set_boundary_condition(h.c1, faces[f], stencil::BC::EVEN());
      dd.set_boundary_condition(h.d2, faces[f], f % 2 ? stencil::BC::VALUE(-1.5) : stencil::BC::ODD(0.0));
      dd.set_boundary_condition(h.f3, faces[f], stencil::BC::VALUE(2.0));
    }
  }
  dd.realize();
  long bad = check_subsets(dd, h, 0);
  dd.swap(); // the other parity's plans
  bad += check_subsets(dd, h, 5);
  long long all = bad;
  MPI_Allreduce(MPI_IN_PLACE, &all, 1, MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
  if (0 == mpi::world_rank())
    std::printf("%-28s on %d rank(s) x %zu subdomain(s): %s (%lld mismatches)\n", name, mpi::world_size(), dd.domains().size(), all ? "FAIL" : "ok", all);
  return long(all);
}

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  long bad = 0;
  bad += run_case(Radius::constant(1), false, "periodic r=1");
  bad += run_case(Radius::constant(2), true, "walled r=2");
  bad += run_case(Radius::face_edge_corner(2, 1, 1), true, "walled faces 2 edges 1");
  if (0 == mpi::world_rank()) std::printf(bad ? "FAILED\n" : "ALL OK\n");
  MPI_Finalize();
  return bad ? 1 : 0;
}
