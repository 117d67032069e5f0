// jacobi3d_b200: the reference's jacobi3d driver (bin/jacobi3d.cu) with its loop body replaced by
// stencil::FusedJacobi3d::step() -- the hand-written sm_90a kernel with the halo push fused in -- so that C++ users
// of the DistributedDomain API reach the roofline kernel.  Same weak-scaling size rule, same CSV line.
//
//   jacobi3d_b200 <x> <y> <z> [-n iters] [--f64] [--trivial] [--reference-schedule] [--dump file]
//
// --reference-schedule: interior || exchange -> exterior with this library's kernels instead of the fused kernel.
// x y z: per-subdomain size, scaled by the prime factors of the subdomain count like bin/jacobi3d.cu:189-199.
// --f64: double instead of the reference's float.  --dump: the global compute region (x fastest) after the last
// iteration, raw bytes -- tests compare it with the reference's own kernel (oracle/_ref/ref_jacobi_golden_ieee).
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "stencil/jacobi3d.hpp"
#include "stencil/numeric.hpp"
#include "stencil/stencil.hpp"

namespace {

double trimean(std::vector<double> v) { // (Q1 + 2 Q2 + Q3) / 4 with linear interpolation, like bin/statistics.cpp
  std::sort(v.begin(), v.end());
  auto q = [&](double f) {
    const double pos = f * double(v.size() - 1);
    const size_t i = size_t(pos);
    const double frac = pos - double(i);
    return (i + 1 < v.size()) ? v[i] * (1 - frac) + v[i + 1] * frac : v[i];
  };
  return (q(0.25) + 2 * q(0.5) + q(0.75)) / 4;
}

template <typename T> int run(size_t x, size_t y, size_t z, int iters, bool trivial, bool refSchedule, const std::string &dump) {
  int devCount = 0;
  CUDA_RUNTIME(cudaGetDeviceCount(&devCount));
  const int size = mpi::world_size(), rank = mpi::world_rank();
  int numSubdoms;
  {
    MpiTopology topo(MPI_COMM_WORLD);
    const int perRank = topo.colocated_size() > devCount ? 1 : devCount / topo.colocated_size();
    numSubdoms = size * perRank;
  }
  for (int pf : prime_factors(numSubdoms)) {
    if (x <= y && x <= z) x *= size_t(pf);
    else if (y <= z) y *= size_t(pf);
    else z *= size_t(pf);
  }
  Radius radius = Radius::constant(0);
  radius.set_face(1);
  std::vector<double> times;
  {
    DistributedDomain dd(x, y, z);
    dd.set_radius(radius);
    dd.set_placement(trivial ? PlacementStrategy::Trivial : PlacementStrategy::NodeAware);
    auto dh = dd.add_data<T>("d");
    dd.realize();
    stencil::FusedJacobi3d jac(dd, dh, !refSchedule);
    jac.init(0.5);
    MPI_Barrier(MPI_COMM_WORLD);
    for (int it = 0; it < iters; ++it) {
      double t0 = MPI_Wtime();
      jac.step();
      jac.synchronize(); // per-iteration wall time like the reference prints; step() itself never blocks
      double el = MPI_Wtime() - t0;
      MPI_Allreduce(MPI_IN_PLACE, &el, 1, MPI_DOUBLE, MPI_MAX, MPI_COMM_WORLD);
      times.push_back(el);
    }
    // the same iterations queued back to back (what a production loop does): one sync at the end
    double queued = 0;
    if (iters > 0) {
      MPI_Barrier(MPI_COMM_WORLD);
      const double t0 = MPI_Wtime();
      for (int it = 0; it < iters; ++it) jac.step();
      jac.synchronize();
      queued = (MPI_Wtime() - t0) / iters;
      MPI_Allreduce(MPI_IN_PLACE, &queued, 1, MPI_DOUBLE, MPI_MAX, MPI_COMM_WORLD);
    }
    if (!dump.empty()) {
      if (size != 1) LOG_FATAL("--dump gathers the local subdomains of one rank only");
      std::vector<T> global(x * y * z);
      for (const LocalDomain &d : dd.domains()) {
        const std::vector<unsigned char> bytes = d.interior_to_host(dh.id());
        const T *v = reinterpret_cast<const T *>(bytes.data());
        const Dim3 o = d.origin(), s = d.size();
        for (int64_t k = 0; k < s.z; ++k)
          for (int64_t j = 0; j < s.y; ++j)
            std::memcpy(&global[size_t(((o.z + k) * int64_t(y) + (o.y + j)) * int64_t(x) + o.x)], v + (k * s.y + j) * s.x, size_t(s.x) * sizeof(T));
      }
      FILE *f = std::fopen(dump.c_str(), "wb");
      if (!f || std::fwrite(global.data(), sizeof(T), global.size(), f) != global.size()) LOG_FATAL("cannot write " << dump);
      std::fclose(f);
    }
    if (0 == rank) {
      const double mn = times.empty() ? 0 : *std::min_element(times.begin(), times.end());
      std::printf("jacobi3d_b200,%s,%d,%d,%zu,%zu,%zu,%llu,%llu,%llu,%llu,%g,%g\n", jac.fused() ? "fused" : "interior|exchange|exterior", size,
                  devCount, x, y, z, (unsigned long long)dd.exchange_bytes_for_method(Method::CudaMpi),
                  (unsigned long long)dd.exchange_bytes_for_method(Method::ColoPackMemcpyUnpack),
                  (unsigned long long)dd.exchange_bytes_for_method(Method::CudaMemcpyPeer),
                  (unsigned long long)dd.exchange_bytes_for_method(Method::CudaKernel), mn, times.empty() ? 0 : trimean(times));
      const double cells = double(x) * double(y) * double(z);
      std::printf("jacobi3d_b200_queued,%s,%zu,%zu,%zu,iters=%d,s_per_iter=%g,cells_per_s=%g,cells_per_s_per_gpu=%g\n", sizeof(T) == 8 ? "f64" : "f32", x, y,
                  z, iters, queued, queued > 0 ? cells / queued : 0, queued > 0 ? cells / queued / double(dd.domains().size() * size_t(size)) : 0);
    }
  }
  return 0;
}

} // namespace

int main(int argc, char **argv) {
  size_t dims[3] = {512, 512, 512};
  int npos = 0, iters = 5;
  bool f64 = false, trivial = false, refSchedule = false;
  std::string dump;
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if ((a == "-n" || a == "--iters") && i + 1 < argc) iters = std::atoi(argv[++i]);
    else if (a == "--f64") f64 = true;
    else if (a == "--trivial") trivial = true;
    else if (a == "--reference-schedule") refSchedule = true;
    else if (a == "--dump" && i + 1 < argc) dump = argv[++i];
    else if (a == "-h" || a == "--help") {
      std::fprintf(stderr, "usage: %s x y z [-n iters] [--f64] [--trivial] [--dump file]\n", argv[0]);
      return 0;
    } else if (npos < 3 && !a.empty() && a[0] != '-') dims[npos++] = size_t(std::atoll(a.c_str()));
    else {
      std::fprintf(stderr, "unknown argument %s\n", a.c_str());
      return EXIT_FAILURE;
    }
  }
  if (npos != 3) {
    std::fprintf(stderr, "usage: %s x y z [-n iters] [--f64] [--trivial] [--dump file]\n", argv[0]);
    return EXIT_FAILURE;
  }
  MPI_Init(&argc, &argv);
  const int rc = f64 ? run<double>(dims[0], dims[1], dims[2], iters, trivial, refSchedule, dump)
                     : run<float>(dims[0], dims[1], dims[2], iters, trivial, refSchedule, dump);
  MPI_Finalize();
  return rc;
}
