// C++ API check of linear stencil systems (DistributedDomain::apply with a stencil::LinearSystem) -- one process with N
// subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs
// than ranks).
//   bin/test_system_multigpu --single N OUT    one process, N subdomains: checks against the host, writes the result bits
//   bin/sb_mpirun -n N bin/test_system_multigpu --expect OUT
//                                             one subdomain per rank: checks against the host, and every rank's bits
//                                             must equal OUT's (the one-process run)
// Runs, in float and double, 6 leapfrog steps of Maxwell's equations on a periodic Yee grid: E = E + dt curl- H, then
// H = H - dt curl+ E, both in place in the curr buffers and overlapped with the exchange.  The host restatement applies
// the same rule on the global periodic grid with the same separately rounded operations.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "stencil/linear_stencil.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::LinearSystem;

template <typename T> __host__ __device__ T field(int q, int64_t x, int64_t y, int64_t z) {
  return T(double((x * 7 + y * 131 + z * 1009 + q * 37) % 8191) * 0.0009765625 - 4.0);
}

template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, int q) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x) acc[Dim3(x, y, z)] = field<T>(q, x, y, z);
}

template <typename T> std::vector<T> host_field(int q, int64_t X, int64_t Y, int64_t Z) {
  std::vector<T> v(size_t(X * Y * Z));
  for (int64_t z = 0; z < Z; ++z)
    for (int64_t y = 0; y < Y; ++y)
      for (int64_t x = 0; x < X; ++x) v[size_t((z * Y + y) * X + x)] = field<T>(q, x, y, z);
  return v;
}

// the rule on the global periodic grid, [z][y][x]: every output computed from the inputs before any is stored (outputs
// may be inputs read at offset 0); volatile keeps the host compiler from contracting multiply and add
template <typename T>
std::vector<std::vector<T>> host_apply(const LinearSystem &sys, const std::vector<const std::vector<T> *> &in, int64_t X, int64_t Y, int64_t Z) {
  std::vector<std::vector<T>> out(size_t(sys.nout()), std::vector<T>(size_t(X * Y * Z)));
  auto at = [&](int64_t x, int64_t y, int64_t z, const int32_t *o) {
    return size_t((((z + o[2] + Z) % Z) * Y + (y + o[1] + Y) % Y) * X + (x + o[0] + X) % X);
  };
  for (int64_t z = 0; z < Z; ++z)
    for (int64_t y = 0; y < Y; ++y)
      for (int64_t x = 0; x < X; ++x) {
        const size_t i = size_t((z * Y + y) * X + x);
        for (int j = 0; j < sys.nout(); ++j) {
          T acc = 0;
          bool first = true;
          for (const sb_stencil_sys_term &t : sys.terms()) {
            if (t.output != j) continue;
            volatile T w = T(t.weight);
            if (t.coef >= 0) w = T(w) * (*in[size_t(t.coef)])[at(x, y, z, t.coef_offset)];
            volatile T m = T(w) * (*in[size_t(t.input)])[at(x, y, z, t.offset)];
            acc = first ? T(m) : T(acc + T(m));
            first = false;
          }
          out[size_t(j)][i] = acc;
        }
      }
  return out;
}

template <typename T> std::vector<T> gather(DistributedDomain &dd, size_t q, int64_t X, int64_t Y, int64_t Z) {
  std::vector<T> out(size_t(X * Y * Z), T(0));
  for (LocalDomain &d : dd.domains()) {
    const Dim3 rs = d.raw_size(), sz = d.size(), o = d.origin(), rl(dd.radius().x(-1), dd.radius().y(-1), dd.radius().z(-1));
    std::vector<T> a(size_t(rs.x * rs.y * rs.z));
    d.set_device();
    CUDA_RUNTIME(cudaMemcpy(a.data(), d.curr_data(q).ptr, a.size() * sizeof(T), cudaMemcpyDeviceToHost));
    for (int64_t z = 0; z < sz.z; ++z)
      for (int64_t y = 0; y < sz.y; ++y)
        for (int64_t x = 0; x < sz.x; ++x)
          out[size_t(((o.z + z) * Y + o.y + y) * X + o.x + x)] = a[size_t(((z + rl.z) * rs.y + y + rl.y) * rs.x + x + rl.x)];
  }
  // every rank contributes its subdomains; the cells are disjoint, so a byte-wise sum of zero-initialised arrays merges them
  if (mpi::world_size() > 1) {
    std::vector<T> all(out.size());
    MPI_Allreduce(out.data(), all.data(), int(out.size() * sizeof(T) / 8), MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
    out.swap(all);
  }
  return out;
}

template <typename T> static std::string hexsum(const std::vector<T> &v) {
  // FNV-1a of the bits
  uint64_t h = 1469598103934665603ull;
  const unsigned char *b = reinterpret_cast<const unsigned char *>(v.data());
  for (size_t i = 0; i < v.size() * sizeof(T); ++i) h = (h ^ b[i]) * 1099511628211ull;
  char buf[32];
  std::snprintf(buf, sizeof(buf), "%016llx", (unsigned long long)h);
  return buf;
}

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits) {
  const int64_t X = 34, Y = 22, Z = 18;
  const double dt = 0.2, hx = 1.0, hy = 0.5, hz = 0.75;
  long bad = 0;
  DistributedDomain dd(X, Y, Z);
  dd.set_gpus(gpus);
  dd.set_radius(Radius::face_edge_corner(1, 0, 0));
  std::vector<DataHandle<T>> q; // Ex, Ey, Ez, Hx, Hy, Hz
  for (const char *name : {"ex", "ey", "ez", "hx", "hy", "hz"}) q.push_back(dd.add_data<T>(name));
  dd.realize();
  std::vector<std::vector<T>> f;
  for (int k = 0; k < 6; ++k) {
    for (auto &d : dd.domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(q[size_t(k)]), d.get_compute_region(), k);
    }
    f.push_back(host_field<T>(k, X, Y, Z));
  }
  LinearSystem ident;
  for (int j = 0; j < 3; ++j) ident.add(j, 3 + j, 0, 0, 0, 1.0);
  const LinearSystem e_sys = ident + LinearSystem::curl(-1, hx, hy, hz).scaled(dt); // inputs H, E -> E
  const LinearSystem h_sys = ident + LinearSystem::curl(1, hx, hy, hz).scaled(-dt); // inputs E, H -> H
  if (e_sys.nin() != 6 || e_sys.nout() != 3 || e_sys.terms().size() != 15 || LinearSystem::grad(1, 1, 1, 1).shifted(2, 1).nin() != 3) {
    std::fprintf(stderr, "LinearSystem: unexpected shape\n");
    ++bad;
  }
  using B = stencil::Buffer<T>;
  const std::vector<B> E = {stencil::curr(q[0]), stencil::curr(q[1]), stencil::curr(q[2])};
  const std::vector<B> H = {stencil::curr(q[3]), stencil::curr(q[4]), stencil::curr(q[5])};
  for (int it = 0; it < 6; ++it) {
    dd.apply(e_sys, E, std::vector<B>{H[0], H[1], H[2], E[0], E[1], E[2]});
    std::vector<std::vector<T>> ne = host_apply<T>(e_sys, {&f[3], &f[4], &f[5], &f[0], &f[1], &f[2]}, X, Y, Z);
    for (int j = 0; j < 3; ++j) f[size_t(j)].swap(ne[size_t(j)]);
    dd.apply(h_sys, H, std::vector<B>{E[0], E[1], E[2], H[0], H[1], H[2]});
    std::vector<std::vector<T>> nh = host_apply<T>(h_sys, {&f[0], &f[1], &f[2], &f[3], &f[4], &f[5]}, X, Y, Z);
    for (int j = 0; j < 3; ++j) f[size_t(3 + j)].swap(nh[size_t(j)]);
  }
  for (int k = 0; k < 6; ++k) {
    const std::vector<T> got = gather<T>(dd, q[size_t(k)].id(), X, Y, Z);
    if (std::memcmp(got.data(), f[size_t(k)].data(), got.size() * sizeof(T))) {
      if (0 == mpi::world_rank()) std::fprintf(stderr, "Yee (%zu-byte elements), field %d: device and host bits differ\n", sizeof(T), k);
      ++bad;
    }
    bits.push_back(hexsum(got));
  }
  return bad;
}

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  if (argc < 3) {
    std::fprintf(stderr, "usage: %s --single N OUT | --expect OUT\n", argv[0]);
    return 2;
  }
  const bool single = std::string(argv[1]) == "--single";
  int ndev = 0;
  CUDA_RUNTIME(cudaGetDeviceCount(&ndev));
  std::vector<int> gpus = single ? std::vector<int>(size_t(std::atoi(argv[2])), 0) : std::vector<int>{mpi::world_rank() % ndev};
  const size_t nsub = single ? gpus.size() : size_t(mpi::world_size());
  std::vector<std::string> bits;
  long bad = run<double>(gpus, bits) + run<float>(gpus, bits);
  if (single) {
    std::ofstream f(argv[3]);
    for (const std::string &b : bits) f << b << "\n";
  } else {
    std::ifstream f(argv[2]);
    std::vector<std::string> want;
    for (std::string line; std::getline(f, line);) want.push_back(line);
    if (want != bits) {
      std::fprintf(stderr, "rank %d: result bits differ from the one-process run of the same partition\n", mpi::world_rank());
      ++bad;
    }
  }
  long long all = bad;
  MPI_Allreduce(MPI_IN_PLACE, &all, 1, MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
  if (0 == mpi::world_rank()) {
    std::printf("DistributedDomain::apply with a LinearSystem (Yee), %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
