// C++ API check of the variable-coefficient linear stencil operators (DistributedDomain::apply with coefficient fields,
// stencil::LinearStencil::div_grad) -- one process with N subdomains on GPU 0, or one subdomain per rank under
// bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs than ranks).
//   bin/test_vstencil_multigpu --single N OUT    one process, N subdomains: checks against the host, writes the result bits
//   bin/sb_mpirun -n N bin/test_vstencil_multigpu --expect OUT
//                                               one subdomain per rank: checks against the host, and every rank's bits
//                                               must equal OUT's (the one-process run)
// Runs, in float and double: a periodic heterogeneous heat equation u + dt div(kappa grad u) with kappa on the faces in
// three quantities (6 steps with swap, overlapped with the exchange), and a variable-speed wave equation
// 2u - u_prev + c^2 lap(u) written over u_prev (dst == aux == next, 6 steps, exchange = false after a manual exchange()).
// The coefficient quantities hold the same cells in curr and next, so they survive every swap.  The host restatement
// applies the same rule on the global periodic grid with the same separately rounded operations.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "stencil/linear_stencil.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::LinearStencil;
using stencil::Source;

// q < 10: a solution field in [-4, 4); q >= 10: a coefficient in [0.25, 2.15)
template <typename T> __host__ __device__ T field(int q, int64_t x, int64_t y, int64_t z) {
  if (q >= 10) return T(double((x * 5 + y * 17 + z * 29 + q * 11) % 61) * 0.03125 + 0.25);
  return T(double((x * 7 + y * 131 + z * 1009 + q * 3) % 8191) * 0.0009765625 - 4.0);
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

// the rule on the global periodic grid, [z][y][x]; volatile keeps the host compiler from contracting multiply and add
template <typename T>
std::vector<T> host_apply(const LinearStencil &op, const std::vector<T> &u, const std::vector<T> &aux, const std::vector<std::vector<T>> &coefs,
                          int64_t X, int64_t Y, int64_t Z) {
  std::vector<T> out(u.size());
  auto at = [&](int64_t x, int64_t y, int64_t z, const int32_t *o) {
    return size_t((((z + o[2] + Z) % Z) * Y + (y + o[1] + Y) % Y) * X + (x + o[0] + X) % X);
  };
  for (int64_t z = 0; z < Z; ++z)
    for (int64_t y = 0; y < Y; ++y)
      for (int64_t x = 0; x < X; ++x) {
        const size_t i = size_t((z * Y + y) * X + x);
        T acc = 0;
        for (size_t k = 0; k < op.vterms().size(); ++k) {
          const sb_stencil_vterm &t = op.vterms()[k];
          const T v = t.source == 0 ? u[at(x, y, z, t.offset)] : aux[i];
          volatile T w = T(t.weight);
          if (t.coef >= 0) w = T(w) * coefs[size_t(t.coef)][at(x, y, z, t.coef_offset)];
          volatile T m = T(w) * v;
          acc = k == 0 ? T(m) : T(acc + T(m));
        }
        out[i] = acc;
      }
  return out;
}

template <typename T> std::vector<T> gather(DistributedDomain &dd, size_t q, stencil::Which w, int64_t X, int64_t Y, int64_t Z) {
  std::vector<T> out(size_t(X * Y * Z), T(0));
  for (LocalDomain &d : dd.domains()) {
    const Dim3 rs = d.raw_size(), sz = d.size(), o = d.origin(), rl(dd.radius().x(-1), dd.radius().y(-1), dd.radius().z(-1));
    std::vector<T> a(size_t(rs.x * rs.y * rs.z));
    d.set_device();
    CUDA_RUNTIME(cudaMemcpy(a.data(), (w == stencil::Which::curr ? d.curr_data(q) : d.next_data(q)).ptr, a.size() * sizeof(T), cudaMemcpyDeviceToHost));
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

template <typename T> static void fill_both(DistributedDomain &dd, const DataHandle<T> &h, int q) {
  for (auto &d : dd.domains()) {
    d.set_device();
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h), d.get_compute_region(), q);
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_next_accessor(h), d.get_compute_region(), q);
  }
}

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits) {
  const int64_t X = 34, Y = 22, Z = 18;
  long bad = 0;
  {
    DistributedDomain dd(X, Y, Z);
    dd.set_gpus(gpus);
    dd.set_radius(Radius::face_edge_corner(1, 0, 0));
    auto h = dd.add_data<T>("u");
    std::vector<DataHandle<T>> ks = {dd.add_data<T>("kx"), dd.add_data<T>("ky"), dd.add_data<T>("kz")};
    dd.realize();
    for (auto &d : dd.domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h), d.get_compute_region(), 0);
    }
    std::vector<std::vector<T>> kh;
    for (int k = 0; k < 3; ++k) {
      fill_both(dd, ks[size_t(k)], 10 + k);
      kh.push_back(host_field<T>(10 + k, X, Y, Z));
    }
    const LinearStencil heat = LinearStencil::div_grad(0.9, 1.0, 1.1).scaled(0.05).add(Source::src, 0, 0, 0, 1.0);
    if (heat.ncoef() != 3 || heat.vterms().size() != 13 || heat.terms().size() != 13) {
      std::fprintf(stderr, "div_grad: %d fields, %zu terms\n", heat.ncoef(), heat.vterms().size());
      ++bad;
    }
    std::vector<T> u = host_field<T>(0, X, Y, Z);
    for (int it = 0; it < 6; ++it) {
      dd.apply(heat, stencil::next(h), h, ks);
      dd.swap();
      u = host_apply(heat, u, u, kh, X, Y, Z);
    }
    const std::vector<T> got = gather<T>(dd, h.id(), stencil::Which::curr, X, Y, Z);
    if (std::memcmp(got.data(), u.data(), u.size() * sizeof(T))) {
      if (0 == mpi::world_rank()) std::fprintf(stderr, "heterogeneous heat (%zu-byte elements): device and host bits differ\n", sizeof(T));
      ++bad;
    }
    bits.push_back(hexsum(got));
  }
  {
    DistributedDomain dd(X, Y, Z);
    dd.set_gpus(gpus);
    dd.set_radius(1);
    auto h = dd.add_data<T>("u");
    auto c = dd.add_data<T>("c2");
    dd.realize();
    for (auto &d : dd.domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h), d.get_compute_region(), 1);
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_next_accessor(h), d.get_compute_region(), 2);
    }
    fill_both(dd, c, 13);
    const std::vector<std::vector<T>> ch = {host_field<T>(13, X, Y, Z)};
    LinearStencil wave;
    wave.add(Source::src, 0, 0, 0, 2.0).add(Source::aux, 0, 0, 0, -1.0);
    const LinearStencil lap = LinearStencil::laplacian(2, 1.0, 1.0, 1.0).scaled(0.1);
    for (const sb_stencil_term &t : lap.terms())
      wave.add(Source(t.source), t.offset[0], t.offset[1], t.offset[2], t.weight, 0, 0, 0, 0);
    std::vector<T> u = host_field<T>(1, X, Y, Z), prev = host_field<T>(2, X, Y, Z);
    for (int it = 0; it < 6; ++it) {
      for (auto &d : dd.domains()) {
        d.set_device();
        CUDA_RUNTIME(cudaDeviceSynchronize());
      }
      dd.exchange();
      dd.apply(wave, stencil::next(h), h, stencil::next(h), std::vector<DataHandle<T>>{c}, false);
      dd.swap();
      std::vector<T> nu = host_apply(wave, u, prev, ch, X, Y, Z);
      prev.swap(u);
      u.swap(nu);
    }
    const std::vector<T> got = gather<T>(dd, h.id(), stencil::Which::curr, X, Y, Z);
    if (std::memcmp(got.data(), u.data(), u.size() * sizeof(T))) {
      if (0 == mpi::world_rank()) std::fprintf(stderr, "variable-speed wave (%zu-byte elements): device and host bits differ\n", sizeof(T));
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
    std::printf("DistributedDomain::apply with coefficient fields, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
