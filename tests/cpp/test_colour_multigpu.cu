// C++ API check of coloured application (DistributedDomain::apply with a stencil::Colour, LinearStencil::relax) -- one
// process with N subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are
// fewer GPUs than ranks).
//   bin/test_colour_multigpu --single N OUT      one process, N subdomains: checks against the host, writes the result bits
//   bin/sb_mpirun -n N bin/test_colour_multigpu --expect OUT
//                                               one subdomain per rank: checks against the host, and every rank's bits
//                                               must equal OUT's (the one-process run)
// Runs, in float and double: 4 red-black SOR sweeps of a periodic Helmholtz problem -lap u + sigma u = f, in place with
// f on aux (overlapped with the exchange), and one 8-colour sweep of a 27-point relaxation (exchange = false after a
// manual exchange()), and 3 red-black sweeps of an upwind relaxation on a radius of 1 on the low faces only, on odd
// periodic x and y lengths.  The host restatement evaluates each colour pass on the state before it, on the global periodic
// grid, with the same separately rounded operations, and keeps every cell of another colour.
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

// a field in [-4, 4)
template <typename T> __host__ __device__ T field(int q, int64_t x, int64_t y, int64_t z) {
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


// the colour pass on the host: the cells of colour c under m take op(u, aux), the others keep u's value
template <typename T>
std::vector<T> host_colour(const LinearStencil &op, const std::vector<T> &u, const std::vector<T> &aux, int64_t X, int64_t Y, int64_t Z, int m, int c) {
  const std::vector<T> all = host_apply(op, u, aux, {}, X, Y, Z);
  std::vector<T> out(u);
  for (int64_t z = 0; z < Z; ++z)
    for (int64_t y = 0; y < Y; ++y)
      for (int64_t x = 0; x < X; ++x) {
        const int col = m == 2 ? int((x + y + z) & 1) : int((x & 1) | (y & 1) << 1 | (z & 1) << 2);
        const size_t i = size_t((z * Y + y) * X + x);
        if (col == c) out[i] = all[i];
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

template <typename T> static long run(const std::vector<int> &gpus, std::vector<std::string> &bits) {
  const int64_t X = 34, Y = 22, Z = 18;
  long bad = 0;
  {
    DistributedDomain dd(X, Y, Z);
    dd.set_gpus(gpus);
    dd.set_radius(Radius::face_edge_corner(1, 0, 0));
    auto h = dd.add_data<T>("u");
    auto f = dd.add_data<T>("f");
    dd.realize();
    for (auto &d : dd.domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h), d.get_compute_region(), 0);
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(f), d.get_compute_region(), 1);
    }
    // A = -lap + sigma, then its SOR update
    LinearStencil A;
    const LinearStencil lap = LinearStencil::laplacian(2, 1.0, 1.0, 1.0);
    A.add(Source::src, 0, 0, 0, -lap.terms()[0].weight + 0.3);
    for (size_t k = 1; k < lap.terms().size(); ++k) {
      const sb_stencil_term &t = lap.terms()[k];
      A.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight);
    }
    const LinearStencil sor = A.relax(1.6);
    if (sor.terms().size() != 8 || sor.terms()[7].source != 1 || sor.terms()[0].weight != 1.0 - 1.6) {
      std::fprintf(stderr, "relax: %zu terms\n", sor.terms().size());
      ++bad;
    }
    std::vector<T> u = host_field<T>(0, X, Y, Z);
    const std::vector<T> fh = host_field<T>(1, X, Y, Z);
    for (int it = 0; it < 4; ++it)
      for (int c = 0; c < 2; ++c) {
        dd.apply(sor, stencil::curr(h), h, stencil::curr(f), stencil::Colour{2, c});
        u = host_colour(sor, u, fh, X, Y, Z, 2, c);
      }
    const std::vector<T> got = gather<T>(dd, h.id(), stencil::Which::curr, X, Y, Z);
    if (std::memcmp(got.data(), u.data(), u.size() * sizeof(T))) {
      if (0 == mpi::world_rank()) std::fprintf(stderr, "red-black SOR (%zu-byte elements): device and host bits differ\n", sizeof(T));
      ++bad;
    }
    bits.push_back(hexsum(got));
  }
  {
    DistributedDomain dd(X, Y, Z);
    dd.set_gpus(gpus);
    dd.set_radius(Radius::face_edge_corner(1, 1, 1));
    auto h = dd.add_data<T>("u");
    auto f = dd.add_data<T>("f");
    dd.realize();
    for (auto &d : dd.domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h), d.get_compute_region(), 2);
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(f), d.get_compute_region(), 3);
    }
    LinearStencil A;
    A.add(Source::src, 0, 0, 0, 30.0);
    for (int z = -1; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x)
          if (x || y || z) A.add(Source::src, x, y, z, -0.125 * double(1 + ((x + 2 * y + 3 * z + 9) % 5)));
    const LinearStencil sor = A.relax(1.2);
    std::vector<T> u = host_field<T>(2, X, Y, Z);
    const std::vector<T> fh = host_field<T>(3, X, Y, Z);
    for (int c = 0; c < 8; ++c) {
      for (auto &d : dd.domains()) {
        d.set_device();
        CUDA_RUNTIME(cudaDeviceSynchronize());
      }
      dd.exchange();
      dd.apply(sor, stencil::curr(h), h, stencil::curr(f), stencil::Colour{8, c}, false);
      u = host_colour(sor, u, fh, X, Y, Z, 8, c);
    }
    const std::vector<T> got = gather<T>(dd, h.id(), stencil::Which::curr, X, Y, Z);
    if (std::memcmp(got.data(), u.data(), u.size() * sizeof(T))) {
      if (0 == mpi::world_rank()) std::fprintf(stderr, "8-colour sweep (%zu-byte elements): device and host bits differ\n", sizeof(T));
      ++bad;
    }
    bits.push_back(hexsum(got));
  }
  {
    // an upwind relaxation in place on a radius of 1 on the low faces only, periodic with odd x and y lengths: the wrapped
    // ghost of x = 0 holds cell X2 - 1, of the same colour, which exchange() reads while the interior runs (an even cell
    // count: gather merges whole 8-byte words)
    const int64_t X2 = 33, Y2 = 21, Z2 = 18;
    DistributedDomain dd(X2, Y2, Z2);
    dd.set_gpus(gpus);
    Radius r = Radius::face_edge_corner(0, 0, 0);
    r.dir(-1, 0, 0) = r.dir(0, -1, 0) = r.dir(0, 0, -1) = 1;
    dd.set_radius(r);
    auto h = dd.add_data<T>("u");
    auto f = dd.add_data<T>("f");
    dd.realize();
    for (auto &d : dd.domains()) {
      d.set_device();
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(h), d.get_compute_region(), 4);
      fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(f), d.get_compute_region(), 5);
    }
    LinearStencil A;
    A.add(Source::src, 0, 0, 0, 4.0).add(Source::src, -1, 0, 0, -1.0).add(Source::src, 0, -1, 0, -0.75).add(Source::src, 0, 0, -1, -0.5);
    const LinearStencil sor = A.relax(1.3);
    std::vector<T> u = host_field<T>(4, X2, Y2, Z2);
    const std::vector<T> fh = host_field<T>(5, X2, Y2, Z2);
    for (int it = 0; it < 3; ++it)
      for (int c = 0; c < 2; ++c) {
        dd.apply(sor, stencil::curr(h), h, stencil::curr(f), stencil::Colour{2, c});
        u = host_colour(sor, u, fh, X2, Y2, Z2, 2, c);
      }
    const std::vector<T> got = gather<T>(dd, h.id(), stencil::Which::curr, X2, Y2, Z2);
    if (std::memcmp(got.data(), u.data(), u.size() * sizeof(T))) {
      if (0 == mpi::world_rank()) std::fprintf(stderr, "upwind, one-sided radius (%zu-byte elements): device and host bits differ\n", sizeof(T));
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
    std::printf("coloured DistributedDomain::apply, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
