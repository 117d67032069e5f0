// C++ API check of the reductions (DistributedDomain::reduce*, FusedJacobi3d::residual) -- one process with N
// subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs
// than ranks).
//   bin/test_reduce_multigpu --single N OUT     one process, N subdomains: checks against the host, writes the result bits
//   bin/sb_mpirun -n N bin/test_reduce_multigpu --expect OUT
//                                               one subdomain per rank: checks against the host, and every rank's bits
//                                               must equal OUT's (the same partition run in one process)
// Ghost cells hold NaN (every byte 0xff), so a reduction that read one would give NaN.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "stencil/jacobi3d.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::ReduceItem;
using stencil::Reduction;
using stencil::Which;

// multiples of 2^-10 in [-4, 4): exact in float and double, so the device (which may contract into an FMA) and the host
// form the same values
template <typename T> __host__ __device__ T field(int q, int64_t x, int64_t y, int64_t z) {
  return T(double((x * 7 + y * 131 + z * 1009 + q * 3) % 8191) * 0.0009765625 - 4.0);
}

template <typename T> __global__ void fill(Accessor<T> acc, Rect3 reg, int q) {
  for (int64_t z = reg.lo.z + blockIdx.z; z < reg.hi.z; z += gridDim.z)
    for (int64_t y = reg.lo.y + blockIdx.y; y < reg.hi.y; y += gridDim.y)
      for (int64_t x = reg.lo.x + threadIdx.x; x < reg.hi.x; x += blockDim.x) acc[Dim3(x, y, z)] = field<T>(q, x, y, z);
}

static std::string hex(const Reduction &r) {
  unsigned char b[40];
  std::memcpy(b, &r.min, 8);
  std::memcpy(b + 8, &r.max, 8);
  std::memcpy(b + 16, &r.sum, 8);
  std::memcpy(b + 24, &r.sumsq, 8);
  std::memcpy(b + 32, &r.count, 8);
  std::string s;
  char c[3];
  for (unsigned char v : b) {
    std::snprintf(c, sizeof(c), "%02x", v);
    s += c;
  }
  return s;
}

// Host restatement over the whole grid: v per cell, exact min / max, sums in long double (the kernel's FP64 sums must be
// within (k + h + 1) * 2^-53 * sum |term| of them, DESIGN section 2.6; 1e-12 relative is far looser for these shapes).
struct Host {
  double mn = INFINITY, mx = -INFINITY;
  long double s = 0, q = 0, as = 0;
  int64_t n = 0;
  void add(double v, double qq) {
    mn = v < mn ? v : mn;
    mx = v > mx ? v : mx;
    s += v;
    q += qq;
    as += std::fabs(v);
    ++n;
  }
};

static long check(const char *what, const Reduction &r, const Host &h) {
  const bool ok = r.count == h.n && r.min == h.mn && r.max == h.mx && std::fabs(double(r.sum - h.s)) <= 1e-12 * double(h.as) &&
                  std::fabs(double(r.sumsq - h.q)) <= 1e-12 * double(h.q);
  if (!ok && 0 == mpi::world_rank())
    std::fprintf(stderr, "%s: got min %.17g max %.17g sum %.17g sumsq %.17g count %ld; want %.17g %.17g %.17Lg %.17Lg %ld\n", what, r.min, r.max, r.sum,
                 r.sumsq, long(r.count), h.mn, h.mx, h.s, h.q, long(h.n));
  return ok ? 0 : 1;
}

template <typename T> static long run_fields(const std::vector<int> &gpus, size_t X, size_t Y, size_t Z, size_t radius, std::vector<std::string> &bits) {
  DistributedDomain dd(X, Y, Z);
  dd.set_gpus(gpus);
  dd.set_radius(radius);
  auto a = dd.add_data<T>("a");
  auto b = dd.add_data<T>("b");
  auto c = dd.add_data<T>("c");
  dd.realize();
  for (auto &d : dd.domains()) {
    d.set_device();
    const Dim3 rs = d.raw_size();
    for (size_t q = 0; q < 3; ++q) {
      CUDA_RUNTIME(cudaMemset(d.curr_data(q).ptr, 0xff, size_t(rs.x * rs.y * rs.z) * sizeof(T)));
      CUDA_RUNTIME(cudaMemset(d.next_data(q).ptr, 0xff, size_t(rs.x * rs.y * rs.z) * sizeof(T)));
    }
    const Rect3 reg = d.get_compute_region();
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(a), reg, 0);
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(b), reg, 1);
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_curr_accessor(c), reg, 2);
    fill<T><<<dim3(1, 8, 8), 64>>>(d.get_next_accessor(a), reg, 3);
  }
  // no synchronisation here: reduce_many waits for the queued fills
  const std::vector<Reduction> rs = dd.reduce_many({ReduceItem::scalar(a), ReduceItem::scalar(a, Which::next), ReduceItem::diff(a), ReduceItem::norm(a, b, c)});
  Host hs, hn, hd, hm;
  for (int64_t z = 0; z < int64_t(Z); ++z)
    for (int64_t y = 0; y < int64_t(Y); ++y)
      for (int64_t x = 0; x < int64_t(X); ++x) {
        const double va = double(field<T>(0, x, y, z)), vb = double(field<T>(1, x, y, z)), vc = double(field<T>(2, x, y, z)),
                     vn = double(field<T>(3, x, y, z));
        hs.add(va, va * va);
        hn.add(vn, vn * vn);
        const double dv = va - vn;
        hd.add(dv, dv * dv);
        const double s = (va * va + vb * vb) + vc * vc;
        hm.add(std::sqrt(s), s);
      }
  long bad = check("scalar", rs[0], hs) + check("scalar next", rs[1], hn) + check("diff", rs[2], hd) + check("norm", rs[3], hm);
  // the single forms give the list form's bits; after swap() the old next is the new curr
  bad += hex(dd.reduce(a)) != hex(rs[0]);
  bad += hex(dd.reduce_diff(a)) != hex(rs[2]);
  bad += hex(dd.reduce_norm(a, b, c)) != hex(rs[3]);
  dd.swap();
  bad += hex(dd.reduce(a)) != hex(rs[1]);
  bad += hex(dd.reduce(a, Which::next)) != hex(rs[0]);
  dd.swap();
  for (const Reduction &r : rs) bits.push_back(hex(r));
  return bad;
}

static long run_jacobi(const std::vector<int> &gpus, size_t n, std::vector<std::string> &bits) {
  DistributedDomain dd(n, n, n);
  dd.set_gpus(gpus);
  dd.set_radius(Radius::face_edge_corner(1, 0, 0));
  auto h = dd.add_data<double>("d");
  dd.realize();
  stencil::FusedJacobi3d jac(dd, h);
  jac.init(0.5);
  for (int it = 0; it < 5; ++it) jac.step();
  const double res = jac.residual(); // ordered after the queued iterations
  jac.synchronize();
  // host: ||curr - next|| over the compute cells of every subdomain, summed over the ranks
  long double part = 0;
  for (auto &d : dd.domains()) {
    const Dim3 rs = d.raw_size(), sz = d.size();
    std::vector<double> cur(size_t(rs.x * rs.y * rs.z)), nxt(cur.size());
    d.set_device();
    CUDA_RUNTIME(cudaMemcpy(cur.data(), d.curr_data(0).ptr, cur.size() * 8, cudaMemcpyDeviceToHost));
    CUDA_RUNTIME(cudaMemcpy(nxt.data(), d.next_data(0).ptr, nxt.size() * 8, cudaMemcpyDeviceToHost));
    for (int64_t z = 1; z <= sz.z; ++z)
      for (int64_t y = 1; y <= sz.y; ++y)
        for (int64_t x = 1; x <= sz.x; ++x) {
          const size_t i = size_t((z * rs.y + y) * rs.x + x);
          const double dv = cur[i] - nxt[i];
          part += dv * dv;
        }
  }
  double mine = double(part), total = 0;
  MPI_Allreduce(&mine, &total, 1, MPI_DOUBLE, MPI_SUM, MPI_COMM_WORLD);
  long bad = 0;
  if (!(res > 0) || std::fabs(res * res - total) > 1e-12 * total) {
    if (0 == mpi::world_rank()) std::fprintf(stderr, "residual %.17g, host %.17g\n", res, std::sqrt(total));
    ++bad;
  }
  char buf[32];
  std::snprintf(buf, sizeof(buf), "%a", res);
  bits.push_back(buf);
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
  long bad = 0;
  bad += run_fields<double>(gpus, 40, 36, 28, 2, bits);
  bad += run_fields<float>(gpus, 33, 30, 26, 1, bits);
  bad += run_jacobi(gpus, 48, bits);
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
    std::printf("reductions and FusedJacobi3d::residual, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
