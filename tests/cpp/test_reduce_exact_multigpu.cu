// C++ API check of the exact reductions (DistributedDomain::reduce*(..., stencil::Sum::exact)) -- one process with N
// subdomains on GPU 0, or one subdomain per rank under bin/sb_mpirun -n N (ranks share GPUs when there are fewer GPUs
// than ranks).
//   bin/test_reduce_exact_multigpu --single N OUT  one process, N subdomains: checks against the host, writes the bits
//   bin/sb_mpirun -n N bin/test_reduce_exact_multigpu --expect OUT
//                                                  one subdomain per rank: checks against the host, and every rank's
//                                                  bits must equal OUT's -- written by a run of ANY partition, since
//                                                  exact sums do not depend on it
// The fields are k * 2^-10 * 2^e with |k| < 4096 and e in [-20, 20): exact in float and double, spread over 40 binades
// so that ordered sums depend on the partition, and summable exactly on the host in __int128.  Ghost cells hold NaN
// (every byte 0xff), so a reduction that read one would give NaN.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::ReduceItem;
using stencil::Reduction;
using stencil::Sum;
using stencil::Which;

__host__ __device__ inline int64_t field_k(int q, int64_t x, int64_t y, int64_t z) { return (x * 7 + y * 131 + z * 1009 + q * 3) % 8191 - 4095; }
__host__ __device__ inline int field_e(int q, int64_t x, int64_t y, int64_t z) { return int((x * 3 + y * 5 + z * 11 + q) % 40) - 20; }
template <typename T> __host__ __device__ T field(int q, int64_t x, int64_t y, int64_t z) {
  return T(ldexp(double(field_k(q, x, y, z)), field_e(q, x, y, z) - 10));
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

// Host: v in units of 2^-30 and q = v * v (rounded as the kernel rounds it; a multiple of 2^-60) in units of 2^-60,
// summed exactly in __int128, converted once (correctly rounded) and scaled by a power of two (exact: the results are
// normal doubles).
struct Host {
  double mn = INFINITY, mx = -INFINITY;
  __int128 s = 0, q = 0;
  int64_t n = 0;
  void add(double v) {
    mn = v < mn ? v : mn;
    mx = v > mx ? v : mx;
    s += __int128(std::ldexp(v, 30)); // exact: v is a multiple of 2^-30 below 2^53 units
    q += __int128(std::ldexp(v * v, 60));
    ++n;
  }
  double sum() const { return std::ldexp(double(s), -30); }
  double sumsq() const { return std::ldexp(double(q), -60); }
};

static long check(const char *what, const Reduction &r, const Host &h) {
  const bool ok = r.count == h.n && r.min == h.mn && r.max == h.mx && r.sum == h.sum() && r.sumsq == h.sumsq();
  if (!ok && 0 == mpi::world_rank())
    std::fprintf(stderr, "%s: got min %a max %a sum %a sumsq %a count %ld; want %a %a %a %a %ld\n", what, r.min, r.max, r.sum, r.sumsq,
                 long(r.count), h.mn, h.mx, h.sum(), h.sumsq(), long(h.n));
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
  const std::vector<ReduceItem> items{ReduceItem::scalar(a), ReduceItem::scalar(a, Which::next), ReduceItem::diff(a), ReduceItem::norm(a, b, c)};
  const std::vector<Reduction> rs = dd.reduce_many(items, Sum::exact);
  Host hs, hn, hd;
  for (int64_t z = 0; z < int64_t(Z); ++z)
    for (int64_t y = 0; y < int64_t(Y); ++y)
      for (int64_t x = 0; x < int64_t(X); ++x) {
        const double va = double(field<T>(0, x, y, z)), vn = double(field<T>(3, x, y, z));
        hs.add(va);
        hn.add(vn);
        hd.add(va - vn); // exact: both are multiples of 2^-30 below 2^21
      }
  long bad = check("scalar", rs[0], hs) + check("scalar next", rs[1], hn) + check("diff", rs[2], hd);
  // the norm's q and sqrt round, so no host value: its bits are checked across partitions (OUT); its min / max / count
  // are the ordered plan's on one subdomain
  const std::vector<Reduction> ord = dd.reduce_many(items);
  if (1 == gpus.size() * size_t(mpi::world_size()))
    for (size_t i = 0; i < rs.size(); ++i) bad += rs[i].min != ord[i].min || rs[i].max != ord[i].max || rs[i].count != ord[i].count;
  // the single forms give the list form's bits; after swap() the old next is the new curr
  bad += hex(dd.reduce(a, Which::curr, Sum::exact)) != hex(rs[0]);
  bad += hex(dd.reduce_diff(a, Sum::exact)) != hex(rs[2]);
  bad += hex(dd.reduce_norm(a, b, c, Sum::exact)) != hex(rs[3]);
  dd.swap();
  bad += hex(dd.reduce(a, Which::curr, Sum::exact)) != hex(rs[1]);
  bad += hex(dd.reduce(a, Which::next, Sum::exact)) != hex(rs[0]);
  dd.swap();
  for (const Reduction &r : rs) bits.push_back(hex(r));
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
  if (single) {
    std::ofstream f(argv[3]);
    for (const std::string &b : bits) f << b << "\n";
  } else {
    std::ifstream f(argv[2]);
    std::vector<std::string> want;
    for (std::string line; std::getline(f, line);) want.push_back(line);
    if (want != bits) {
      std::fprintf(stderr, "rank %d: exact result bits differ from the one-process run\n", mpi::world_rank());
      ++bad;
    }
  }
  long long all = bad;
  MPI_Allreduce(MPI_IN_PLACE, &all, 1, MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
  if (0 == mpi::world_rank()) {
    std::printf("exact reductions, %zu subdomain(s) on %d rank(s): %s\n", nsub, mpi::world_size(), all ? "FAIL" : "ok");
    std::printf(all ? "FAILED\n" : "ALL OK\n");
  }
  MPI_Finalize();
  return all ? 1 : 0;
}
