// Golden-vector generator: links the REFERENCE's own host code (compiled where it lies under
// the reference checkout, never copied) and dumps its answers for the geometry / partition / ordering
// functions of the halo-exchange path as JSON.  Runs without a GPU (only
// host functions are called).  Output is committed as tests/golden/ref_geometry.json by
// oracle/ref/make_golden.sh.  TEST INFRASTRUCTURE.
#include <cstdio>
#include <vector>
#include <algorithm>

#include "stencil/align.cuh"
#include "stencil/dim3.hpp"
#include "stencil/local_domain.cuh"
#include "stencil/numeric.hpp"
#include "stencil/partition.hpp"
#include "stencil/radius.hpp"
#include "stencil/tx_common.hpp"

static void pd(const Dim3 &d) { std::printf("[%ld,%ld,%ld]", (long)d.x, (long)d.y, (long)d.z); }

struct RadSpec {
  const char *name;
  Radius r;
};

static std::vector<RadSpec> radii() {
  std::vector<RadSpec> v;
  v.push_back({"c0", Radius::constant(0)});
  v.push_back({"c1", Radius::constant(1)});
  v.push_back({"c2", Radius::constant(2)});
  v.push_back({"c3", Radius::constant(3)});
  v.push_back({"c4", Radius::constant(4)});
  v.push_back({"f1", Radius::face_edge_corner(1, 0, 0)});
  v.push_back({"f2e1", Radius::face_edge_corner(2, 1, 0)});
  v.push_back({"f3e2c1", Radius::face_edge_corner(3, 2, 1)});
  {
    Radius r = Radius::constant(0);
    r.dir(1, 0, 0) = 2;
    r.dir(-1, 0, 0) = 1;
    v.push_back({"px2mx1", r});
  }
  {
    Radius r = Radius::constant(0);
    r.dir(1, 0, 0) = 2;
    v.push_back({"px2", r});
  }
  {
    Radius r = Radius::constant(1);
    r.dir(0, 1, 0) = 3;
    r.dir(0, 0, -1) = 2;
    v.push_back({"c1py3mz2", r});
  }
  return v;
}

static void dump_radius(const Radius &r) {
  std::printf("[");
  bool first = true;
  for (int z = -1; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) {
        std::printf("%s%zu", first ? "" : ",", r.dir(x, y, z));
        first = false;
      }
  std::printf("]");
}

int main() {
  std::printf("{\n");

  // ---- prime_factors (src/numeric.cpp)
  std::printf("\"prime_factors\": {");
  {
    const int64_t ns[] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 16, 18, 24, 27, 30, 32, 36, 49, 64, 97, 128, 210, 1024, 1001};
    bool first = true;
    for (int64_t n : ns) {
      std::printf("%s\"%ld\": [", first ? "" : ", ", (long)n);
      first = false;
      auto f = prime_factors(n);
      for (size_t i = 0; i < f.size(); ++i) std::printf("%s%ld", i ? "," : "", (long)f[i]);
      std::printf("]");
    }
  }
  std::printf("},\n");

  // ---- RankPartition (partition.hpp:20-116)
  std::printf("\"rank_partition\": [\n");
  {
    struct C {
      Dim3 sz;
      int n;
    };
    const C cs[] = {{Dim3(10, 5, 5), 2},    {Dim3(10, 3, 1), 4},     {Dim3(10, 5, 5), 3},     {Dim3(13, 7, 7), 4},
                    {Dim3(10, 14, 2), 9},   {Dim3(512, 512, 512), 8}, {Dim3(512, 512, 512), 6}, {Dim3(100, 200, 300), 12},
                    {Dim3(17, 19, 23), 30}, {Dim3(64, 64, 64), 1},    {Dim3(7, 7, 7), 7},      {Dim3(1024, 512, 512), 2}};
    bool first = true;
    for (const C &c : cs) {
      RankPartition p(c.sz, c.n);
      std::printf("%s{\"size\": ", first ? "" : ",\n");
      first = false;
      pd(c.sz);
      std::printf(", \"n\": %d, \"dim\": ", c.n);
      pd(p.dim());
      std::printf(", \"subdomains\": [");
      Dim3 dim = p.dim();
      bool f2 = true;
      for (int64_t z = 0; z < dim.z; ++z)
        for (int64_t y = 0; y < dim.y; ++y)
          for (int64_t x = 0; x < dim.x; ++x) {
            Dim3 idx(x, y, z);
            std::printf("%s{\"idx\": ", f2 ? "" : ", ");
            f2 = false;
            pd(idx);
            std::printf(", \"size\": ");
            pd(p.subdomain_size(idx));
            std::printf(", \"origin\": ");
            pd(p.subdomain_origin(idx));
            std::printf(", \"lin\": %zu}", p.linearize(idx));
          }
      std::printf("]}");
    }
  }
  std::printf("\n],\n");

  // ---- NodePartition (partition.hpp:120-256)
  std::printf("\"node_partition\": [\n");
  {
    struct C {
      Dim3 sz;
      int nodes, gpus;
    };
    const C cs[] = {{Dim3(512, 512, 512), 1, 1},  {Dim3(512, 512, 512), 1, 2}, {Dim3(512, 512, 512), 1, 4},
                    {Dim3(512, 512, 512), 1, 8},  {Dim3(1024, 512, 512), 1, 2}, {Dim3(1024, 1024, 512), 1, 4},
                    {Dim3(1024, 1024, 1024), 1, 8}, {Dim3(10, 10, 10), 1, 2},   {Dim3(10, 10, 10), 2, 2},
                    {Dim3(100, 60, 30), 1, 6},    {Dim3(13, 17, 19), 3, 4},    {Dim3(256, 256, 256), 2, 8},
                    {Dim3(30, 40, 50), 1, 3}};
    bool first = true;
    for (auto &rs : radii()) {
      for (const C &c : cs) {
        NodePartition p(c.sz, rs.r, c.nodes, c.gpus);
        std::printf("%s{\"size\": ", first ? "" : ",\n");
        first = false;
        pd(c.sz);
        std::printf(", \"radius\": \"%s\", \"nodes\": %d, \"gpus\": %d, \"sys_dim\": ", rs.name, c.nodes, c.gpus);
        pd(p.sys_dim());
        std::printf(", \"node_dim\": ");
        pd(p.node_dim());
        std::printf(", \"subdomains\": [");
        Dim3 dim = p.dim();
        bool f2 = true;
        for (int64_t z = 0; z < dim.z; ++z)
          for (int64_t y = 0; y < dim.y; ++y)
            for (int64_t x = 0; x < dim.x; ++x) {
              Dim3 idx(x, y, z);
              std::printf("%s{\"idx\": ", f2 ? "" : ", ");
              f2 = false;
              pd(idx);
              std::printf(", \"size\": ");
              pd(p.subdomain_size(idx));
              std::printf(", \"origin\": ");
              pd(p.subdomain_origin(idx));
              std::printf("}");
            }
        std::printf("]}");
      }
    }
  }
  std::printf("\n],\n");

  // ---- radius tables
  std::printf("\"radii\": {");
  {
    bool first = true;
    for (auto &rs : radii()) {
      std::printf("%s\"%s\": ", first ? "" : ", ", rs.name);
      first = false;
      dump_radius(rs.r);
    }
  }
  std::printf("},\n");

  // ---- halo_pos / halo_extent (src/local_domain.cu:86-125, local_domain.cuh:212-222)
  std::printf("\"halo\": [\n");
  {
    const Dim3 szs[] = {Dim3(3, 4, 5), Dim3(30, 40, 50), Dim3(512, 512, 512), Dim3(1, 1, 1), Dim3(5, 10, 10)};
    bool first = true;
    for (auto &rs : radii()) {
      for (const Dim3 &sz : szs) {
        std::printf("%s{\"size\": ", first ? "" : ",\n");
        first = false;
        pd(sz);
        std::printf(", \"radius\": \"%s\", \"dirs\": [", rs.name);
        bool f2 = true;
        for (int z = -1; z <= 1; ++z)
          for (int y = -1; y <= 1; ++y)
            for (int x = -1; x <= 1; ++x) {
              Dim3 dir(x, y, z);
              std::printf("%s{\"dir\": ", f2 ? "" : ", ");
              f2 = false;
              pd(dir);
              std::printf(", \"pos_halo\": ");
              pd(LocalDomain::halo_pos(dir, sz, rs.r, true));
              std::printf(", \"pos_interior\": ");
              pd(LocalDomain::halo_pos(dir, sz, rs.r, false));
              std::printf(", \"extent\": ");
              pd(LocalDomain::halo_extent(dir, sz, rs.r));
              std::printf("}");
            }
        std::printf("]}");
      }
    }
  }
  std::printf("\n],\n");

  // ---- LocalDomain members that need no allocation: raw_size, halo_coords, full region, accessor origin
  std::printf("\"local_domain\": [\n");
  {
    struct C {
      Dim3 sz, origin;
    };
    const C cs[] = {{Dim3(3, 4, 5), Dim3(0, 0, 0)}, {Dim3(30, 40, 50), Dim3(30, 0, 100)}, {Dim3(5, 10, 10), Dim3(5, 0, 0)}};
    bool first = true;
    for (auto &rs : radii()) {
      for (const C &c : cs) {
        // leaked on purpose: ~LocalDomain makes CUDA runtime calls, which are fatal without a GPU
        LocalDomain &ld = *new LocalDomain(c.sz, c.origin, 0);
        ld.set_radius(rs.r);
        std::printf("%s{\"size\": ", first ? "" : ",\n");
        first = false;
        pd(c.sz);
        std::printf(", \"origin\": ");
        pd(c.origin);
        std::printf(", \"radius\": \"%s\", \"raw_size\": ", rs.name);
        pd(ld.raw_size());
        Rect3 fr = ld.get_full_region();
        std::printf(", \"full_lo\": ");
        pd(fr.lo);
        std::printf(", \"full_hi\": ");
        pd(fr.hi);
        std::printf(", \"coords\": [");
        bool f2 = true;
        for (int z = -1; z <= 1; ++z)
          for (int y = -1; y <= 1; ++y)
            for (int x = -1; x <= 1; ++x) {
              Dim3 dir(x, y, z);
              Rect3 h = ld.halo_coords(dir, true), i = ld.halo_coords(dir, false);
              std::printf("%s{\"dir\": ", f2 ? "" : ", ");
              f2 = false;
              pd(dir);
              std::printf(", \"halo_lo\": ");
              pd(h.lo);
              std::printf(", \"halo_hi\": ");
              pd(h.hi);
              std::printf(", \"int_lo\": ");
              pd(i.lo);
              std::printf(", \"int_hi\": ");
              pd(i.hi);
              std::printf("}");
            }
        std::printf("]}");
      }
    }
  }
  std::printf("\n],\n");

  // ---- Message::by_size ordering (tx_common.hpp:25-36) with the planner's extents
  std::printf("\"message_order\": [\n");
  {
    const Dim3 szs[] = {Dim3(3, 4, 5), Dim3(30, 40, 50), Dim3(8, 8, 8)};
    bool first = true;
    for (auto &rs : radii()) {
      for (const Dim3 &sz : szs) {
        std::vector<Message> msgs;
        for (int z = -1; z <= 1; ++z)
          for (int y = -1; y <= 1; ++y)
            for (int x = -1; x <= 1; ++x) {
              Dim3 dir(x, y, z);
              if (dir == Dim3(0, 0, 0)) continue;
              if (0 == rs.r.dir(dir * -1)) continue;
              msgs.push_back(Message(dir, 0, 0, LocalDomain::halo_extent(dir * -1, sz, rs.r)));
            }
        std::sort(msgs.begin(), msgs.end(), Message::by_size);
        std::printf("%s{\"size\": ", first ? "" : ",\n");
        first = false;
        pd(sz);
        std::printf(", \"radius\": \"%s\", \"order\": [", rs.name);
        for (size_t i = 0; i < msgs.size(); ++i) {
          std::printf("%s", i ? "," : "");
          pd(msgs[i].dir_);
        }
        std::printf("]}");
      }
    }
  }
  std::printf("\n],\n");

  // ---- make_block_dim (dim3.hpp:233-254), next_align_of (align.cuh), wrap (dim3.hpp:208-229)
  std::printf("\"make_block_dim\": [");
  {
    const Dim3 es[] = {Dim3(510, 510, 510), Dim3(1, 512, 512), Dim3(512, 1, 512), Dim3(512, 512, 1), Dim3(3, 4, 5),
                       Dim3(2, 2, 512),     Dim3(100, 3, 7),   Dim3(1, 1, 1)};
    const int64_t ts[] = {256, 512, 1024, 2048};
    bool first = true;
    for (auto &e : es)
      for (auto t : ts) {
        std::printf("%s{\"ext\": ", first ? "" : ", ");
        first = false;
        pd(e);
        std::printf(", \"threads\": %ld, \"block\": ", (long)t);
        pd(Dim3::make_block_dim(e, t));
        std::printf("}");
      }
  }
  std::printf("],\n\"next_align_of\": [");
  {
    bool first = true;
    for (size_t a : {size_t(1), size_t(2), size_t(4), size_t(8), size_t(16)})
      for (size_t x : {size_t(0), size_t(1), size_t(3), size_t(4), size_t(7), size_t(8), size_t(100), size_t(104), size_t(1021)}) {
        std::printf("%s[%zu,%zu,%zu]", first ? "" : ",", x, a, next_align_of(x, a));
        first = false;
      }
  }
  std::printf("],\n\"wrap\": [");
  {
    bool first = true;
    const Dim3 lims[] = {Dim3(2, 2, 2), Dim3(1, 1, 1), Dim3(3, 2, 1), Dim3(4, 4, 4)};
    for (auto &l : lims)
      for (int z = -1; z <= l.z; ++z)
        for (int y = -1; y <= l.y; ++y)
          for (int x = -1; x <= l.x; ++x) {
            Dim3 p(x, y, z);
            Dim3 w = Dim3(p).wrap(l);
            std::printf("%s[", first ? "" : ",");
            first = false;
            pd(p);
            std::printf(",");
            pd(l);
            std::printf(",");
            pd(w);
            std::printf("]");
          }
  }
  std::printf("]\n}\n");
  return 0;
}
