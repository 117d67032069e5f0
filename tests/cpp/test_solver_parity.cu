// The C++ solvers against the numpy oracles (DESIGN.md section 2.14): a harness driven by case directories that
// tests/test_gpu_cpp_solvers.py writes, so each problem is defined once, in Python, and the C++ results are compared
// bit for bit with tests/mg_oracle.py, vmg_oracle.py, krylov_oracle.py and bicgstab_oracle.py.
//   bin/test_solver_parity --single N OUT CASE...   one process, N subdomains on GPU 0
//   bin/sb_mpirun -n N bin/test_solver_parity --ranks OUT CASE...
//                                                    one subdomain per rank (ranks share GPUs when there are fewer)
// Rank 0 writes the gathered results of case directory CASE into OUT/<last component of CASE>/: raw little-endian
// arrays of the global interior ([z][y][x], the case's type) and info.txt (one "key value..." line per scalar, the
// histories as hex doubles).
//
// CASE/case.txt, one item per line:
//   size NX NY NZ | dtype f32|f64 | periodic 0|1 | solver mg|pcg|bicgstab|passes | precond 0|1 | levels L
//   nu NU1 NU2 COARSE_SWEEPS | iters K | coef_kinds KIND... | inputs NAME...
//   bc NAME FACE odd|even|value C        the BC of quantity NAME on face FACE (0 -x, 1 +x, .., 5 +z), C a hex double
//   op LEVEL NTERMS                       then NTERMS lines "SRC OX OY OZ W COEF CX CY CZ" (W a hex double, COEF -1: none)
// The quantities of each solver are the names below, then k0 .. k(n-1) for n coef_kinds; every name in `inputs` is
// loaded from CASE/NAME.bin before the first pass and again before every solve.
//   mg        u f r u2 f2       3 cycles (cycle1..3.bin); with coefficients the fields from ks<i>.bin,
//                               update_coefficients() and one cycle (update.bin); one cycle(u2, f2) from u2.bin and
//                               f2.bin (pair.bin); info: levels, colours
//   pcg       x f r z p q       solve(0, k) from x.bin for k = 1 .. K (x<k>.bin, hist<k>, breakdown<k>), then dd.swap(),
//   bicgstab  x f r r0 p v phat shat t   the inputs reloaded and solve(0, K) (swap.bin, hist_swap, breakdown_swap)
//   passes    u f r              on a second domain of half the size with w and cu (bc lines on cu are its BCs):
//                               apply (apply.bin), relax of colour 0 and 1 in place (relax0/1.bin), the coefficient
//                               residual restricted (restrict.bin), the face restriction of k0 .. k2 (face0..2.bin)
//                               and u += P cu with cu from cu.bin (prolong.bin)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
#include <string>
#include <sys/stat.h>
#include <vector>

#include "stencil/bicgstab.hpp"
#include "stencil/krylov.hpp"
#include "stencil/linear_stencil.hpp"
#include "stencil/multigrid.hpp"
#include "stencil/stencil.hpp"
#include "stencil_b200.h"

using stencil::curr;
using stencil::LinearStencil;
using stencil::Source;

struct Term {
  int src, o[3], coef, c[3];
  double w;
};

struct Case {
  std::string dir, name, dtype, solver;
  int64_t size[3] = {0, 0, 0};
  bool periodic = false, precond = true;
  int levels = 0, nu1 = 2, nu2 = 2, coarse = 30, iters = 3;
  std::vector<std::string> kinds, inputs;
  struct Wall {
    std::string q;
    int face;
    stencil::BC bc;
  };
  std::vector<Wall> bcs;
  std::vector<std::vector<Term>> ops;
};

static double hexd(const std::string &s) { return std::strtod(s.c_str(), nullptr); }

static Case parse(const std::string &dir) {
  Case c;
  c.dir = dir;
  const size_t slash = dir.find_last_of('/');
  c.name = slash == std::string::npos ? dir : dir.substr(slash + 1);
  std::ifstream in(dir + "/case.txt");
  if (!in) LOG_FATAL("cannot read " << dir << "/case.txt");
  std::string line;
  while (std::getline(in, line)) {
    std::istringstream ls(line);
    std::string key;
    if (!(ls >> key)) continue;
    if (key == "size") {
      ls >> c.size[0] >> c.size[1] >> c.size[2];
    } else if (key == "dtype") {
      ls >> c.dtype;
    } else if (key == "periodic") {
      int p;
      ls >> p;
      c.periodic = p != 0;
    } else if (key == "solver") {
      ls >> c.solver;
    } else if (key == "precond") {
      int p;
      ls >> p;
      c.precond = p != 0;
    } else if (key == "levels") {
      ls >> c.levels;
    } else if (key == "nu") {
      ls >> c.nu1 >> c.nu2 >> c.coarse;
    } else if (key == "iters") {
      ls >> c.iters;
    } else if (key == "coef_kinds" || key == "inputs") {
      std::vector<std::string> &v = key == "inputs" ? c.inputs : c.kinds;
      for (std::string s; ls >> s;) v.push_back(s);
    } else if (key == "bc") {
      std::string q, kind, val;
      int face;
      ls >> q >> face >> kind >> val;
      const stencil::BC bc = kind == "odd" ? stencil::BC::ODD(hexd(val)) : kind == "even" ? stencil::BC::EVEN() : stencil::BC::VALUE(hexd(val));
      c.bcs.push_back(Case::Wall{q, face, bc});
    } else if (key == "op") {
      size_t l, n;
      ls >> l >> n;
      if (c.ops.size() <= l) c.ops.resize(l + 1);
      for (size_t i = 0; i < n && std::getline(in, line); ++i) {
        std::istringstream ts(line);
        Term t;
        std::string w;
        ts >> t.src >> t.o[0] >> t.o[1] >> t.o[2] >> w >> t.coef >> t.c[0] >> t.c[1] >> t.c[2];
        t.w = hexd(w);
        c.ops[l].push_back(t);
      }
    } else {
      LOG_FATAL(dir << "/case.txt: unknown item " << key);
    }
  }
  return c;
}

static LinearStencil op_of(const Case &c, int l) {
  if (l < 0 || size_t(l) >= c.ops.size()) LOG_FATAL(c.name << ": no op for level " << l);
  LinearStencil A;
  for (const Term &t : c.ops[size_t(l)]) A.add(Source(t.src), t.o[0], t.o[1], t.o[2], t.w, t.coef, t.c[0], t.c[1], t.c[2]);
  return A;
}

static Dim3 face_dir(int fc) {
  const int s = fc % 2 ? 1 : -1;
  return Dim3(fc / 2 == 0 ? s : 0, fc / 2 == 1 ? s : 0, fc / 2 == 2 ? s : 0);
}

// the global interior [z][y][x] of quantity q into the curr allocation of every local subdomain (ghost cells NaN)
template <typename T> void scatter(DistributedDomain &dd, size_t q, const std::vector<T> &g) {
  const Dim3 n = dd.size();
  for (LocalDomain &d : dd.domains()) {
    const Dim3 rs = d.raw_size(), sz = d.size(), o = d.origin();
    std::vector<T> a(size_t(rs.x * rs.y * rs.z), T(NAN));
    for (int64_t z = 0; z < sz.z; ++z)
      for (int64_t y = 0; y < sz.y; ++y)
        for (int64_t x = 0; x < sz.x; ++x) a[size_t(((z + 1) * rs.y + y + 1) * rs.x + x + 1)] = g[size_t(((o.z + z) * n.y + o.y + y) * n.x + o.x + x)];
    d.set_device();
    CUDA_RUNTIME(cudaMemcpy(d.curr_data(q).ptr, a.data(), a.size() * sizeof(T), cudaMemcpyHostToDevice));
  }
  for (LocalDomain &d : dd.domains()) {
    d.set_device();
    CUDA_RUNTIME(cudaDeviceSynchronize());
  }
}

// the reverse: the global interior of quantity q, the same on every rank (collective)
template <typename T> std::vector<T> gather(DistributedDomain &dd, size_t q) {
  const Dim3 n = dd.size();
  std::vector<T> out(size_t(n.x * n.y * n.z), T(0));
  for (LocalDomain &d : dd.domains()) {
    const Dim3 rs = d.raw_size(), sz = d.size(), o = d.origin();
    std::vector<T> a(size_t(rs.x * rs.y * rs.z));
    d.set_device();
    CUDA_RUNTIME(cudaDeviceSynchronize());
    CUDA_RUNTIME(cudaMemcpy(a.data(), d.curr_data(q).ptr, a.size() * sizeof(T), cudaMemcpyDeviceToHost));
    for (int64_t z = 0; z < sz.z; ++z)
      for (int64_t y = 0; y < sz.y; ++y)
        for (int64_t x = 0; x < sz.x; ++x) out[size_t(((o.z + z) * n.y + o.y + y) * n.x + o.x + x)] = a[size_t(((z + 1) * rs.y + y + 1) * rs.x + x + 1)];
  }
  if (mpi::world_size() > 1) { // disjoint cells: a sum of zero-initialised 8-byte words merges them
    std::vector<T> all(out.size());
    MPI_Allreduce(out.data(), all.data(), int(out.size() * sizeof(T) / 8), MPI_LONG_LONG, MPI_SUM, MPI_COMM_WORLD);
    out.swap(all);
  }
  return out;
}

template <typename T> std::vector<T> read_array(const std::string &path, size_t count) {
  std::vector<T> v(count);
  std::ifstream in(path, std::ios::binary);
  if (!in.read(reinterpret_cast<char *>(v.data()), std::streamsize(count * sizeof(T)))) LOG_FATAL("cannot read " << count << " values from " << path);
  return v;
}

// one case on one partition: the quantities by name, the results written by rank 0
template <typename T> class Run {
public:
  Run(const Case &c, const std::vector<int> &gpus, const std::string &out) : c_(c), gpus_(gpus), out_(out + "/" + c.name) {
    if (0 == mpi::world_rank()) mkdir(out_.c_str(), 0755);
  }

  void go() {
    static const std::map<std::string, std::vector<std::string>> kNames = {{"mg", {"u", "f", "r", "u2", "f2"}},
                                                                           {"pcg", {"x", "f", "r", "z", "p", "q"}},
                                                                           {"bicgstab", {"x", "f", "r", "r0", "p", "v", "phat", "shat", "t"}},
                                                                           {"passes", {"u", "f", "r"}}};
    auto it = kNames.find(c_.solver);
    if (it == kNames.end()) LOG_FATAL(c_.name << ": unknown solver " << c_.solver);
    dd_.reset(domain(c_.size[0], c_.size[1], c_.size[2], it->second, true));
    if (c_.solver == "mg")
      multigrid();
    else if (c_.solver == "passes")
      passes();
    else
      krylov();
    std::ofstream f(out_ + "/info.txt");
    f << info_.str();
  }

private:
  const Case &c_;
  std::vector<int> gpus_;
  std::string out_;
  std::unique_ptr<DistributedDomain> dd_;
  std::map<std::string, DataHandle<T>> q_;  // the fine domain's quantities
  std::map<std::string, DataHandle<T>> cq_; // the coarse domain's (passes)
  std::vector<DataHandle<T>> k_;
  std::ostringstream info_;

  // a realized domain of the named quantities (and, on the fine one, the coefficient fields) with the case's BCs
  DistributedDomain *domain(int64_t nx, int64_t ny, int64_t nz, const std::vector<std::string> &names, bool fine) {
    DistributedDomain *dd = new DistributedDomain(nx, ny, nz);
    dd->set_gpus(gpus_);
    dd->set_radius(Radius::constant(1));
    std::map<std::string, DataHandle<T>> &qs = fine ? q_ : cq_;
    for (const std::string &n : names) qs.emplace(n, dd->add_data<T>(n));
    if (fine)
      for (size_t i = 0; i < c_.kinds.size(); ++i) {
        k_.push_back(dd->add_data<T>("k" + std::to_string(i)));
        qs.emplace("k" + std::to_string(i), k_.back());
      }
    dd->set_boundary(c_.periodic ? Topology::Boundary::PERIODIC : Topology::Boundary::FIXED);
    for (const Case::Wall &w : c_.bcs) {
      auto q = qs.find(w.q);
      if (q != qs.end()) dd->set_boundary_condition(q->second, face_dir(w.face), w.bc);
    }
    dd->realize();
    return dd;
  }

  size_t cells(const DistributedDomain &dd) const { return size_t(dd.size().x * dd.size().y * dd.size().z); }
  void load(DistributedDomain &dd, DataHandle<T> h, const std::string &file) { scatter<T>(dd, h.id(), read_array<T>(c_.dir + "/" + file, cells(dd))); }
  void load_inputs() {
    for (const std::string &n : c_.inputs) load(*dd_, q_.at(n), n + ".bin");
  }
  void write(DistributedDomain &dd, DataHandle<T> h, const std::string &name) {
    const std::vector<T> v = gather<T>(dd, h.id());
    if (0 != mpi::world_rank()) return;
    std::ofstream f(out_ + "/" + name + ".bin", std::ios::binary);
    f.write(reinterpret_cast<const char *>(v.data()), std::streamsize(v.size() * sizeof(T)));
  }
  void hist(const std::string &key, const std::vector<double> &h) {
    info_ << key;
    char buf[64];
    for (double v : h) {
      std::snprintf(buf, sizeof(buf), " %a", v);
      info_ << buf;
    }
    info_ << "\n";
  }
  std::function<LinearStencil(int)> op_at() const {
    const Case *c = &c_;
    return [c](int l) { return op_of(*c, l); };
  }

  void multigrid() {
    DataHandle<T> u = q_.at("u"), f = q_.at("f"), r = q_.at("r");
    load_inputs();
    stencil::Multigrid<T> mg(*dd_, u, f, r, op_at(), k_, c_.kinds, c_.nu1, c_.nu2, c_.coarse, c_.levels);
    info_ << "levels " << mg.num_levels() << "\ncolours " << mg.colours() << "\n";
    for (int k = 1; k <= c_.iters; ++k) {
      mg.cycle();
      write(*dd_, u, "cycle" + std::to_string(k));
    }
    if (!k_.empty()) {
      for (size_t i = 0; i < k_.size(); ++i) load(*dd_, k_[i], "ks" + std::to_string(i) + ".bin");
      mg.update_coefficients();
      mg.cycle();
      write(*dd_, u, "update");
    }
    DataHandle<T> u2 = q_.at("u2"), f2 = q_.at("f2");
    load(*dd_, u2, "u2.bin");
    load(*dd_, f2, "f2.bin");
    mg.cycle(u2, f2);
    write(*dd_, u2, "pair");
  }

  template <typename S> void solves(S &s) {
    DataHandle<T> x = q_.at("x");
    for (int k = 1; k <= c_.iters; ++k) {
      load_inputs();
      hist("hist" + std::to_string(k), s.solve(0.0, k));
      info_ << "breakdown" << k << " " << s.breakdown() << "\n";
      write(*dd_, x, "x" + std::to_string(k));
    }
    dd_->swap();
    load_inputs();
    hist("hist_swap", s.solve(0.0, c_.iters));
    info_ << "breakdown_swap " << s.breakdown() << "\n";
    write(*dd_, x, "swap");
  }

  void krylov() {
    auto Q = [this](const char *n) { return q_.at(n); };
    load_inputs(); // the preconditioner coarsens the coefficient fields when it is built
    if (c_.solver == "pcg") {
      stencil::PCG<T> s(*dd_, Q("x"), Q("f"), Q("r"), Q("z"), Q("p"), Q("q"), op_at(), k_, c_.kinds, c_.precond, c_.nu1, c_.nu2, c_.coarse, c_.levels);
      if (s.preconditioner()) info_ << "levels " << s.preconditioner()->num_levels() << "\ncolours " << s.preconditioner()->colours() << "\n";
      solves(s);
    } else {
      stencil::BiCGStab<T> s(*dd_, Q("x"), Q("f"), Q("r"), Q("r0"), Q("p"), Q("v"), Q("phat"), Q("shat"), Q("t"), op_at(), k_, c_.kinds, c_.nu1, c_.nu2,
                             c_.coarse, c_.levels);
      info_ << "levels " << s.preconditioner()->num_levels() << "\ncolours " << s.preconditioner()->colours() << "\n";
      solves(s);
    }
  }

  // single passes of the transfers and sweeps the cycle is made of, so a disagreement of a solver can be located
  void passes() {
    DistributedDomain &dd = *dd_;
    std::unique_ptr<DistributedDomain> cd(domain(c_.size[0] / 2, c_.size[1] / 2, c_.size[2] / 2, {"w", "cu"}, false));
    DataHandle<T> u = q_.at("u"), f = q_.at("f"), r = q_.at("r"), w = cq_.at("w"), cu = cq_.at("cu");
    const LinearStencil A = op_of(c_, 0);
    load_inputs();
    dd.apply(A, curr(r), u, k_);
    write(dd, r, "apply");
    for (int c = 0; c < 2; ++c) {
      dd.relax(A, curr(u), u, curr(f), k_, stencil::Colour{2, c}, 1.0);
      write(dd, u, "relax" + std::to_string(c));
    }
    LinearStencil res;
    res.add(Source::aux, 0, 0, 0, 1.0);
    for (const sb_stencil_vterm &t : A.vterms())
      res.add(Source::src, t.offset[0], t.offset[1], t.offset[2], -t.weight, t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2]);
    dd.restrict_to(*cd, curr(w), res, u, curr(f), k_);
    write(*cd, w, "restrict");
    for (int a = 0; a < 3; ++a) {
      dd.restrict_to(*cd, curr(w), curr(k_[size_t(a)]), a);
      write(*cd, w, "face" + std::to_string(a));
    }
    load(*cd, cu, "cu.bin");
    dd.prolong_from(*cd, curr(u), curr(cu), curr(u));
    write(dd, u, "prolong");
  }
};

int main(int argc, char **argv) {
  MPI_Init(&argc, &argv);
  const bool single = argc >= 4 && std::string(argv[1]) == "--single";
  if (!(single && argc >= 5) && !(argc >= 4 && std::string(argv[1]) == "--ranks")) {
    std::fprintf(stderr, "usage: %s --single N OUT CASE... | --ranks OUT CASE...\n", argv[0]);
    MPI_Finalize();
    return 2;
  }
  int ndev = 0;
  CUDA_RUNTIME(cudaGetDeviceCount(&ndev));
  const std::vector<int> gpus = single ? std::vector<int>(size_t(std::atoi(argv[2])), 0) : std::vector<int>{mpi::world_rank() % ndev};
  const std::string out = argv[single ? 3 : 2];
  if (0 == mpi::world_rank()) mkdir(out.c_str(), 0755);
  int ncase = 0;
  for (int i = single ? 4 : 3; i < argc; ++i, ++ncase) {
    const Case c = parse(argv[i]);
    if (c.dtype == "f64")
      Run<double>(c, gpus, out).go();
    else if (c.dtype == "f32")
      Run<float>(c, gpus, out).go();
    else
      LOG_FATAL(c.name << ": dtype must be f32 or f64, not " << c.dtype);
  }
  if (0 == mpi::world_rank())
    std::printf("test_solver_parity: %d case(s), %zu subdomain(s) on %d rank(s) done\n", ncase, single ? gpus.size() : size_t(mpi::world_size()),
                mpi::world_size());
  MPI_Finalize();
  return 0;
}
