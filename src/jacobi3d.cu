// stencil::FusedJacobi3d (include/stencil/jacobi3d.hpp): the jacobi3d iteration of bin/jacobi3d.cu:296-368 over this
// library's kernels, for C++ users.  Host logic only; the kernels live behind the C ABI (stencil_b200.h).
#include "stencil/jacobi3d.hpp"

#include "stencil_b200.h"

namespace stencil {

namespace {
sb_pitched as_sb(const cudaPitchedPtr &p) { return sb_pitched{p.ptr, int64_t(p.pitch), int64_t(p.ysize)}; }
void set3(int64_t out[3], const Dim3 &d) {
  out[0] = d.x;
  out[1] = d.y;
  out[2] = d.z;
}
const Dim3 kFaces[6] = {Dim3(-1, 0, 0), Dim3(1, 0, 0), Dim3(0, -1, 0), Dim3(0, 1, 0), Dim3(0, 0, -1), Dim3(0, 0, 1)};
} // namespace

struct FusedJacobi3d::Call {
  sb_pitched dst, src;
  int64_t acc[3], lo[3], hi[3], clo[3], chi[3];
  int64_t ilo[3], ihi[3];          // interior box (reference schedule)
  std::vector<int64_t> elo, ehi;   // exterior slabs (reference schedule)
  sb_halo_push push;
};

FusedJacobi3d::FusedJacobi3d(DistributedDomain &dd, size_t quantity, size_t elemSize, bool allowFused)
    : dd_(dd), q_(quantity), es_(elemSize), fused_(allowFused), ghostsCurrent_(false), parity_(0), calls_(new std::vector<Call>()) {
  if (4 != es_ && 8 != es_) LOG_FATAL("FusedJacobi3d: float or double quantities only");
  std::vector<LocalDomain> &doms = dd_.domains();
  if (doms.empty()) LOG_FATAL("FusedJacobi3d: call DistributedDomain::realize() first");
  const Radius &r = doms[0].radius();
  for (const Dim3 &f : kFaces)
    if (1 != r.dir(f)) fused_ = false;
  for (const LocalDomain &d : doms) // the fused kernel wants >= 16 cells along x and neighbours of its own extent
    if (d.size().x < 16 || !(d.size() == doms[0].size())) fused_ = false;
  if (dd_.has_boundary_conditions()) fused_ = false; // the wall ghost cells are filled by exchange(), which the fused kernel replaces

  Placement *pl = dd_.get_placement();
  const Topology &topo = dd_.get_topology();
  // neighbours owned by another rank: the exchange() of the reference schedule reaches them (CUDA-IPC direct writes +
  // device-side flags); the fused kernel's in-kernel handshake across ranks is wired up in the Python layer only
  for (size_t di = 0; fused_ && di < doms.size(); ++di)
    for (const Dim3 &f : kFaces) {
      const Topology::OptionalNeighbor nb = topo.get_neighbor(dd_.domain_index(di), f);
      if (nb.exists && pl->get_rank(nb.index) != dd_.rank()) fused_ = false;
    }
  const Rect3 whole = dd_.get_compute_region();
  const std::vector<Rect3> interiors = dd_.get_interior();
  const std::vector<std::vector<Rect3>> exteriors = dd_.get_exterior();
  nbrs_.assign(doms.size(), {});
  for (size_t di = 0; di < doms.size(); ++di) {
    streams_.push_back(RcStream(doms[di].gpu()));
    cudaEvent_t ev;
    CUDA_RUNTIME(cudaSetDevice(doms[di].gpu()));
    CUDA_RUNTIME(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    done_.push_back(ev);
  }
  for (int rel = 0; rel < 2; ++rel) {
    for (size_t di = 0; di < doms.size(); ++di) {
      const LocalDomain &d = doms[di];
      Call c{};
      const cudaPitchedPtr cur = d.curr_data(q_), nxt = d.next_data(q_);
      c.src = as_sb(0 == rel ? cur : nxt);
      c.dst = as_sb(0 == rel ? nxt : cur);
      set3(c.acc, d.get_full_region().lo);
      const Rect3 reg = d.get_compute_region();
      set3(c.lo, reg.lo);
      set3(c.hi, reg.hi);
      set3(c.clo, whole.lo);
      set3(c.chi, whole.hi);
      set3(c.ilo, interiors[di].lo);
      set3(c.ihi, interiors[di].hi);
      for (const Rect3 &e : exteriors[di]) {
        for (int64_t v : {e.lo.x, e.lo.y, e.lo.z}) c.elo.push_back(v);
        for (int64_t v : {e.hi.x, e.hi.y, e.hi.z}) c.ehi.push_back(v);
      }
      if (fused_) {
        const Dim3 idx = pl->get_idx(mpi::world_rank(), int(di));
        for (int k = 0; k < 6; ++k) {
          const Topology::OptionalNeighbor nb = topo.get_neighbor(idx, kFaces[k]);
          if (!nb.exists) continue; // non-periodic boundary: nothing to push
          const size_t dj = size_t(pl->get_subdomain_id(nb.index));
          const LocalDomain &n = doms[dj];
          // the neighbour's OUTPUT buffer of this iteration
          c.push.nbr[k] = as_sb(0 == rel ? n.next_data(q_) : n.curr_data(q_));
          c.push.nbr_zsize[k] = n.raw_size().z;
          if (0 == rel && dj != di && std::find(nbrs_[di].begin(), nbrs_[di].end(), dj) == nbrs_[di].end()) nbrs_[di].push_back(dj);
        }
      }
      calls_->push_back(c);
    }
  }
}

FusedJacobi3d::~FusedJacobi3d() {
  synchronize();
  for (size_t di = 0; di < done_.size(); ++di) {
    cudaSetDevice(dd_.domains()[di].gpu());
    cudaEventDestroy(done_[di]);
  }
  delete calls_;
}

void FusedJacobi3d::init(double value) {
  std::vector<LocalDomain> &doms = dd_.domains();
  for (size_t di = 0; di < doms.size(); ++di) {
    const Call &c = (*calls_)[size_t(parity_) * doms.size() + di];
    if (SB_OK != sb_fill(c.src, int(es_), c.acc, c.lo, c.hi, value, streams_[di])) LOG_FATAL("FusedJacobi3d::init: " << sb_last_error());
  }
  synchronize();
  ghostsCurrent_ = false;
}

double FusedJacobi3d::residual() { return dd_.reduce_many(std::vector<ReduceItem>(1, ReduceItem{SB_REDUCE_DIFF, {q_, q_, q_}, Which::curr}))[0].l2(); }

void FusedJacobi3d::synchronize() {
  for (size_t di = 0; di < streams_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(streams_[di].device()));
    CUDA_RUNTIME(cudaStreamSynchronize(streams_[di]));
  }
}

void FusedJacobi3d::step_reference_schedule() {
  std::vector<LocalDomain> &doms = dd_.domains();
  const size_t n = doms.size();
  for (size_t di = 0; di < n; ++di) {
    const Call &c = (*calls_)[size_t(parity_) * n + di];
    CUDA_RUNTIME(cudaSetDevice(doms[di].gpu()));
    if (SB_OK != sb_jacobi3d(c.dst, c.src, int(es_), c.acc, c.ilo, c.ihi, c.clo, c.chi, streams_[di])) LOG_FATAL("sb_jacobi3d: " << sb_last_error());
  }
  dd_.exchange();
  for (size_t di = 0; di < n; ++di) {
    const Call &c = (*calls_)[size_t(parity_) * n + di];
    CUDA_RUNTIME(cudaSetDevice(doms[di].gpu()));
    if (SB_OK != sb_jacobi3d_regions(c.dst, c.src, int(es_), c.acc, int(c.elo.size() / 3), c.elo.data(), c.ehi.data(), c.clo, c.chi, streams_[di]))
      LOG_FATAL("sb_jacobi3d_regions: " << sb_last_error());
  }
  synchronize();
}

void FusedJacobi3d::step() {
  std::vector<LocalDomain> &doms = dd_.domains();
  const size_t n = doms.size();
  if (!fused_) {
    step_reference_schedule();
  } else {
    if (!ghostsCurrent_) { // ghost cells of curr, once; afterwards every iteration leaves them filled for the next
      synchronize();
      dd_.exchange();
      ghostsCurrent_ = true;
    } else {
      for (size_t di = 0; di < n; ++di) {
        CUDA_RUNTIME(cudaSetDevice(doms[di].gpu()));
        for (size_t dj : nbrs_[di]) CUDA_RUNTIME(cudaStreamWaitEvent(streams_[di], done_[dj], 0));
      }
    }
    for (size_t di = 0; di < n; ++di) {
      const Call &c = (*calls_)[size_t(parity_) * n + di];
      CUDA_RUNTIME(cudaSetDevice(doms[di].gpu()));
      if (SB_OK != sb_jacobi3d_fused(c.dst, c.src, int(es_), c.acc, c.lo, c.hi, c.clo, c.chi, &c.push, streams_[di]))
        LOG_FATAL("sb_jacobi3d_fused: " << sb_last_error());
    }
    for (size_t di = 0; di < n; ++di) {
      CUDA_RUNTIME(cudaSetDevice(doms[di].gpu()));
      CUDA_RUNTIME(cudaEventRecord(done_[di], streams_[di]));
    }
  }
  dd_.swap();
  parity_ ^= 1;
}

} // namespace stencil
