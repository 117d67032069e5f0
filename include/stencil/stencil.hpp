#pragma once
// DistributedDomain: a periodic 3-D grid cut into one subdomain per GPU, with a halo exchange between
// the 26 neighbours of every subdomain.  Public API of the reference's include/stencil/stencil.hpp;
// the implementation (src/stencil.cu) is H100-native: realize() plans, for every local subdomain,
// ONE fused kernel that reads the outgoing halo regions of all quantities and stores them directly
// into the ghost cells of the destination subdomains -- on the same GPU, or on a peer GPU through
// NVLink/NVSwitch peer mappings -- with no send or receive buffers.

#include <algorithm>
#include <cassert>
#include <cstdlib>
#include <fstream>
#include <functional>
#include <map>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include <mpi.h>

#include <nvToolsExt.h>
#include <nvml.h>

#include "stencil/cuda_runtime.hpp"

#include "stencil/boundary_condition.hpp"
#include "stencil/dim3.hpp"
#include "stencil/direction_map.hpp"
#include "stencil/gpu_topology.hpp"
#include "stencil/linear_stencil.hpp"
#include "stencil/local_domain.cuh"
#include "stencil/logging.hpp"
#include "stencil/machine.hpp"
#include "stencil/method.hpp"
#include "stencil/mpi_topology.hpp"
#include "stencil/nvml.hpp"
#include "stencil/partition.hpp"
#include "stencil/pitched_ptr.hpp"
#include "stencil/placement_intranoderandom.hpp"
#include "stencil/radius.hpp"
#include "stencil/rcstream.hpp"
#include "stencil/reduce.hpp"
#include "stencil/topology.hpp"
#include "stencil/tx.hpp"

struct sb_copy_plan;
struct sb_bc_plan;
struct sb_reduce_plan;
struct sb_reduce_exact_plan;
struct sb_krylov_plan;
struct sb_stencil_plan;
struct sb_transfer_plan;

namespace stencil {
template <typename T> class Multigrid;
namespace detail {
template <typename T> class KrylovSolver;
}
}

class DistributedDomain {
  template <typename T> friend class stencil::Multigrid;
  template <typename T> friend class stencil::detail::KrylovSolver;

private:
  Dim3 size_; // compute extent of the whole grid

  int rank_;
  int worldSize_;

  std::vector<int> gpus_; // CUDA devices this rank drives, one subdomain each

  MpiTopology mpiTopology_;
  Placement *placement_;
  Topology topology_;
  Radius radius_;

  std::vector<LocalDomain> domains_;
  std::vector<Dim3> domainIdx_;

  std::vector<size_t> dataElemSize_;
  std::vector<std::string> dataName_;

  Method flags_;
  PlacementStrategy strategy_;
  Topology::Boundary boundary_[3]; // per axis: PERIODIC (the reference's only kind) or FIXED

  // boundary conditions on the wall faces: (quantity, face 0..5 = -x,+x,-y,+y,-z,+z) -> BC, and each quantity's sb_dtype
  std::map<std::pair<size_t, int>, stencil::BC> bcs_;
  std::vector<int> dataDtype_;
  // after the exchange: bcPlans_[parity][local domain] (nullptr where the subdomain has no BC to apply), launched on the
  // subdomain's exchange stream after its phase 2 and after the phase 1 of bcSenders_[domain] (local subdomains)
  std::vector<sb_bc_plan *> bcPlans_[2];
  std::vector<std::vector<size_t>> bcSenders_;
  void plan_boundaries(std::ofstream &planFile);

  // the fused exchange: plans_[parity][local domain]; parity = number of swap() calls mod 2.
  // Phase 1 (plans_): each subdomain stores its outgoing halos into the neighbours' ghost cells -- except
  // thin rows bound for ANOTHER GPU (x-faces, x-edges, corners), which are packed into a dense staging
  // buffer in the neighbour's memory (one tiny NVLink transaction per 8-byte row is what kills both the
  // exchange and the concurrently running compute kernel).  Phase 2 (unpackPlans_): each receiver
  // scatters its staging buffers into its ghost cells.
  std::vector<sb_copy_plan *> plans_[2];
  std::vector<sb_copy_plan *> unpackPlans_[2];       // nullptr where a subdomain receives nothing staged
  std::vector<std::vector<size_t>> stageSenders_;    // per receiver: local domains that stage into it
  std::vector<void *> stagingBufs_;                  // device allocations (on the receivers' GPUs)
  std::vector<int> stagingDevs_;
  std::vector<cudaEvent_t> phase1Done_;              // one per local domain
  // exchanges of a quantity subset (DESIGN.md section 2.15): the full plans' box copies, BC quantities and phase-2 copies
  // per [parity][local domain], each copy with its quantity, from which a subset's plans are cut on its first use and
  // kept per (parity, set); agreedSets_: the sets every rank has been checked to pass alike
  struct TaggedCopy {
    size_t q;
    sb_box_copy c;
  };
  std::vector<std::vector<TaggedCopy>> fullCopies_[2], fullScatter_[2];
  std::vector<std::vector<sb_bc_quantity>> bcQuantities_[2];
  struct SubsetPlans {
    std::vector<sb_copy_plan *> copy, scatter;
    std::vector<sb_bc_plan *> bc;
  };
  std::map<std::pair<int, uint64_t>, SubsetPlans> subsetPlans_;
  std::set<uint64_t> agreedSets_;
  const SubsetPlans &subset_plans(uint64_t set);
  void exchange_async_set(uint64_t set);
  std::vector<RcStream> streams_; // one high-priority stream per local domain
  int parity_;

  // Other ranks of this node (one process per GPU, started by sb_mpirun / mpirun).  Their allocations, staging buffers
  // and flag mailboxes are mapped once, at realize(), through CUDA IPC handles that travel over MPI (the reference ships
  // them the same way: include/stencil/tx_cuda.cuh:225-315, src/tx_ipc.cpp).  After that the data path is the fused
  // copy kernel storing into the mapped ghost cells; the only cross-rank synchronisation of an exchange is a pair of
  // device-side flags per neighbour rank (ready: "my ghost cells may be overwritten for exchange e"; done: "my writes
  // into you for exchange e have landed"), st.release.sys / ld.acquire.sys by tiny kernels -- no MPI call, no host sync.
  struct RemoteDomain {
    Dim3 raw;
    std::vector<char *> curr, next; // mapped allocations per quantity, in the owner's parity-0 naming
  };
  std::map<Dim3, RemoteDomain> remote_;                       // neighbour subdomains of other ranks
  std::map<std::pair<Dim3, Dim3>, char *> remoteStage_;       // (src idx, dst idx) -> staging buffer in the dst rank
  std::vector<void *> ipcOpened_;
  uint32_t *mailbox_;                // my mailbox: ready[worldSize] then done[worldSize]
  std::vector<uint32_t *> peerFlags_; // per rank: its mailbox (mapped), nullptr for non-neighbours
  std::vector<int> nbrRanks_;
  uint32_t epoch_;
  void share_with_ranks(const std::map<std::pair<Dim3, Dim3>, char *> &myStage);
  void close_ranks();
  void flags_begin();
  void flags_finish();

  // reductions: per (item list, swap parity), one plan and one device result buffer per local domain
  struct ReduceCache {
    std::vector<sb_reduce_plan *> plans; // Sum::ordered
    std::vector<sb_reduce_result *> out;
    std::vector<sb_reduce_exact_plan *> xplans; // Sum::exact
    std::vector<sb_reduce_exact_part *> xout;
  };
  std::map<std::vector<int64_t>, ReduceCache> reducePlans_;
  void destroy_reduce_plans();
  // every rank's byte records (MPI_Allgatherv, in rank order), the gather of reduce(..., Sum::exact) and of the Krylov sums
  std::vector<unsigned char> allgather_records(const std::vector<unsigned char> &mine) const;

  // Krylov vector passes (DESIGN.md section 2.13): per (mode, quantities, swap parity), one sb_krylov_plan over the
  // compute region and one device buffer of its exact parts per local domain
  struct KrylovCache {
    std::vector<sb_krylov_plan *> plans;
    std::vector<sb_reduce_exact_part *> out;
    int nparts = 0;
  };
  std::map<std::vector<int64_t>, KrylovCache> krylovPlans_;
  void destroy_krylov_plans();
  KrylovCache &krylov_plans(int mode, const std::vector<size_t> &qs);
  // one launch per local domain with the scalar s: queued (after the previous exterior, on the interior apply stream) or
  // on the exchange streams after all work queued on the local devices
  void krylov_launch(KrylovCache &c, double s, bool queued) { krylov_launch(c, s, 0.0, queued); }
  // the same with a second scalar t (SB_KRYLOV_BICG_P's omega; the other modes ignore it)
  void krylov_launch(KrylovCache &c, double s, double t, bool queued);
  // the host wait: the parts of the last launch of each cache (on the streams krylov_launch used), gathered from every
  // rank in one MPI_Allgatherv, combined and rounded once; one sum per part, in the order of the caches
  std::vector<double> krylov_sums(const std::vector<KrylovCache *> &cs, bool queued);

  // linear stencil operators: per (op, buffers, exchange, swap parity), per local domain the interior and exterior plans
  // (exchange = true) or the whole-region plan; two streams per local domain (interior, exterior)
  std::map<std::vector<int64_t>, std::vector<std::vector<sb_stencil_plan *>>> stencilPlans_;
  std::vector<cudaStream_t> applyStreams_;
  void destroy_stencil_plans();
  // omega non-NULL: relax()'s diagonal relaxation (sb_stencil_dplan_create), aq the right-hand side f
  void apply_op(const stencil::LinearStencil &op, int dtype, size_t dq, stencil::Which dw, size_t sq, int64_t aq, stencil::Which aw,
                const std::vector<size_t> &cq, stencil::Exchange exchange, stencil::Colour colour = stencil::Colour{}, const double *omega = nullptr);
  void apply_sys(const stencil::LinearSystem &sys, int dtype, const std::vector<std::pair<size_t, stencil::Which>> &outs,
                 const std::vector<std::pair<size_t, stencil::Which>> &ins, stencil::Exchange exchange);
  // the bit set an operator call exchanges (0: none): every quantity for true, `reads` for Exchange::reads() (the full
  // set when it names every quantity), the given set for Exchange::only
  uint64_t exchange_set(const char *name, const stencil::Exchange &exchange, uint64_t reads) const;
  // the plans apply_op and apply_sys share: the cached per-domain plans of key (built by make(domain, boxes) on first
  // use), run by queued_schedule: the interior plans while exchange() runs and the exterior plans after it, or the one
  // whole-region plan per domain.  writes_src: the launch writes src (a coloured apply in place), so the interior also
  // keeps clear of the slabs exchange() sends, which are as wide as the radius on the opposite side.
  void run_stencil_plans(const std::vector<int64_t> &key, uint64_t exchange, bool writes_src,
                         const std::function<sb_stencil_plan *(size_t, const std::vector<Rect3> &)> &make);

  // The schedule of every operator call (DESIGN.md section 2.11), ordered by CUDA events only.  Each interior (or
  // whole-region launch) waits for the previous exterior of its subdomain; queue_exchange() makes every exchange stream
  // wait for every local apply stream before exchange_async(), so an exchange neither sends a value still being written
  // nor overwrites a ghost cell an earlier launch still reads (and, across ranks, signals its neighbours only after those
  // waits); wait_exchange(other, interior) makes this domain's exterior (and interior) apply streams wait for other's
  // exchange.  The apply streams are blocking streams, so a call follows the work on the legacy default stream.  A
  // public call ends with one host wait (wait_queued); while queued_ is set (a solver that owns the schedule) it returns
  // at once.
  bool queued_ = false;
  bool sharedApplyStreams_ = false; // applyStreams_ belong to another domain (a solver's finer level)
  std::vector<cudaEvent_t> applyEvents_, exchangeEvents_; // one per apply / exchange stream, recorded again on each use
  void queue_after_exterior();
  // quantity q's whole curr allocation set to +0 (ghost cells included; an exchange refills them before any read), on
  // each interior apply stream after the previous exterior
  void clear_queued(size_t q);
  void queue_exchange(uint64_t quantities = ~uint64_t(0));
  void wait_exchange(DistributedDomain &other, bool interior);
  void ensure_queue_events();
  // the interior / exchange / exterior schedule: launch(domain, part, stream), part 0 the interior (or the whole region
  // without exchange), 1 the exterior; then, unless queued_, wait_queued({this})
  void queued_schedule(const std::function<void(size_t, int, cudaStream_t)> &launch, uint64_t exchange);
  // returns when the work queued on the apply and exchange streams of every domain in doms is complete: the end of a
  // public operator call, of a Multigrid cycle and of a Krylov solve (apply streams several domains share are waited for
  // once)
  static void wait_queued(const std::vector<DistributedDomain *> &doms);

  // multigrid transfers: per (coarse domain, kind, buffers, the swap parity of both domains), one plan per local domain.
  // serial_ names a domain for the lifetime of the process (an address can be reused by a later domain)
  uint64_t serial_;
  std::map<std::vector<int64_t>, std::vector<sb_transfer_plan *>> transferPlans_;
  std::set<std::pair<uint64_t, bool>> paired_; // (coarse serial, with ghosts) that passed the pairing check
  // op: the fused residual-restriction (sb_transfer_oplan_create, or sb_transfer_voplan_create over the fine coefficient
  // quantities cq; restriction only), with apply's schedule when exchange.  face >= 0: the face-coefficient restriction
  // of the faces normal to that axis (sb_transfer_fplan_create).
  void transfer(DistributedDomain &coarse, bool prolong, int dtype, size_t dq, stencil::Which dw, size_t sq, stencil::Which sw, int64_t aq,
                stencil::Which aw, stencil::Exchange exchange, const stencil::LinearStencil *op = nullptr, const std::vector<size_t> &cq = {},
                int face = -1);
  void check_pairing(DistributedDomain &coarse, bool ghosts);
  void destroy_transfer_plans();
  void create_apply_streams(); // two per local domain (interior, exterior), on first use

  std::string outputPrefix_;

  // payload bytes per exchange, attributed the way the reference's planner attributes them
  uint64_t numBytesCudaMpi_;
  uint64_t numBytesColoDirectAccess_;
  uint64_t numBytesColoPackMemcpyUnpack_;
  uint64_t numBytesCudaMemcpyPeer_;
  uint64_t numBytesCudaKernel_;

  void plan_exchange();
  void destroy_plans();

public:
#ifdef STENCIL_EXCHANGE_STATS
  double timeExchange_;
  double timeSwap_;
#endif

#ifdef STENCIL_SETUP_STATS
  double timeMpiTopo_;
  double timeNodeGpus_;
  double timePeerEn_;
  double timePlacement_;
  double timePlan_;
  double timeRealize_;
  double timeCreate_;
#endif

  DistributedDomain(size_t x, size_t y, size_t z);
  ~DistributedDomain();
  DistributedDomain(const DistributedDomain &) = delete;
  DistributedDomain &operator=(const DistributedDomain &) = delete;

  const Dim3 &size() const noexcept { return size_; }
  std::vector<LocalDomain> &domains() noexcept { return domains_; }
  const std::vector<LocalDomain> &domains() const noexcept { return domains_; }

  void set_radius(size_t r) noexcept { radius_ = Radius::constant(r); }
  void set_radius(const Radius &r) noexcept { radius_ = r; }

  template <typename T> DataHandle<T> add_data(const std::string &name = "") {
    dataElemSize_.push_back(sizeof(T));
    dataName_.push_back(name);
    dataDtype_.push_back(stencil::bc_dtype<T>());
    return DataHandle<T>(dataElemSize_.size() - 1, name);
  }

  // choose transports (before realize):  d.set_methods(Method::CudaMpi | Method::CudaKernel);
  void set_methods(Method flags) noexcept;
  void set_placement(PlacementStrategy strategy) noexcept { strategy_ = strategy; }
  // how the grid closes at its faces (before realize), for all axes or per axis.  PERIODIC is the reference's behaviour;
  // FIXED plans no messages across the faces of the whole grid along that axis (the ghost cells there keep what the
  // application put into them, unless set_boundary_condition gives them a BC)
  void set_boundary(Topology::Boundary boundary) noexcept { boundary_[0] = boundary_[1] = boundary_[2] = boundary; }
  void set_boundary(Topology::Boundary x, Topology::Boundary y, Topology::Boundary z) noexcept {
    boundary_[0] = x;
    boundary_[1] = y;
    boundary_[2] = z;
  }
  // the BC of quantity h on the wall face `face` ((+-1,0,0), (0,+-1,0) or (0,0,+-1)) of the whole grid (before realize):
  // exchange() fills the ghost cells behind it.  realize() rejects a BC on a periodic axis, VALUE / ODD on a quantity
  // that is not float or double, and EVEN / ODD with a ghost width larger than a subdomain.
  template <typename T> void set_boundary_condition(const DataHandle<T> &h, const Dim3 &face, const stencil::BC &bc) {
    int f = -1;
    for (int a = 0; a < 3; ++a) {
      const int64_t c = a == 0 ? face.x : a == 1 ? face.y : face.z;
      if (c != 0) f = (f == -1 && (c == 1 || c == -1)) ? 2 * a + (c > 0) : -2;
    }
    if (f < 0) LOG_FATAL("set_boundary_condition: " << face << " is not a face direction");
    if (dataDtype_.size() <= h.id() || dataDtype_[h.id()] != stencil::bc_dtype<T>()) LOG_FATAL("set_boundary_condition: unknown data handle");
    bcs_[std::make_pair(h.id(), f)] = bc;
  }
  bool has_boundary_conditions() const noexcept {
    for (const auto &kv : bcs_)
      if (kv.second.kind != stencil::BC::Kind::NONE) return true;
    return false;
  }
  bool any_methods(Method methods) const noexcept { return methods && flags_; }
  // CUDA devices for this rank (before realize); repeats are allowed (several subdomains per GPU)
  void set_gpus(const std::vector<int> &cudaIds) { gpus_ = cudaIds; }
  void set_output_prefix(const std::string &prefix);

  const Dim3 &get_origin(int64_t i) const { return domains_[i].origin(); }
  const Rect3 get_compute_region() const noexcept;

  // total payload bytes per exchange carried by `method` (after realize)
  uint64_t exchange_bytes_for_method(const Method &method) const;

  void do_placement(); // partition + placement only
  void realize();      // allocate, plan
  void swap();         // current <-> next in every local subdomain

  // per local subdomain: the box whose stencil inputs no exchange can touch / the rest as <= 6 slabs
  std::vector<Rect3> get_interior() const;
  std::vector<std::vector<Rect3>> get_exterior() const;

  int rank() const noexcept { return rank_; }
  const Radius &radius() const noexcept { return radius_; }
  const Dim3 &domain_index(size_t i) const { return domainIdx_[i]; }
  const Topology &get_topology() const noexcept { return topology_; }
  Placement *get_placement() const noexcept { return placement_; }

  // halo exchange of the current quantities; returns when all ghost cells of this rank are filled
  void exchange();
  // same, but only enqueues the work: stream(i) of local domain i carries the writes INTO the
  // neighbours; call exchange_wait() (or synchronize all of them) before reading ghost cells
  void exchange_async();
  void exchange_wait();
  // Exchange of a subset of the quantities (DESIGN.md section 2.15): only their boxes are copied and only their walls'
  // BCs filled, through the full exchange's kernels and staging buffers; every byte of the other quantities is left as
  // it was.  A list naming every quantity is the full exchange.  An empty list, a quantity named twice or one that is
  // not a quantity of this domain (or >= 64) is fatal.  The plans of a subset are built on its first use and kept per
  // (swap parity, subset); collective like exchange(): every rank passes the same subset, which the first use of each
  // subset checks with one MPI_Allreduce.
  void exchange(const std::vector<size_t> &quantities);
  void exchange_async(const std::vector<size_t> &quantities);
  // the bit set of a quantity list (fatal on the errors above); every bit set when it names every quantity
  uint64_t quantity_set(const std::vector<size_t> &quantities) const;
  cudaStream_t exchange_stream(size_t domain) const { return streams_[domain]; }

  // Reductions over the whole compute region (DESIGN.md section 2.6), the same bits on every rank.  Each call waits for
  // all work queued on the local devices, launches one plan per local subdomain on its exchange stream, gathers every
  // rank's per-subdomain results with MPI_Allgather and merges them with sb_reduce_combine in global subdomain-index order
  // (x fastest).  Collective: every rank must call it with the same items.  The plans (tile tables, scratch, result
  // buffer) are built once per item list and swap parity and kept until the domain is destroyed, so a program should
  // reduce a fixed set of item lists rather than build new ones every iteration.
  // With stencil::Sum::exact the per-subdomain exact parts are gathered with MPI_Allgatherv, combined with
  // sb_reduce_exact_combine and rounded once with sb_reduce_exact_round on every rank: sum and sumsq are correctly rounded
  // and the same bits for every partition and rank count.  Plans are cached per item list, exactness and swap parity.
  template <typename T> stencil::Reduction reduce(const DataHandle<T> &h, stencil::Which which = stencil::Which::curr) {
    return reduce_many(std::vector<stencil::ReduceItem>(1, stencil::ReduceItem::scalar(h, which)))[0];
  }
  template <typename T> stencil::Reduction reduce(const DataHandle<T> &h, stencil::Which which, stencil::Sum sum) {
    return reduce_many(std::vector<stencil::ReduceItem>(1, stencil::ReduceItem::scalar(h, which)), sum)[0];
  }
  template <typename T> stencil::Reduction reduce_diff(const DataHandle<T> &h) { return reduce_many(std::vector<stencil::ReduceItem>(1, stencil::ReduceItem::diff(h)))[0]; }
  template <typename T> stencil::Reduction reduce_diff(const DataHandle<T> &h, stencil::Sum sum) {
    return reduce_many(std::vector<stencil::ReduceItem>(1, stencil::ReduceItem::diff(h)), sum)[0];
  }
  template <typename T> stencil::Reduction reduce_norm(const DataHandle<T> &x, const DataHandle<T> &y, const DataHandle<T> &z) {
    return reduce_many(std::vector<stencil::ReduceItem>(1, stencil::ReduceItem::norm(x, y, z)))[0];
  }
  template <typename T>
  stencil::Reduction reduce_norm(const DataHandle<T> &x, const DataHandle<T> &y, const DataHandle<T> &z, stencil::Sum sum) {
    return reduce_many(std::vector<stencil::ReduceItem>(1, stencil::ReduceItem::norm(x, y, z)), sum)[0];
  }
  std::vector<stencil::Reduction> reduce_many(const std::vector<stencil::ReduceItem> &items) { return reduce_many(items, stencil::Sum::ordered); }
  std::vector<stencil::Reduction> reduce_many(const std::vector<stencil::ReduceItem> &items, stencil::Sum sum);
  // The exact inner product <a, b> of the curr buffers of two float or double quantities over the whole compute region
  // (DESIGN.md section 2.13): the exact sum over the cells of fl64(double(a) * double(b)), rounded once, so the bits do
  // not depend on the partition or the rank count (a may be b).  Like reduce(..., Sum::exact): waits for all work queued
  // on the local devices, runs on the exchange streams, gathers the parts with MPI_Allgatherv; collective.  Plans are
  // cached per pair and swap parity.
  template <typename T> double dot(const DataHandle<T> &a, const DataHandle<T> &b) {
    KrylovCache &c = krylov_plans(SB_KRYLOV_DOT, {a.id(), b.id()});
    krylov_launch(c, 0.0, false);
    return krylov_sums({&c}, false)[0];
  }

  // dst = op(src, aux) over the whole compute region of every local subdomain (DESIGN.md section 2.7).  src is the curr
  // buffer (the one exchange() fills); dst is curr or next of any quantity of the same type, never src itself; aux is curr
  // or next and may be dst.  Fails loudly unless realize() has run and sb_stencil_check accepts the op for this domain's
  // radius.  exchange = true: the interior runs on its own stream while exchange() fills the ghost cells, then one launch
  // per subdomain covers its exterior slabs; exchange = false: one launch over the whole region, the caller guarantees the
  // ghost cells are current.  The launches and the exchange follow the work on the legacy default stream, and the call
  // returns when the update is complete.  The plans are kept, per (op, buffers, exchange, swap parity), until the domain
  // is destroyed.
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), -1, stencil::Which::curr, {}, exchange);
  }
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, const stencil::Buffer<T> &aux,
             stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), int64_t(aux.h.id()), aux.which, {}, exchange);
  }
  // The same with coefficient fields: coefs[k] is field k of the op (op.ncoef() of them), read from its curr buffer, which
  // exchange() fills like src's (with the quantity's own BC on a wall); a coefficient may alias src or aux, never dst.
  // swap() turns every quantity's buffers, coefficients included: a static coefficient holds the same compute cells in
  // curr and next.
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, const std::vector<DataHandle<T>> &coefs,
             stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), -1, stencil::Which::curr, ids_of(coefs), exchange);
  }
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, const stencil::Buffer<T> &aux,
             const std::vector<DataHandle<T>> &coefs, stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), int64_t(aux.h.id()), aux.which, ids_of(coefs), exchange);
  }
  // Coloured applies (DESIGN.md section 2.9): only the cells of colour colour.c of the colouring colour.m are written,
  // each from the buffers as they were before the call; with m > 1 dst may be src (curr(src)), and every src term with a
  // non-zero offset must read another colour (sb_stencil_ccheck).  A Gauss-Seidel / SOR sweep is one call per colour:
  //     for (int c = 0; c < 2; ++c) dd.apply(sor, stencil::curr(u), u, stencil::curr(f), stencil::Colour{2, c});
  // Schedule, plan cache (with the colouring in its key) and failure rules are the uncoloured apply's.
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, stencil::Colour colour,
             stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), -1, stencil::Which::curr, {}, exchange, colour);
  }
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, const stencil::Buffer<T> &aux,
             stencil::Colour colour, stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), int64_t(aux.h.id()), aux.which, {}, exchange, colour);
  }
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, const std::vector<DataHandle<T>> &coefs,
             stencil::Colour colour, stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), -1, stencil::Which::curr, ids_of(coefs), exchange, colour);
  }
  template <typename T>
  void apply(const stencil::LinearStencil &op, const stencil::Buffer<T> &dst, const DataHandle<T> &src, const stencil::Buffer<T> &aux,
             const std::vector<DataHandle<T>> &coefs, stencil::Colour colour, stencil::Exchange exchange = true) {
    apply_op(op, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), int64_t(aux.h.id()), aux.which, ids_of(coefs), exchange, colour);
  }
  // One relaxation pass of A u = f that divides by A's own diagonal (DESIGN.md section 2.12, sb_stencil_dplan_create):
  // dst = u + omega (f - A u) / d, d the sum of the factors of A's offset-0 terms, on the cells of the colour (none: every
  // cell, weighted Jacobi, dst must not be u).  A has src terms only (plain or coefficient) and a term at offset 0; f is a
  // buffer of A's type; coefs as apply's.  Schedule, plan cache (omega in its key) and failure rules are apply's.
  //     for (int c = 0; c < 2; ++c) dd.relax(A, stencil::curr(u), u, stencil::curr(f), {kx, ky, kz}, stencil::Colour{2, c});
  template <typename T>
  void relax(const stencil::LinearStencil &A, const stencil::Buffer<T> &dst, const DataHandle<T> &u, const stencil::Buffer<T> &f,
             const std::vector<DataHandle<T>> &coefs, stencil::Colour colour, double omega = 1.0, stencil::Exchange exchange = true) {
    apply_op(A, stencil::bc_dtype<T>(), dst.h.id(), dst.which, u.id(), int64_t(f.h.id()), f.which, ids_of(coefs), exchange, colour, &omega);
  }
  template <typename T>
  void relax(const stencil::LinearStencil &A, const stencil::Buffer<T> &dst, const DataHandle<T> &u, const stencil::Buffer<T> &f,
             const std::vector<DataHandle<T>> &coefs, double omega = 1.0, stencil::Exchange exchange = true) {
    apply_op(A, stencil::bc_dtype<T>(), dst.h.id(), dst.which, u.id(), int64_t(f.h.id()), f.which, ids_of(coefs), exchange, stencil::Colour{}, &omega);
  }
  template <typename T>
  void relax(const stencil::LinearStencil &A, const stencil::Buffer<T> &dst, const DataHandle<T> &u, const stencil::Buffer<T> &f,
             stencil::Colour colour, double omega = 1.0, stencil::Exchange exchange = true) {
    apply_op(A, stencil::bc_dtype<T>(), dst.h.id(), dst.which, u.id(), int64_t(f.h.id()), f.which, {}, exchange, colour, &omega);
  }

  // outputs = sys(inputs) over the whole compute region of every local subdomain (DESIGN.md section 2.8): sys.nout()
  // outputs and sys.nin() inputs, each the curr or next buffer of a quantity of the system's type.  An input read at a
  // non-zero offset must be a curr buffer (the one exchange() fills); outputs are pairwise distinct; an output may be an
  // input only if every read of that input is at offset 0 (an in-place update).  Schedule, plan cache and failure rules
  // are the operator apply's.
  template <typename T>
  void apply(const stencil::LinearSystem &sys, const std::vector<stencil::Buffer<T>> &outputs, const std::vector<stencil::Buffer<T>> &inputs,
             stencil::Exchange exchange = true) {
    std::vector<std::pair<size_t, stencil::Which>> o, i;
    for (const stencil::Buffer<T> &b : outputs) o.emplace_back(b.h.id(), b.which);
    for (const stencil::Buffer<T> &b : inputs) i.emplace_back(b.h.id(), b.which);
    apply_sys(sys, stencil::bc_dtype<T>(), o, i, exchange);
  }
  template <typename T> static std::vector<size_t> ids_of(const std::vector<DataHandle<T>> &hs) {
    std::vector<size_t> ids;
    for (const DataHandle<T> &h : hs) ids.push_back(h.id());
    return ids;
  }

  // Multigrid transfers (DESIGN.md section 2.10) between this domain and `coarse`, a realized domain twice as coarse on
  // every axis: the same partition dim, every subdomain's origin and size exactly half of this one's, on the same rank and
  // GPU (sb_transfer_check over every subdomain index, checked once per coarse domain), quantities of the same type.
  // restrict_to: dst (a quantity of coarse) = the 8-cell average of src (a quantity of this domain), curr or next, over
  // every coarse compute cell; no ghost cells are read.
  // prolong_from: dst = aux + P src (or P src) over every fine compute cell, P trilinear; dst and aux are quantities of
  // this domain and aux may be dst (the in-place correction u <- u + P e); src is a curr buffer of coarse, whose radius
  // must be >= 1 in all 26 directions.  exchange = true runs coarse.exchange() first (collective), exchange = false
  // leaves the coarse ghost cells to the caller.
  // One launch per local subdomain on the apply streams; the launches and any exchange follow the work on the legacy
  // default stream, and the call returns when they are complete.  Plans are kept, per (coarse domain, kind, buffers,
  // swap parity of both domains), until this domain is destroyed.
  //     fine.restrict_to(coarse, stencil::curr(f2), stencil::curr(r));
  //     fine.prolong_from(coarse, stencil::curr(u), stencil::curr(e), stencil::curr(u));
  template <typename T> void restrict_to(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::Buffer<T> &src) {
    transfer(coarse, false, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.h.id(), src.which, -1, stencil::Which::curr, false);
  }
  // restrict_to with an op (DESIGN.md section 2.11): dst = the 8-cell average of op(src, aux), the fine values never
  // stored; op has plain terms of reach <= 1, src is a curr buffer (its ghost cells are read).  exchange = true: the
  // coarse interior (the compute region cut by 1) runs while exchange() fills the ghost cells, then the exterior slabs;
  // exchange = false: one launch, the caller guarantees the ghost cells.  The op is part of the plan key.
  //     fine.restrict_to(coarse, stencil::curr(f2), residual, u, stencil::curr(f));   // f2 = R (f - A u)
  template <typename T>
  void restrict_to(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::LinearStencil &op, const DataHandle<T> &src,
                   const stencil::Buffer<T> &aux, stencil::Exchange exchange = true) {
    transfer(coarse, false, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), stencil::Which::curr, int64_t(aux.h.id()), aux.which, exchange, &op);
  }
  template <typename T>
  void restrict_to(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::LinearStencil &op, const DataHandle<T> &src,
                   stencil::Exchange exchange = true) {
    transfer(coarse, false, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), stencil::Which::curr, -1, stencil::Which::curr, exchange, &op);
  }
  // restrict_to with a coefficient op (DESIGN.md section 2.12): coefs are op.ncoef() fine quantities (curr buffers,
  // exchanged like src); the result is the bits of apply() into a scratch quantity followed by restrict_to().
  //     fine.restrict_to(coarse, stencil::curr(f2), residual, u, stencil::curr(f), {kx, ky, kz});
  template <typename T>
  void restrict_to(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::LinearStencil &op, const DataHandle<T> &src,
                   const stencil::Buffer<T> &aux, const std::vector<DataHandle<T>> &coefs, stencil::Exchange exchange = true) {
    transfer(coarse, false, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.id(), stencil::Which::curr, int64_t(aux.h.id()), aux.which, exchange, &op,
             ids_of(coefs));
  }
  // the face-coefficient restriction (DESIGN.md section 2.12): src holds values on the faces normal to axis (0, 1, 2),
  // C_a(p) on the face between p - e_a and p; dst = the average of the four fine faces of each coarse face.
  //     fine.restrict_to(coarse, stencil::curr(kx2), stencil::curr(kx), 0);
  template <typename T> void restrict_to(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::Buffer<T> &src, int axis) {
    if (axis < 0 || axis > 2) LOG_FATAL("restrict_to: face axis " << axis << " must be 0, 1 or 2");
    transfer(coarse, false, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.h.id(), src.which, -1, stencil::Which::curr, false, nullptr, {}, axis);
  }
  template <typename T>
  void prolong_from(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::Buffer<T> &src, stencil::Exchange exchange = true) {
    transfer(coarse, true, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.h.id(), src.which, -1, stencil::Which::curr, exchange);
  }
  template <typename T>
  void prolong_from(DistributedDomain &coarse, const stencil::Buffer<T> &dst, const stencil::Buffer<T> &src, const stencil::Buffer<T> &aux,
                    stencil::Exchange exchange = true) {
    transfer(coarse, true, stencil::bc_dtype<T>(), dst.h.id(), dst.which, src.h.id(), src.which, int64_t(aux.h.id()), aux.which, exchange);
  }

  // one CSV file per subdomain: Z,Y,X,<quantities...>
  void write_paraview(const std::string &prefix, bool zeroNaNs = false);

protected:
  bool poll_advance_sends() { return false; } // nothing is host-driven any more
};
