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
#include <map>
#include <set>
#include <string>
#include <vector>

#include <mpi.h>

#include <nvToolsExt.h>
#include <nvml.h>

#include "stencil/cuda_runtime.hpp"

#include "stencil/dim3.hpp"
#include "stencil/direction_map.hpp"
#include "stencil/gpu_topology.hpp"
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
#include "stencil/topology.hpp"
#include "stencil/tx.hpp"

struct sb_copy_plan;

class DistributedDomain {
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
  Topology::Boundary boundary_; // PERIODIC (the reference's only kind) or FIXED

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
    return DataHandle<T>(dataElemSize_.size() - 1, name);
  }

  // choose transports (before realize):  d.set_methods(Method::CudaMpi | Method::CudaKernel);
  void set_methods(Method flags) noexcept;
  void set_placement(PlacementStrategy strategy) noexcept { strategy_ = strategy; }
  // how the grid closes at its faces (before realize).  PERIODIC is the reference's behaviour; FIXED plans no messages
  // across the faces of the whole grid (the ghost cells there keep what the application put into them)
  void set_boundary(Topology::Boundary boundary) noexcept { boundary_ = boundary; }
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
  cudaStream_t exchange_stream(size_t domain) const { return streams_[domain]; }

  // one CSV file per subdomain: Z,Y,X,<quantities...>
  void write_paraview(const std::string &prefix, bool zeroNaNs = false);

protected:
  bool poll_advance_sends() { return false; } // nothing is host-driven any more
};
