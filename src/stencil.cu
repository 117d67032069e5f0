// DistributedDomain for one NVSwitch node (see include/stencil/stencil.hpp).
//
// Where the reference plans, per message, one of six sender/receiver state machines and then polls
// them from the host (reference src/stencil.cu:327-464, 1002-1186), this implementation plans ONE
// fused copy kernel per local subdomain: every outgoing (direction x quantity) halo region is a
// segment of that kernel, read from the subdomain's outermost compute cells and stored straight
// into the ghost cells of the destination subdomain -- same GPU, or a peer GPU through the
// NVLink/NVSwitch peer mapping.  exchange() = N launches + N stream syncs, nothing else.
#include "stencil/stencil.hpp"
#include "stencil/exchange_plan.hpp"

#include "stencil_b200.h"

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <sstream>

namespace {

sb_pitched as_sb(const cudaPitchedPtr &p) { return sb_pitched{p.ptr, int64_t(p.pitch), int64_t(p.ysize)}; }

void set3(int64_t out[3], const Dim3 &d) {
  out[0] = d.x;
  out[1] = d.y;
  out[2] = d.z;
}

} // namespace

DistributedDomain::DistributedDomain(size_t x, size_t y, size_t z)
    : size_(x, y, z), placement_(nullptr), radius_(Radius::constant(0)), flags_(Method::Default),
      strategy_(PlacementStrategy::NodeAware), boundary_{Topology::Boundary::PERIODIC, Topology::Boundary::PERIODIC, Topology::Boundary::PERIODIC}, parity_(0), mailbox_(nullptr), epoch_(0), numBytesCudaMpi_(0), numBytesColoDirectAccess_(0),
      numBytesColoPackMemcpyUnpack_(0), numBytesCudaMemcpyPeer_(0), numBytesCudaKernel_(0) {
#ifdef STENCIL_SETUP_STATS
  timeMpiTopo_ = timeNodeGpus_ = timePeerEn_ = timePlacement_ = timePlan_ = timeRealize_ = timeCreate_ = 0;
#endif
#ifdef STENCIL_EXCHANGE_STATS
  timeExchange_ = timeSwap_ = 0;
#endif
  static std::atomic<uint64_t> domains_made{0};
  serial_ = ++domains_made;
  MPI_Comm_rank(MPI_COMM_WORLD, &rank_);
  MPI_Comm_size(MPI_COMM_WORLD, &worldSize_);
  if (const char *s = std::getenv("STENCIL_OUTPUT_PREFIX")) outputPrefix_ = s;

  mpiTopology_ = MpiTopology(MPI_COMM_WORLD);

  int deviceCount = 0;
  CUDA_RUNTIME(cudaGetDeviceCount(&deviceCount));
  if (deviceCount < 1) {
    LOG_FATAL("no CUDA device: this library has no CPU path");
  }

  // default device choice: colocated ranks deal the node's GPUs round-robin; more ranks than GPUs share
  const int coloSize = mpiTopology_.colocated_size(), coloRank = mpiTopology_.colocated_rank();
  if (coloSize <= deviceCount) {
    for (int id = coloRank; id < deviceCount; id += coloSize) gpus_.push_back(id);
  } else {
    gpus_.push_back(coloRank % deviceCount);
  }

  // all-pairs peer access between the devices of this node
  nvtxRangePush("peer_en");
  for (int a = 0; a < deviceCount; ++a)
    for (int b = 0; b < deviceCount; ++b) gpu_topo::enable_peer(a, b);
  nvtxRangePop();
  CUDA_RUNTIME(cudaGetLastError());
}

DistributedDomain::~DistributedDomain() {
  close_ranks();
  destroy_plans();
  streams_.clear();
  delete placement_;
  placement_ = nullptr;
}

void DistributedDomain::destroy_plans() {
  destroy_reduce_plans();
  destroy_krylov_plans();
  destroy_transfer_plans();
  destroy_stencil_plans();
  for (auto *sides : {&plans_, &unpackPlans_}) {
    for (int parity = 0; parity < 2; ++parity) {
      for (sb_copy_plan *p : (*sides)[parity])
        if (p) sb_copy_plan_destroy(p);
      (*sides)[parity].clear();
    }
  }
  for (int parity = 0; parity < 2; ++parity) {
    for (sb_bc_plan *p : bcPlans_[parity])
      if (p) sb_bc_plan_destroy(p);
    bcPlans_[parity].clear();
    fullCopies_[parity].clear();
    fullScatter_[parity].clear();
    bcQuantities_[parity].clear();
  }
  for (auto &kv : subsetPlans_) {
    for (auto *v : {&kv.second.copy, &kv.second.scatter})
      for (sb_copy_plan *p : *v)
        if (p) sb_copy_plan_destroy(p);
    for (sb_bc_plan *p : kv.second.bc)
      if (p) sb_bc_plan_destroy(p);
  }
  subsetPlans_.clear();
  agreedSets_.clear();
  bcSenders_.clear();
  for (size_t i = 0; i < stagingBufs_.size(); ++i) {
    cudaSetDevice(stagingDevs_[i]);
    cudaFree(stagingBufs_[i]);
  }
  stagingBufs_.clear();
  stagingDevs_.clear();
  for (size_t i = 0; i < phase1Done_.size(); ++i) {
    cudaSetDevice(domains_[i].gpu());
    cudaEventDestroy(phase1Done_[i]);
  }
  phase1Done_.clear();
  stageSenders_.clear();
}

void DistributedDomain::set_methods(Method flags) noexcept {
  if ((flags && Method::ColoQuantityKernel) && (flags && Method::ColoPackMemcpyUnpack)) {
    LOG_FATAL("can't use Direct Access and Pack-Memcpy-Unpack for colocated ranks");
  }
  flags_ = flags;
}

void DistributedDomain::set_output_prefix(const std::string &prefix) { outputPrefix_ = prefix; }

uint64_t DistributedDomain::exchange_bytes_for_method(const Method &method) const {
  uint64_t total = 0;
  if (method && Method::CudaMpi) total += numBytesCudaMpi_;
  if (method && Method::ColoQuantityKernel) total += numBytesColoDirectAccess_;
  if (method && Method::ColoPackMemcpyUnpack) total += numBytesColoPackMemcpyUnpack_;
  if (method && Method::CudaMemcpyPeer) total += numBytesCudaMemcpyPeer_;
  if (method && Method::CudaKernel) total += numBytesCudaKernel_;
  return total;
}

void DistributedDomain::do_placement() {
  nvtxRangePush("placement");
  assert(!placement_);
  switch (strategy_) {
  case PlacementStrategy::NodeAware:
    placement_ = new NodeAware(size_, mpiTopology_, radius_, gpus_);
    break;
  case PlacementStrategy::Trivial:
    placement_ = new Trivial(size_, mpiTopology_, gpus_);
    break;
  case PlacementStrategy::IntraNodeRandom:
    placement_ = new IntraNodeRandom(size_, mpiTopology_, radius_, gpus_);
    break;
  }
  nvtxRangePop();
  topology_ = Topology(placement_->dim(), boundary_[0], boundary_[1], boundary_[2]);
}

void DistributedDomain::realize() {
  do_placement();
  for (const auto &kv : bcs_) { // the BC errors that need no subdomain geometry (sb_bc_plan_create checks the rest)
    const stencil::BC &bc = kv.second;
    const size_t q = kv.first.first;
    const int f = kv.first.second;
    if (bc.kind == stencil::BC::Kind::NONE) continue;
    if (boundary_[f / 2] == Topology::Boundary::PERIODIC)
      LOG_FATAL("quantity " << q << ": a boundary condition on face " << f << " (-x,+x,-y,+y,-z,+z) of a periodic axis; set_boundary FIXED first");
    if ((bc.kind == stencil::BC::Kind::VALUE || bc.kind == stencil::BC::Kind::ODD) && 0 == dataDtype_[q])
      LOG_FATAL("quantity " << q << ": VALUE and ODD boundary conditions need a float or double quantity (EVEN copies any type)");
  }

  // LocalDomain copies share raw device pointers: fill the vector while they are still null,
  // then allocate in place.
  domains_.reserve(gpus_.size());
  for (int64_t id = 0; id < int64_t(gpus_.size()); ++id) {
    const Dim3 idx = placement_->get_idx(rank_, int(id));
    LocalDomain sd(placement_->subdomain_size(idx), placement_->subdomain_origin(idx), placement_->get_cuda(idx));
    sd.set_radius(radius_);
    for (size_t q = 0; q < dataElemSize_.size(); ++q) sd.add_data(dataElemSize_[q], dataName_[q]);
    domains_.push_back(sd);
    domainIdx_.push_back(idx);
  }
  for (LocalDomain &d : domains_) d.realize();

  streams_.clear();
  for (const LocalDomain &d : domains_) streams_.push_back(RcStream(d.gpu(), RcStream::Priority::HIGH));

  nvtxRangePush("DistributedDomain::realize() plan");
  plan_exchange();
  nvtxRangePop();
  MPI_Barrier(MPI_COMM_WORLD);
}

// ---- other ranks of the node ------------------------------------------------------------------------------------------
namespace {
constexpr int kMaxDomPerRank = 8, kMaxQuantities = 16, kMaxStagePerRank = kMaxDomPerRank * 26;
struct DomRecord {
  int64_t idx[3], raw[3];
  int nq;
  cudaIpcMemHandle_t curr[kMaxQuantities], next[kMaxQuantities]; // handle of the cudaMalloc block ...
  uint64_t currOff[kMaxQuantities], nextOff[kMaxQuantities];     // ... and the allocation's offset inside it (lead_bytes)
};
struct StageRecord {
  int64_t src[3], dst[3];
  cudaIpcMemHandle_t handle;
};
struct RankRecord {
  int ndom, nstage;
  cudaIpcMemHandle_t flags;
  DomRecord dom[kMaxDomPerRank];
  StageRecord stage[kMaxStagePerRank];
};
} // namespace

// Collective.  Publishes this rank's allocations, staging buffers and mailbox; maps what its neighbours published.
void DistributedDomain::share_with_ranks(const std::map<std::pair<Dim3, Dim3>, char *> &myStage) {
  if (domains_.size() > size_t(kMaxDomPerRank) || dataElemSize_.size() > size_t(kMaxQuantities) || myStage.size() > size_t(kMaxStagePerRank))
    LOG_FATAL("multi-rank exchange supports <= " << kMaxDomPerRank << " subdomains per rank and <= " << kMaxQuantities << " quantities");
  const int dev0 = domains_[0].gpu();
  for (const LocalDomain &d : domains_)
    if (d.gpu() != dev0) LOG_FATAL("with several ranks every rank drives ONE GPU (the IPC mappings are opened on one device)");
  CUDA_RUNTIME(cudaSetDevice(dev0));
  CUDA_RUNTIME(cudaMalloc(&mailbox_, 2 * size_t(worldSize_) * sizeof(uint32_t)));
  CUDA_RUNTIME(cudaMemset(mailbox_, 0, 2 * size_t(worldSize_) * sizeof(uint32_t)));
  CUDA_RUNTIME(cudaDeviceSynchronize());

  std::vector<RankRecord> all;
  all.resize(size_t(worldSize_));
  RankRecord &me = all[size_t(rank_)];
  std::memset(&me, 0, sizeof(me));
  me.ndom = int(domains_.size());
  CUDA_RUNTIME(cudaIpcGetMemHandle(&me.flags, mailbox_));
  for (size_t di = 0; di < domains_.size(); ++di) {
    const LocalDomain &d = domains_[di];
    DomRecord &r = me.dom[di];
    set3(r.idx, domainIdx_[di]);
    set3(r.raw, d.raw_size());
    r.nq = int(d.num_data());
    CUDA_RUNTIME(cudaSetDevice(d.gpu()));
    for (int64_t q = 0; q < d.num_data(); ++q) {
      const size_t lead = d.lead_bytes(size_t(q));
      CUDA_RUNTIME(cudaIpcGetMemHandle(&r.curr[q], static_cast<char *>(d.curr_data(size_t(q)).ptr) - lead));
      CUDA_RUNTIME(cudaIpcGetMemHandle(&r.next[q], static_cast<char *>(d.next_data(size_t(q)).ptr) - lead));
      r.currOff[q] = r.nextOff[q] = lead;
    }
  }
  for (const auto &kv : myStage) {
    StageRecord &sr = me.stage[me.nstage++];
    set3(sr.src, kv.first.first);
    set3(sr.dst, kv.first.second);
    CUDA_RUNTIME(cudaIpcGetMemHandle(&sr.handle, kv.second));
  }
  {
    const RankRecord mine = me; // Allgather's send buffer must not alias the receive buffer
    MPI_Allgather(&mine, int(sizeof(RankRecord)), MPI_BYTE, all.data(), int(sizeof(RankRecord)), MPI_BYTE, MPI_COMM_WORLD);
  }

  // which subdomains of other ranks do mine talk to?
  std::set<Dim3> wanted;
  std::set<int> nbrs;
  for (size_t di = 0; di < domains_.size(); ++di)
    for (int z = -1; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x) {
          if (0 == x && 0 == y && 0 == z) continue;
          const Topology::OptionalNeighbor nb = topology_.get_neighbor(domainIdx_[di], Dim3(x, y, z));
          if (!nb.exists) continue;
          const int r = placement_->get_rank(nb.index);
          if (r == rank_) continue;
          wanted.insert(nb.index);
          nbrs.insert(r);
        }
  nbrRanks_.assign(nbrs.begin(), nbrs.end());
  peerFlags_.assign(size_t(worldSize_), nullptr);
  CUDA_RUNTIME(cudaSetDevice(dev0));
  auto open = [&](const cudaIpcMemHandle_t &h) {
    void *p = nullptr;
    CUDA_RUNTIME(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    ipcOpened_.push_back(p);
    return static_cast<char *>(p);
  };
  for (int r : nbrRanks_) {
    const RankRecord &rec = all[size_t(r)];
    peerFlags_[size_t(r)] = reinterpret_cast<uint32_t *>(open(rec.flags));
    for (int i = 0; i < rec.ndom; ++i) {
      const DomRecord &dr = rec.dom[i];
      const Dim3 idx(dr.idx[0], dr.idx[1], dr.idx[2]);
      if (!wanted.count(idx)) continue;
      RemoteDomain rd;
      rd.raw = Dim3(dr.raw[0], dr.raw[1], dr.raw[2]);
      for (int q = 0; q < dr.nq; ++q) {
        rd.curr.push_back(open(dr.curr[q]) + dr.currOff[q]);
        rd.next.push_back(open(dr.next[q]) + dr.nextOff[q]);
      }
      remote_[idx] = rd;
    }
    for (int i = 0; i < rec.nstage; ++i) {
      const StageRecord &sr = rec.stage[i];
      const Dim3 src(sr.src[0], sr.src[1], sr.src[2]), dst(sr.dst[0], sr.dst[1], sr.dst[2]);
      if (placement_->get_rank(src) == rank_) remoteStage_[std::make_pair(src, dst)] = open(sr.handle);
    }
  }
}

void DistributedDomain::close_ranks() {
  if (!mailbox_) return;
  for (const LocalDomain &d : domains_) {
    cudaSetDevice(d.gpu());
    cudaDeviceSynchronize();
  }
  MPI_Barrier(MPI_COMM_WORLD); // nobody unmaps while a neighbour could still be writing
  cudaSetDevice(domains_[0].gpu());
  for (void *p : ipcOpened_) cudaIpcCloseMemHandle(p);
  ipcOpened_.clear();
  remote_.clear();
  remoteStage_.clear();
  MPI_Barrier(MPI_COMM_WORLD); // ... and nobody frees what a neighbour still has mapped
  cudaFree(mailbox_);
  mailbox_ = nullptr;
}

// exchange e, before the copies: tell every neighbour rank that my ghost cells may be overwritten, wait until they said so
void DistributedDomain::flags_begin() {
  if (nbrRanks_.empty()) return;
  const int dev = domains_[0].gpu();
  std::vector<uint32_t *> slots;
  for (int r : nbrRanks_) slots.push_back(peerFlags_[size_t(r)] + rank_);
  if (SB_OK != sb_signal(slots.data(), int(slots.size()), epoch_, dev, streams_[0])) LOG_FATAL("exchange: " << sb_last_error());
  for (int r : nbrRanks_)
    if (SB_OK != sb_wait(mailbox_ + r, 1, epoch_, dev, streams_[0])) LOG_FATAL("exchange: " << sb_last_error());
  if (streams_.size() > 1) { // the other local subdomains start after the handshake
    cudaEvent_t ev = phase1Done_[0];
    CUDA_RUNTIME(cudaSetDevice(dev));
    CUDA_RUNTIME(cudaEventRecord(ev, streams_[0]));
    for (size_t di = 1; di < streams_.size(); ++di) {
      CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
      CUDA_RUNTIME(cudaStreamWaitEvent(streams_[di], ev, 0));
    }
  }
}

// after the copies of every local subdomain: tell the neighbours they have landed, wait for theirs
void DistributedDomain::flags_finish() {
  if (nbrRanks_.empty()) return;
  const int dev = domains_[0].gpu();
  for (size_t di = 1; di < streams_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
    CUDA_RUNTIME(cudaEventRecord(phase1Done_[di], streams_[di]));
    CUDA_RUNTIME(cudaSetDevice(dev));
    CUDA_RUNTIME(cudaStreamWaitEvent(streams_[0], phase1Done_[di], 0));
  }
  std::vector<uint32_t *> slots;
  for (int r : nbrRanks_) slots.push_back(peerFlags_[size_t(r)] + worldSize_ + rank_);
  if (SB_OK != sb_signal(slots.data(), int(slots.size()), epoch_, dev, streams_[0])) LOG_FATAL("exchange: " << sb_last_error());
  for (int r : nbrRanks_)
    if (SB_OK != sb_wait(mailbox_ + worldSize_ + r, 1, epoch_, dev, streams_[0])) LOG_FATAL("exchange: " << sb_last_error());
  if (streams_.size() > 1) {
    CUDA_RUNTIME(cudaSetDevice(dev));
    CUDA_RUNTIME(cudaEventRecord(phase1Done_[0], streams_[0]));
    for (size_t di = 1; di < streams_.size(); ++di) {
      CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
      CUDA_RUNTIME(cudaStreamWaitEvent(streams_[di], phase1Done_[0], 0));
    }
  }
}

// For each local subdomain and each of the 26 directions with a non-zero radius on the receiving
// side: source box = outermost compute cells on side `dir`, destination box = ghost cells on side
// -dir of the neighbour, extent = the neighbour's halo extent on side -dir.  The neighbour may be a
// local subdomain (same or peer GPU) or a subdomain of another rank of this node (CUDA IPC mapping).
void DistributedDomain::plan_exchange() {
  destroy_plans();
  numBytesCudaMpi_ = numBytesColoDirectAccess_ = numBytesColoPackMemcpyUnpack_ = numBytesCudaMemcpyPeer_ = numBytesCudaKernel_ = 0;

  std::ofstream planFile(outputPrefix_ + "plan_" + std::to_string(rank_) + ".txt");
  planFile << "rank=" << rank_ << "\n\ndomains\n";
  for (size_t di = 0; di < domains_.size(); ++di)
    planFile << di << ":cuda" << domains_[di].gpu() << ":" << domainIdx_[di] << " sz=" << domains_[di].size() << "\n";
  planFile << "\n== fused direct-write messages ==\n";

  auto gpu_key = [&](const Dim3 &idx) { return std::make_pair(placement_->get_rank(idx), placement_->get_cuda(idx)); };
  auto local_id = [&](const Dim3 &idx) { return placement_->get_rank(idx) == rank_ ? placement_->get_subdomain_id(idx) : -1; };
  auto neighbors = [&](const Dim3 &idx) {
    std::set<Dim3> out;
    for (int z = -1; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x) {
          if (0 == x && 0 == y && 0 == z) continue;
          const Topology::OptionalNeighbor nb = topology_.get_neighbor(idx, Dim3(x, y, z));
          if (nb.exists) out.insert(nb.index);
        }
    return out;
  };

  // ---- the plan (include/stencil/exchange_plan.hpp), computed once: the messages of every subdomain that sends to or
  // receives from a local one, and the staging layout of every such (src, dst) pair on different GPUs
  std::map<Dim3, std::vector<stencil::Message>> sends;
  for (const Dim3 &idx : domainIdx_) {
    sends[idx];
    for (const Dim3 &nb : neighbors(idx)) sends[nb];
  }
  for (auto &kv : sends)
    kv.second = stencil::messages_from(kv.first, topology_, radius_, [&](const Dim3 &idx) { return placement_->subdomain_size(idx); });
  const std::vector<int64_t> elemSizes(dataElemSize_.begin(), dataElemSize_.end());
  struct Layout {
    std::vector<stencil::Staged> entries;
    int64_t total = 0;
  };
  std::map<std::pair<Dim3, Dim3>, Layout> layouts; // only pairs with something staged
  for (const auto &kv : sends)
    for (const stencil::Message &m : kv.second) {
      const auto key = std::make_pair(m.srcIdx, m.dstIdx);
      if ((local_id(m.srcIdx) < 0 && local_id(m.dstIdx) < 0) || gpu_key(m.srcIdx) == gpu_key(m.dstIdx) || layouts.count(key)) continue;
      Layout l;
      l.entries = stencil::staging_layout(kv.second, m.dstIdx, elemSizes, &l.total);
      if (l.total > 0) layouts[key] = l;
    }

  // ---- staging buffers I receive into (allocated here, published to the senders) ----------------------------
  std::map<std::pair<Dim3, Dim3>, char *> myStage; // (src idx, dst idx) -> buffer on dst's GPU
  stageSenders_.assign(domains_.size(), {});
  for (size_t dj = 0; dj < domains_.size(); ++dj) {
    for (const Dim3 &srcIdx : neighbors(domainIdx_[dj])) {
      const auto key = std::make_pair(srcIdx, domainIdx_[dj]);
      const auto it = layouts.find(key);
      if (it == layouts.end()) continue;
      void *buf = nullptr;
      CUDA_RUNTIME(cudaSetDevice(domains_[dj].gpu()));
      CUDA_RUNTIME(cudaMalloc(&buf, size_t(it->second.total)));
      stagingBufs_.push_back(buf);
      stagingDevs_.push_back(domains_[dj].gpu());
      myStage[key] = static_cast<char *>(buf);
      if (local_id(srcIdx) >= 0) stageSenders_[dj].push_back(size_t(local_id(srcIdx)));
    }
  }
  for (size_t di = 0; di < domains_.size(); ++di) {
    cudaEvent_t ev;
    CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
    CUDA_RUNTIME(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    phase1Done_.push_back(ev);
  }
  if (worldSize_ > 1) share_with_ranks(myStage);

  // pointer of quantity q of subdomain idx, in the naming of swap parity `parity` (all ranks swap in lock step)
  auto pitched_of = [&](const Dim3 &idx, size_t q, int parity) {
    const int id = local_id(idx);
    if (id >= 0) {
      const LocalDomain &d = domains_[size_t(id)];
      return as_sb(0 == parity ? d.curr_data(q) : d.next_data(q));
    }
    auto it = remote_.find(idx);
    if (it == remote_.end()) LOG_FATAL("subdomain " << idx << " of rank " << placement_->get_rank(idx) << " was not shared");
    const RemoteDomain &rd = it->second;
    return sb_pitched{0 == parity ? rd.curr[q] : rd.next[q], rd.raw.x * int64_t(dataElemSize_[q]), rd.raw.y};
  };

  // ---- the two plans per subdomain and swap parity -----------------------------------------------------
  const size_t nq = dataElemSize_.size();
  for (int parity = 0; parity < 2; ++parity) {
    for (size_t di = 0; di < domains_.size(); ++di) {
      const LocalDomain &src = domains_[di];
      const std::vector<stencil::Message> &msgs = sends.at(domainIdx_[di]);
      // staging offset of quantity q of message i at [i * nq + q], -1 where it goes straight into the ghost cells
      std::vector<int64_t> stagedAt(msgs.size() * nq, -1);
      for (const auto &kv : layouts)
        if (kv.first.first == domainIdx_[di])
          for (const stencil::Staged &st : kv.second.entries) stagedAt[st.msg * nq + size_t(st.q)] = st.offset;
      std::vector<sb_box_copy> copies;
      std::vector<TaggedCopy> tagged;
      for (size_t i = 0; i < msgs.size(); ++i) {
        const stencil::Message &m = msgs[i];
        const bool sameGpu = gpu_key(m.srcIdx) == gpu_key(m.dstIdx);
        const bool remote = placement_->get_rank(m.dstIdx) != rank_;
        if (!remote && !gpu_topo::peer(src.gpu(), placement_->get_cuda(m.dstIdx)))
          LOG_FATAL("GPU " << src.gpu() << " cannot map GPU " << placement_->get_cuda(m.dstIdx) << " (no P2P): unsupported on this path");
        // where this pair's thin rows go, if anywhere
        const auto key = std::make_pair(m.srcIdx, m.dstIdx);
        char *stageBase = nullptr;
        if (layouts.count(key)) {
          stageBase = remote ? remoteStage_[key] : myStage[key];
          if (!stageBase) LOG_FATAL("no staging buffer for " << m.srcIdx << " -> " << m.dstIdx);
        }
        uint64_t msgBytes = 0;
        for (size_t q = 0; q < nq; ++q) {
          sb_box_copy c{};
          c.elem_size = int64_t(dataElemSize_[q]);
          msgBytes += uint64_t(c.elem_size) * m.ext.flatten();
          c.src = pitched_of(m.srcIdx, q, parity);
          set3(c.src_pos, m.srcPos);
          set3(c.extent, m.ext);
          const int64_t offset = stagedAt[i * nq + q];
          if (offset >= 0) { // dense staging buffer in the receiver's memory
            c.dst = sb_pitched{stageBase + offset, m.ext.x * c.elem_size, m.ext.y};
          } else {
            c.dst = pitched_of(m.dstIdx, q, parity);
            set3(c.dst_pos, m.dstPos);
          }
          copies.push_back(c);
          tagged.push_back(TaggedCopy{q, c});
        }
        if (0 == parity) { // attribute the bytes the way the reference's planner picks a transport (src/stencil.cu:383-445)
          const char *how = "";
          if (remote) {
            if (any_methods(Method::ColoPackMemcpyUnpack)) numBytesColoPackMemcpyUnpack_ += msgBytes, how = "colo-rank";
            else if (any_methods(Method::ColoQuantityKernel)) numBytesColoDirectAccess_ += msgBytes, how = "colo-rank";
            else if (any_methods(Method::CudaMpi)) numBytesCudaMpi_ += msgBytes, how = "colo-rank(mpi)";
            else LOG_FATAL("No method available to send required message " << m.dir << "\n");
          } else if (any_methods(Method::CudaKernel) && sameGpu) {
            numBytesCudaKernel_ += msgBytes, how = "same-gpu";
          } else if (any_methods(Method::CudaMemcpyPeer)) {
            numBytesCudaMemcpyPeer_ += msgBytes, how = "peer";
          } else if (any_methods(Method::CudaMpi)) {
            numBytesCudaMpi_ += msgBytes, how = "self-mpi";
          } else {
            LOG_FATAL("No method available to send required message " << m.dir << "\n");
          }
          planFile << m.srcIdx << "->" << m.dstIdx << " " << m.dir << " " << msgBytes << "B " << how << (stageBase ? " (thin rows staged)" : "") << "\n";
        }
      }
      sb_copy_plan *plan = nullptr;
      if (SB_OK != sb_copy_plan_create(&plan, src.gpu(), copies.data(), int64_t(copies.size()))) {
        LOG_FATAL("exchange plan: " << sb_last_error());
      }
      plans_[parity].push_back(plan);
      fullCopies_[parity].push_back(std::move(tagged));

      // phase 2 of this subdomain as a receiver
      std::vector<sb_box_copy> scatter;
      std::vector<TaggedCopy> taggedScatter;
      for (const auto &kv : layouts) {
        if (!(kv.first.second == domainIdx_[di])) continue;
        for (const stencil::Staged &st : kv.second.entries) {
          const stencil::Message &m = sends.at(kv.first.first)[st.msg];
          sb_box_copy c{};
          c.elem_size = int64_t(dataElemSize_[size_t(st.q)]);
          c.src = sb_pitched{myStage[kv.first] + st.offset, m.ext.x * c.elem_size, m.ext.y};
          c.dst = pitched_of(domainIdx_[di], size_t(st.q), parity);
          set3(c.dst_pos, m.dstPos);
          set3(c.extent, m.ext);
          scatter.push_back(c);
          taggedScatter.push_back(TaggedCopy{size_t(st.q), c});
        }
      }
      sb_copy_plan *up = nullptr;
      if (!scatter.empty() && SB_OK != sb_copy_plan_create(&up, src.gpu(), scatter.data(), int64_t(scatter.size()))) {
        LOG_FATAL("exchange scatter plan: " << sb_last_error());
      }
      unpackPlans_[parity].push_back(up);
      fullScatter_[parity].push_back(std::move(taggedScatter));
    }
  }
  plan_boundaries(planFile);
  planFile.close();
  parity_ = 0;

  // rank x rank payload bytes per exchange, for numpy.loadtxt (the reference dumps the same file: src/stencil.cu:476-503)
  {
    std::vector<double> mat(size_t(worldSize_) * size_t(worldSize_), 0.0);
    for (size_t di = 0; di < domains_.size(); ++di)
      for (const stencil::Message &m : sends.at(domainIdx_[di])) {
        double bytes = 0;
        for (size_t q = 0; q < dataElemSize_.size(); ++q) bytes += double(dataElemSize_[q]) * double(m.ext.flatten());
        mat[size_t(rank_) * size_t(worldSize_) + size_t(placement_->get_rank(m.dstIdx))] += bytes;
      }
    MPI_Allreduce(MPI_IN_PLACE, mat.data(), int(mat.size()), MPI_DOUBLE, MPI_SUM, MPI_COMM_WORLD);
    if (0 == rank_) {
      std::ofstream matFile(outputPrefix_ + "mat_npy_loadtxt.txt");
      for (int r = 0; r < worldSize_; ++r) {
        for (int c = 0; c < worldSize_; ++c) matFile << mat[size_t(r) * size_t(worldSize_) + size_t(c)] << " ";
        matFile << "\n";
      }
    }
  }

  // every rank learns the global volume
  for (uint64_t *b : {&numBytesCudaMpi_, &numBytesColoDirectAccess_, &numBytesColoPackMemcpyUnpack_, &numBytesCudaMemcpyPeer_, &numBytesCudaKernel_})
    MPI_Allreduce(MPI_IN_PLACE, b, 1, MPI_UINT64_T, MPI_SUM, MPI_COMM_WORLD);
}

// Boundary conditions: per local subdomain and swap parity, one sb_bc_plan over the BCs of its wall faces (faces with no
// neighbour), and the local subdomains whose phase 1 writes into it.
void DistributedDomain::plan_boundaries(std::ofstream &planFile) {
  bcSenders_.assign(domains_.size(), {});
  if (!has_boundary_conditions()) return;
  static const char *const kKind[4] = {"NONE", "VALUE", "EVEN", "ODD"};
  static const char *const kFace[6] = {"-x", "+x", "-y", "+y", "-z", "+z"};
  const Dim3 faceDir[6] = {Dim3(-1, 0, 0), Dim3(1, 0, 0), Dim3(0, -1, 0), Dim3(0, 1, 0), Dim3(0, 0, -1), Dim3(0, 0, 1)};
  int64_t r27[27];
  for (int z = -1, i = 0; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(radius_.dir(x, y, z));
  planFile << "\n== boundary conditions ==\n";
  for (int parity = 0; parity < 2; ++parity) {
    for (size_t di = 0; di < domains_.size(); ++di) {
      const LocalDomain &d = domains_[di];
      std::vector<sb_bc_quantity> qs(dataElemSize_.size());
      for (size_t q = 0; q < qs.size(); ++q) {
        sb_bc_quantity &Q = qs[q];
        Q = sb_bc_quantity{};
        Q.data = as_sb(0 == parity ? d.curr_data(q) : d.next_data(q));
        Q.elem_size = int64_t(dataElemSize_[q]);
        Q.dtype = dataDtype_[q];
        for (int f = 0; f < 6; ++f) {
          const auto it = bcs_.find(std::make_pair(q, f));
          if (it == bcs_.end() || topology_.get_neighbor(domainIdx_[di], faceDir[f]).exists) continue;
          Q.kind[f] = int32_t(it->second.kind);
          Q.value[f] = it->second.value;
          if (0 == parity && it->second.kind != stencil::BC::Kind::NONE)
            planFile << domainIdx_[di] << " q" << q << " " << kFace[f] << " " << kKind[int(it->second.kind)] << "(" << it->second.value << ")\n";
        }
      }
      int64_t sz[3];
      set3(sz, d.size());
      sb_bc_plan *plan = nullptr;
      if (SB_OK != sb_bc_plan_create(&plan, d.gpu(), qs.data(), int64_t(qs.size()), sz, r27)) LOG_FATAL("boundary conditions: " << sb_last_error());
      if (0 == parity) planFile << domainIdx_[di] << " BC plan: " << sb_bc_plan_bytes(plan) << "B per exchange\n";
      if (0 == sb_bc_plan_bytes(plan)) {
        sb_bc_plan_destroy(plan);
        plan = nullptr;
      }
      bcPlans_[parity].push_back(plan);
      bcQuantities_[parity].push_back(qs);
    }
  }
  for (size_t di = 0; di < domains_.size(); ++di) {
    std::set<size_t> senders;
    for (int z = -1; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x) {
          const Topology::OptionalNeighbor nb = topology_.get_neighbor(domainIdx_[di], Dim3(x, y, z));
          if ((x || y || z) && nb.exists && placement_->get_rank(nb.index) == rank_) senders.insert(size_t(placement_->get_subdomain_id(nb.index)));
        }
    bcSenders_[di].assign(senders.begin(), senders.end());
  }
}

void DistributedDomain::swap() {
#ifdef STENCIL_EXCHANGE_STATS
  MPI_Barrier(MPI_COMM_WORLD);
  const double start = MPI_Wtime();
#endif
  for (LocalDomain &d : domains_) d.swap();
  parity_ ^= 1; // the exchange plans exist for both identities of "current"
#ifdef STENCIL_EXCHANGE_STATS
  double elapsed = MPI_Wtime() - start, maxElapsed = -1;
  MPI_Reduce(&elapsed, &maxElapsed, 1, MPI_DOUBLE, MPI_MAX, 0, MPI_COMM_WORLD);
  if (0 == rank_) timeSwap_ += maxElapsed;
#endif
}

void DistributedDomain::destroy_reduce_plans() {
  for (auto &kv : reducePlans_) {
    for (size_t di = 0; di < kv.second.plans.size(); ++di) {
      sb_reduce_plan_destroy(kv.second.plans[di]);
      cudaSetDevice(domains_[di].gpu());
      cudaFree(kv.second.out[di]);
    }
    for (size_t di = 0; di < kv.second.xplans.size(); ++di) {
      sb_reduce_exact_plan_destroy(kv.second.xplans[di]);
      cudaSetDevice(domains_[di].gpu());
      cudaFree(kv.second.xout[di]);
    }
  }
  reducePlans_.clear();
}

void DistributedDomain::destroy_stencil_plans() {
  for (auto &kv : stencilPlans_)
    for (auto &per_dom : kv.second)
      for (sb_stencil_plan *p : per_dom) sb_stencil_plan_destroy(p);
  stencilPlans_.clear();
  for (size_t i = 0; i < applyStreams_.size() && !sharedApplyStreams_; ++i) {
    cudaSetDevice(domains_[i / 2].gpu());
    cudaStreamDestroy(applyStreams_[i]);
  }
  applyStreams_.clear();
  for (size_t i = 0; i < applyEvents_.size(); ++i) {
    cudaSetDevice(domains_[i / 2].gpu());
    cudaEventDestroy(applyEvents_[i]);
  }
  applyEvents_.clear();
  for (size_t i = 0; i < exchangeEvents_.size(); ++i) {
    cudaSetDevice(domains_[i].gpu());
    cudaEventDestroy(exchangeEvents_[i]);
  }
  exchangeEvents_.clear();
}

void DistributedDomain::apply_op(const stencil::LinearStencil &op, int dtype, size_t dq, stencil::Which dw, size_t sq, int64_t aq,
                                 stencil::Which aw, const std::vector<size_t> &cq, stencil::Exchange exchange, stencil::Colour colour,
                                 const double *omega) {
  using stencil::Which;
  const char *name = omega ? "relax" : "apply";
  if (domains_.empty() || plans_[0].size() != domains_.size()) LOG_FATAL(name << ": call realize() first");
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL(name << ": a stencil operator computes in float or double");
  for (const int64_t q : {int64_t(dq), int64_t(sq), aq})
    if (q >= 0 && (size_t(q) >= dataDtype_.size() || dataDtype_[size_t(q)] != dtype)) LOG_FATAL(name << ": unknown data handle " << q);
  if ((colour.m != 1 && colour.m != 2 && colour.m != 8) || colour.c < 0 || colour.c >= colour.m)
    LOG_FATAL(name << ": colour (" << colour.m << ", " << colour.c << ") must have m = 1, 2 or 8 and 0 <= c < m");
  if (dq == sq && dw == Which::curr && colour.m == 1) LOG_FATAL(name << ": dst must not be src");
  if (op.has_aux() && aq < 0) LOG_FATAL(name << ": the op has a term on aux, but no aux buffer was given");
  if (omega) {
    if (op.has_aux()) LOG_FATAL("relax: A has a term on aux; A reads u only (f is the right-hand side)");
    bool centre = false;
    for (const sb_stencil_vterm &t : op.vterms()) centre = centre || (t.source == 0 && !t.offset[0] && !t.offset[1] && !t.offset[2]);
    if (!centre) LOG_FATAL("relax: A has no term at offset (0, 0, 0), so no diagonal");
    if (!std::isfinite(*omega)) LOG_FATAL("relax: omega = " << *omega << " must be finite");
  }
  if (int(cq.size()) != op.ncoef()) LOG_FATAL(name << ": the op reads " << op.ncoef() << " coefficient fields, but " << cq.size() << " were given");
  for (size_t k = 0; k < cq.size(); ++k) {
    if (cq[k] >= dataDtype_.size() || dataDtype_[cq[k]] != dtype) LOG_FATAL(name << ": coefficient " << k << " is not a quantity of the op's type");
    if (cq[k] == dq && dw == Which::curr) LOG_FATAL(name << ": coefficient " << k << " must not be dst");
  }
  int64_t r27[27];
  for (int z = -1, i = 0; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(radius_.dir(x, y, z));
  const std::vector<sb_stencil_vterm> &terms = op.vterms();
  if (SB_OK != sb_stencil_ccheck(terms.data(), int(terms.size()), r27, colour.m)) LOG_FATAL(name << ": " << sb_last_error());
  if (!op.has_aux() && !omega) aq = -1;
  uint64_t reads = sq < 64 ? uint64_t(1) << sq : 0; // src and the coefficient fields read at a non-zero offset
  for (const sb_stencil_vterm &t : terms)
    if (t.coef >= 0 && (t.coef_offset[0] || t.coef_offset[1] || t.coef_offset[2]) && cq[size_t(t.coef)] < 64) reads |= uint64_t(1) << cq[size_t(t.coef)];
  const uint64_t xq = exchange_set(name, exchange, reads);
  std::vector<int64_t> key = {dtype, int64_t(dq), int64_t(dw == Which::next), int64_t(sq), aq, int64_t(aw == Which::next), int64_t(xq != 0), parity_,
                              colour.m, colour.c, int64_t(cq.size())};
  for (const size_t q : cq) key.push_back(int64_t(q));
  if (omega) { // the diagonal mode and omega's bits (the plain key ends with a term's 9 entries, so the two never collide)
    int64_t obits;
    std::memcpy(&obits, omega, 8);
    key.insert(key.end(), {-2, obits});
  }
  for (const sb_stencil_vterm &t : terms) {
    int64_t wbits;
    std::memcpy(&wbits, &t.weight, 8);
    key.insert(key.end(), {t.source, t.offset[0], t.offset[1], t.offset[2], t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2], wbits});
  }
  run_stencil_plans(key, xq, dq == sq && dw == Which::curr, [&](size_t di, const std::vector<Rect3> &boxes) {
    LocalDomain &d = domains_[di];
    const sb_pitched dst = as_sb(dw == Which::curr ? d.curr_data(dq) : d.next_data(dq)), src = as_sb(d.curr_data(sq));
    const sb_pitched aux = aq < 0 ? sb_pitched{nullptr, 0, 0} : as_sb(aw == Which::curr ? d.curr_data(size_t(aq)) : d.next_data(size_t(aq)));
    std::vector<sb_pitched> coef;
    for (const size_t q : cq) coef.push_back(as_sb(d.curr_data(q)));
    int64_t acc[3];
    set3(acc, d.origin() - Dim3(radius_.x(-1), radius_.y(-1), radius_.z(-1)));
    std::vector<int64_t> lo, hi;
    for (const Rect3 &b : boxes) {
      lo.insert(lo.end(), {b.lo.x, b.lo.y, b.lo.z});
      hi.insert(hi.end(), {b.hi.x, b.hi.y, b.hi.z});
    }
    sb_stencil_plan *p = nullptr;
    const int rc = omega ? sb_stencil_dplan_create(&p, d.gpu(), dtype, terms.data(), int(terms.size()), dst, src, aux, coef.data(), int(coef.size()),
                                                   *omega, colour.m, colour.c, acc, d.raw_size().z, int(boxes.size()), lo.data(), hi.data())
                         : sb_stencil_cplan_create(&p, d.gpu(), dtype, terms.data(), int(terms.size()), dst, src, aux, coef.data(), int(coef.size()),
                                                   colour.m, colour.c, acc, d.raw_size().z, int(boxes.size()), lo.data(), hi.data());
    if (SB_OK != rc) LOG_FATAL(name << ": " << sb_last_error());
    return p;
  });
}

void DistributedDomain::apply_sys(const stencil::LinearSystem &sys, int dtype, const std::vector<std::pair<size_t, stencil::Which>> &outs,
                                  const std::vector<std::pair<size_t, stencil::Which>> &ins, stencil::Exchange exchange) {
  using stencil::Which;
  if (domains_.empty() || plans_[0].size() != domains_.size()) LOG_FATAL("apply: call realize() first");
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL("apply: a stencil system computes in float or double");
  if (int(outs.size()) != sys.nout() || int(ins.size()) != sys.nin())
    LOG_FATAL("apply: the system has " << sys.nin() << " inputs and " << sys.nout() << " outputs, but " << ins.size() << " inputs and "
                                       << outs.size() << " outputs were given");
  for (const auto *v : {&outs, &ins})
    for (const auto &b : *v)
      if (b.first >= dataDtype_.size() || dataDtype_[b.first] != dtype) LOG_FATAL("apply: unknown data handle or type for " << b.first);
  const std::vector<sb_stencil_sys_term> &terms = sys.terms();
  std::vector<bool> moved(ins.size(), false);
  for (const sb_stencil_sys_term &t : terms) {
    if (t.input >= 0 && size_t(t.input) < ins.size() && (t.offset[0] || t.offset[1] || t.offset[2])) moved[size_t(t.input)] = true;
    if (t.coef >= 0 && size_t(t.coef) < ins.size() && (t.coef_offset[0] || t.coef_offset[1] || t.coef_offset[2])) moved[size_t(t.coef)] = true;
  }
  for (size_t i = 0; i < ins.size(); ++i)
    if (moved[i] && ins[i].second != Which::curr)
      LOG_FATAL("apply: input " << i << " is read at a non-zero offset, so it must be a curr buffer (the one exchange() fills)");
  for (size_t j = 0; j < outs.size(); ++j) {
    for (size_t k = 0; k < j; ++k)
      if (outs[k] == outs[j]) LOG_FATAL("apply: outputs " << k << " and " << j << " are the same buffer");
    for (size_t i = 0; i < ins.size(); ++i)
      if (moved[i] && ins[i] == outs[j]) LOG_FATAL("apply: output " << j << " is input " << i << ", which is read at a non-zero offset");
  }
  int64_t r27[27];
  for (int z = -1, i = 0; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(radius_.dir(x, y, z));
  if (SB_OK != sb_stencil_sys_check(terms.data(), int(terms.size()), sys.nin(), sys.nout(), r27)) LOG_FATAL("apply: " << sb_last_error());
  // -1 first: a system's key never equals an operator's, whose first entry is a dtype code
  uint64_t reads = 0; // the inputs read at a non-zero offset
  for (size_t i = 0; i < ins.size(); ++i)
    if (moved[i] && ins[i].first < 64) reads |= uint64_t(1) << ins[i].first;
  const uint64_t xq = exchange_set("apply", exchange, reads);
  std::vector<int64_t> key = {-1, dtype, int64_t(xq != 0), parity_, sys.nin(), sys.nout()};
  for (const auto *v : {&outs, &ins})
    for (const auto &b : *v) key.insert(key.end(), {int64_t(b.first), int64_t(b.second == Which::next)});
  for (const sb_stencil_sys_term &t : terms) {
    int64_t wbits;
    std::memcpy(&wbits, &t.weight, 8);
    key.insert(key.end(), {t.output, t.input, t.offset[0], t.offset[1], t.offset[2], t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2], wbits});
  }
  run_stencil_plans(key, xq, false, [&](size_t di, const std::vector<Rect3> &boxes) {
    LocalDomain &d = domains_[di];
    std::vector<sb_pitched> o, i;
    for (const auto &b : outs) o.push_back(as_sb(b.second == Which::curr ? d.curr_data(b.first) : d.next_data(b.first)));
    for (const auto &b : ins) i.push_back(as_sb(b.second == Which::curr ? d.curr_data(b.first) : d.next_data(b.first)));
    int64_t acc[3];
    set3(acc, d.origin() - Dim3(radius_.x(-1), radius_.y(-1), radius_.z(-1)));
    std::vector<int64_t> lo, hi;
    for (const Rect3 &b : boxes) {
      lo.insert(lo.end(), {b.lo.x, b.lo.y, b.lo.z});
      hi.insert(hi.end(), {b.hi.x, b.hi.y, b.hi.z});
    }
    sb_stencil_plan *p = nullptr;
    if (SB_OK != sb_stencil_sys_plan_create(&p, d.gpu(), dtype, terms.data(), int(terms.size()), o.data(), int(o.size()), i.data(), int(i.size()),
                                            acc, d.raw_size().z, int(boxes.size()), lo.data(), hi.data()))
      LOG_FATAL("apply: " << sb_last_error());
    return p;
  });
}

uint64_t DistributedDomain::exchange_set(const char *name, const stencil::Exchange &exchange, uint64_t reads) const {
  const uint64_t all = dataElemSize_.size() >= 64 ? ~uint64_t(0) : (uint64_t(1) << dataElemSize_.size()) - 1;
  switch (exchange.mode) {
  case stencil::Exchange::kNone: return 0;
  case stencil::Exchange::kAll: return stencil::kAllQuantities;
  case stencil::Exchange::kReads: return reads == all ? stencil::kAllQuantities : reads;
  case stencil::Exchange::kOnly:
    if (exchange.quantities & ~all) LOG_FATAL(name << ": Exchange::only names a quantity the domain does not have");
    return exchange.quantities == all ? stencil::kAllQuantities : exchange.quantities;
  }
  return stencil::kAllQuantities;
}

void DistributedDomain::run_stencil_plans(const std::vector<int64_t> &key, uint64_t exchange, bool writes_src,
                                          const std::function<sb_stencil_plan *(size_t, const std::vector<Rect3> &)> &make) {
  auto found = stencilPlans_.find(key);
  if (found == stencilPlans_.end()) {
    // exchange() sends from side s of a subdomain a slab as wide as the radius on side -s; an apply that writes src
    // (a coloured one in place) keeps its interior clear of both, so the interior writes no cell exchange() reads
    Radius cut = radius_;
    if (writes_src)
      for (int z = -1; z <= 1; ++z)
        for (int y = -1; y <= 1; ++y)
          for (int x = -1; x <= 1; ++x) cut.dir(x, y, z) = std::max(radius_.dir(x, y, z), radius_.dir(-x, -y, -z));
    std::vector<std::vector<sb_stencil_plan *>> per_dom;
    for (size_t di = 0; di < domains_.size(); ++di) {
      const Rect3 compute = domains_[di].get_compute_region();
      if (exchange)
        per_dom.push_back({make(di, {stencil::geom::interior(compute, cut)}), make(di, stencil::geom::exterior(compute, cut))});
      else
        per_dom.push_back({make(di, {domains_[di].get_compute_region()})});
    }
    found = stencilPlans_.emplace(key, std::move(per_dom)).first;
  }
  const std::vector<std::vector<sb_stencil_plan *>> &plans = found->second;
  queued_schedule([&](size_t di, int part, cudaStream_t s) {
    if (SB_OK != sb_stencil_plan_launch(plans[di][size_t(part)], s)) LOG_FATAL("apply: " << sb_last_error());
  }, exchange);
}

void DistributedDomain::ensure_queue_events() {
  create_apply_streams();
  for (size_t i = applyEvents_.size(); i < applyStreams_.size(); ++i) {
    CUDA_RUNTIME(cudaSetDevice(domains_[i / 2].gpu()));
    cudaEvent_t e;
    CUDA_RUNTIME(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    applyEvents_.push_back(e);
  }
  for (size_t i = exchangeEvents_.size(); i < streams_.size(); ++i) {
    CUDA_RUNTIME(cudaSetDevice(domains_[i].gpu()));
    cudaEvent_t e;
    CUDA_RUNTIME(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    exchangeEvents_.push_back(e);
  }
}

void DistributedDomain::queue_after_exterior() {
  ensure_queue_events();
  for (size_t di = 0; di < domains_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
    CUDA_RUNTIME(cudaEventRecord(applyEvents_[2 * di + 1], applyStreams_[2 * di + 1]));
    CUDA_RUNTIME(cudaStreamWaitEvent(applyStreams_[2 * di], applyEvents_[2 * di + 1], 0));
  }
}

void DistributedDomain::clear_queued(size_t q) {
  queue_after_exterior();
  for (size_t di = 0; di < domains_.size(); ++di) {
    LocalDomain &d = domains_[di];
    d.set_device();
    const cudaPitchedPtr p = d.curr_data(q);
    CUDA_RUNTIME(cudaMemsetAsync(p.ptr, 0, p.pitch * p.ysize * size_t(d.raw_size().z), applyStreams_[2 * di]));
  }
}

void DistributedDomain::queue_exchange(uint64_t quantities) {
  ensure_queue_events();
  for (size_t i = 0; i < applyStreams_.size(); ++i) {
    CUDA_RUNTIME(cudaSetDevice(domains_[i / 2].gpu()));
    CUDA_RUNTIME(cudaEventRecord(applyEvents_[i], applyStreams_[i]));
  }
  for (size_t di = 0; di < streams_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
    for (cudaEvent_t e : applyEvents_) CUDA_RUNTIME(cudaStreamWaitEvent(streams_[di], e, 0));
  }
  exchange_async_set(quantities);
}

void DistributedDomain::wait_exchange(DistributedDomain &other, bool interior) {
  ensure_queue_events();
  other.ensure_queue_events();
  for (size_t di = 0; di < other.streams_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(other.domains_[di].gpu()));
    CUDA_RUNTIME(cudaEventRecord(other.exchangeEvents_[di], other.streams_[di]));
  }
  for (size_t di = 0; di < domains_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
    for (cudaEvent_t e : other.exchangeEvents_) {
      CUDA_RUNTIME(cudaStreamWaitEvent(applyStreams_[2 * di + 1], e, 0));
      if (interior) CUDA_RUNTIME(cudaStreamWaitEvent(applyStreams_[2 * di], e, 0));
    }
  }
}

void DistributedDomain::queued_schedule(const std::function<void(size_t, int, cudaStream_t)> &launch, uint64_t exchange) {
  queue_after_exterior();
  if (exchange) queue_exchange(exchange); // waits for the apply streams as they are before this interior
  for (size_t di = 0; di < domains_.size(); ++di) {
    domains_[di].set_device();
    launch(di, 0, applyStreams_[2 * di]);
  }
  if (exchange) {
    wait_exchange(*this, false);
    for (size_t di = 0; di < domains_.size(); ++di) {
      domains_[di].set_device();
      launch(di, 1, applyStreams_[2 * di + 1]);
    }
  }
  if (!queued_) wait_queued({this});
}

void DistributedDomain::wait_queued(const std::vector<DistributedDomain *> &doms) {
  std::set<cudaStream_t> waited; // a solver's levels share the finest level's apply streams
  for (DistributedDomain *dd : doms) {
    for (size_t i = 0; i < dd->applyStreams_.size(); ++i)
      if (waited.insert(dd->applyStreams_[i]).second) {
        CUDA_RUNTIME(cudaSetDevice(dd->domains_[i / 2].gpu()));
        CUDA_RUNTIME(cudaStreamSynchronize(dd->applyStreams_[i]));
      }
    dd->exchange_wait();
  }
}

void DistributedDomain::create_apply_streams() {
  if (!applyStreams_.empty()) return;
  // blocking streams: ordered after the work the caller queued on the legacy default stream
  for (LocalDomain &d : domains_) {
    d.set_device();
    for (int k = 0; k < 2; ++k) {
      cudaStream_t s;
      CUDA_RUNTIME(cudaStreamCreate(&s));
      applyStreams_.push_back(s);
    }
  }
}

// ---- multigrid transfers (DESIGN.md section 2.10) ------------------------------------------------------------------------
void DistributedDomain::destroy_transfer_plans() {
  for (auto &kv : transferPlans_)
    for (sb_transfer_plan *p : kv.second) sb_transfer_plan_destroy(p);
  transferPlans_.clear();
  paired_.clear();
}

void DistributedDomain::check_pairing(DistributedDomain &coarse, bool ghosts) {
  if (paired_.count(std::make_pair(coarse.serial_, ghosts))) return;
  const Dim3 fdim = placement_->dim(), cdim = coarse.placement_->dim();
  int64_t fd[3], cd[3];
  set3(fd, fdim);
  set3(cd, cdim);
  // every subdomain index, x fastest: global information, so every rank reaches the same verdict
  std::vector<Dim3> idx;
  for (int64_t z = 0; z < fdim.z; ++z)
    for (int64_t y = 0; y < fdim.y; ++y)
      for (int64_t x = 0; x < fdim.x; ++x) idx.push_back(Dim3(x, y, z));
  std::vector<int64_t> fo(3 * idx.size()), fs(3 * idx.size()), co(3 * idx.size()), cs(3 * idx.size());
  for (size_t k = 0; k < idx.size(); ++k) {
    set3(&fo[3 * k], placement_->subdomain_origin(idx[k]));
    set3(&fs[3 * k], placement_->subdomain_size(idx[k]));
    if (fdim == cdim) { // otherwise sb_transfer_check stops at the dims
      set3(&co[3 * k], coarse.placement_->subdomain_origin(idx[k]));
      set3(&cs[3 * k], coarse.placement_->subdomain_size(idx[k]));
    }
  }
  int64_t r27[27];
  for (int z = -1, i = 0; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(coarse.radius_.dir(x, y, z));
  if (SB_OK != sb_transfer_check(fd, cd, fo.data(), fs.data(), co.data(), cs.data(), ghosts ? r27 : nullptr))
    LOG_FATAL("transfer: " << sb_last_error());
  for (const Dim3 &i : idx) {
    if (placement_->get_rank(i) != coarse.placement_->get_rank(i) || placement_->get_subdomain_id(i) != coarse.placement_->get_subdomain_id(i))
      LOG_FATAL("transfer: subdomain " << i << " belongs to another rank or local slot on the coarse level");
    if (placement_->get_cuda(i) != coarse.placement_->get_cuda(i))
      LOG_FATAL("transfer: subdomain " << i << " is on GPU " << placement_->get_cuda(i) << " on the fine level and GPU " << coarse.placement_->get_cuda(i)
                                       << " on the coarse one");
  }
  paired_.insert(std::make_pair(coarse.serial_, ghosts));
}

void DistributedDomain::transfer(DistributedDomain &coarse, bool prolong, int dtype, size_t dq, stencil::Which dw, size_t sq, stencil::Which sw,
                                 int64_t aq, stencil::Which aw, stencil::Exchange exchange, const stencil::LinearStencil *op, const std::vector<size_t> &cq,
                                 int face) {
  using stencil::Which;
  const char *name = prolong ? "prolong_from" : "restrict_to";
  if (&coarse == this) LOG_FATAL(name << ": coarse must be another DistributedDomain");
  if (domains_.empty() || plans_[0].size() != domains_.size() || coarse.domains_.empty() || coarse.plans_[0].size() != coarse.domains_.size())
    LOG_FATAL(name << ": call realize() on both domains first");
  if (dtype != SB_DTYPE_F32 && dtype != SB_DTYPE_F64) LOG_FATAL(name << ": a transfer computes in float or double");
  DistributedDomain &D = prolong ? *this : coarse, &S = prolong ? coarse : *this;
  if (dq >= D.dataDtype_.size() || D.dataDtype_[dq] != dtype) LOG_FATAL(name << ": dst " << dq << " is not a quantity of that type");
  if (sq >= S.dataDtype_.size() || S.dataDtype_[sq] != dtype) LOG_FATAL(name << ": src " << sq << " is not a quantity of that type");
  if (aq >= 0 && (size_t(aq) >= dataDtype_.size() || dataDtype_[size_t(aq)] != dtype)) LOG_FATAL(name << ": aux " << aq << " is not a quantity of that type");
  if (prolong && sw != Which::curr) LOG_FATAL(name << ": src must be a curr buffer (the one coarse.exchange() fills)");
  // what the call exchanges: before a prolongation the coarse src, in a fused restriction the fine src and the
  // coefficient fields read at a non-zero offset (Exchange::reads()); nothing for a plain restriction
  uint64_t xq = prolong ? coarse.exchange_set(name, exchange, sq < 64 ? uint64_t(1) << sq : 0) : 0;
  std::vector<int64_t> key = {int64_t(coarse.serial_), int64_t(prolong), int64_t(dq), int64_t(dw == Which::next), int64_t(sq),
                              int64_t(sw == Which::next), aq, int64_t(aw == Which::next), parity_, coarse.parity_};
  if (op) {
    if (prolong) LOG_FATAL(name << ": only a restriction takes an op");
    if (int(cq.size()) != op->ncoef()) LOG_FATAL(name << ": the op reads " << op->ncoef() << " coefficient fields, but " << cq.size() << " were given");
    for (size_t k = 0; k < cq.size(); ++k)
      if (cq[k] >= dataDtype_.size() || dataDtype_[cq[k]] != dtype) LOG_FATAL(name << ": coefficient " << k << " is not a quantity of that type");
    if (sw != Which::curr) LOG_FATAL(name << ": with an op, src must be a curr buffer (the one exchange() fills)");
    if (op->has_aux() && aq < 0) LOG_FATAL(name << ": the op has a term on aux, but no aux buffer was given");
    int64_t r27[27];
    for (int z = -1, i = 0; z <= 1; ++z)
      for (int y = -1; y <= 1; ++y)
        for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(radius_.dir(x, y, z));
    if (SB_OK != sb_stencil_vcheck(op->vterms().data(), int(op->vterms().size()), r27)) LOG_FATAL(name << ": " << sb_last_error());
    if (!op->has_aux()) {
      aq = -1;
      key[6] = -1;
      key[7] = 0;
    }
    uint64_t reads = sq < 64 ? uint64_t(1) << sq : 0;
    for (const sb_stencil_vterm &t : op->vterms())
      if (t.coef >= 0 && (t.coef_offset[0] || t.coef_offset[1] || t.coef_offset[2]) && cq[size_t(t.coef)] < 64) reads |= uint64_t(1) << cq[size_t(t.coef)];
    xq = exchange_set(name, exchange, reads);
    key.push_back(int64_t(xq != 0));
    if (cq.empty()) {
      for (const sb_stencil_term &t : op->terms()) {
        int64_t wbits;
        std::memcpy(&wbits, &t.weight, 8);
        key.insert(key.end(), {t.source, t.offset[0], t.offset[1], t.offset[2], wbits});
      }
    } else { // a coefficient op: a marker, the fields, then every term with its coefficient
      key.insert(key.end(), {-2, int64_t(cq.size())});
      for (const size_t q : cq) key.push_back(int64_t(q));
      for (const sb_stencil_vterm &t : op->vterms()) {
        int64_t wbits;
        std::memcpy(&wbits, &t.weight, 8);
        key.insert(key.end(), {t.source, t.offset[0], t.offset[1], t.offset[2], t.coef, t.coef_offset[0], t.coef_offset[1], t.coef_offset[2], wbits});
      }
    }
  }
  if (face >= 0) {
    if (op || prolong) LOG_FATAL(name << ": a face restriction takes no op");
    key.insert(key.end(), {-3, int64_t(face)});
  }
  const bool split = op && xq; // the fused restriction with apply's schedule: interior and exterior plans
  check_pairing(coarse, prolong);
  auto found = transferPlans_.find(key);
  if (found == transferPlans_.end()) {
    auto pick = [](LocalDomain &d, size_t q, Which w) { return as_sb(w == Which::curr ? d.curr_data(q) : d.next_data(q)); };
    std::vector<sb_transfer_plan *> per_dom; // per local domain: one plan, or (interior, exterior) when split
    Radius one = Radius::constant(1);
    for (size_t di = 0; di < domains_.size() && op; ++di) {
      LocalDomain &f = domains_[di], &cd = coarse.domains_[di];
      int64_t dacc[3], sacc[3];
      set3(dacc, cd.origin() - Dim3(coarse.radius_.x(-1), coarse.radius_.y(-1), coarse.radius_.z(-1)));
      set3(sacc, f.origin() - Dim3(radius_.x(-1), radius_.y(-1), radius_.z(-1)));
      const sb_pitched aux = aq < 0 ? sb_pitched{nullptr, 0, 0} : pick(f, size_t(aq), aw);
      const Rect3 compute = cd.get_compute_region();
      std::vector<std::vector<Rect3>> parts;
      if (split)
        parts = {{stencil::geom::interior(compute, one)}, stencil::geom::exterior(compute, one)};
      else
        parts = {{compute}};
      for (const std::vector<Rect3> &boxes : parts) {
        std::vector<int64_t> lo, hi;
        for (const Rect3 &b : boxes) {
          lo.insert(lo.end(), {b.lo.x, b.lo.y, b.lo.z});
          hi.insert(hi.end(), {b.hi.x, b.hi.y, b.hi.z});
        }
        sb_transfer_plan *p = nullptr;
        std::vector<sb_pitched> coef;
        for (const size_t q : cq) coef.push_back(as_sb(f.curr_data(q)));
        const int rc = cq.empty() ? sb_transfer_oplan_create(&p, f.gpu(), dtype, op->terms().data(), int(op->terms().size()), pick(cd, dq, dw), dacc,
                                                             cd.raw_size().z, pick(f, sq, sw), sacc, f.raw_size().z, aux, int(boxes.size()), lo.data(),
                                                             hi.data())
                                  : sb_transfer_voplan_create(&p, f.gpu(), dtype, op->vterms().data(), int(op->vterms().size()), pick(cd, dq, dw), dacc,
                                                              cd.raw_size().z, pick(f, sq, sw), sacc, f.raw_size().z, aux, coef.data(), int(coef.size()),
                                                              int(boxes.size()), lo.data(), hi.data());
        if (SB_OK != rc) LOG_FATAL(name << ": " << sb_last_error());
        per_dom.push_back(p);
      }
    }
    for (size_t di = 0; di < domains_.size() && !op; ++di) {
      LocalDomain &f = domains_[di], &dd = prolong ? f : coarse.domains_[di], &sd = prolong ? coarse.domains_[di] : f;
      int64_t dacc[3], sacc[3], lo[3], hi[3];
      set3(dacc, dd.origin() - Dim3(D.radius_.x(-1), D.radius_.y(-1), D.radius_.z(-1)));
      set3(sacc, sd.origin() - Dim3(S.radius_.x(-1), S.radius_.y(-1), S.radius_.z(-1)));
      const Rect3 box = dd.get_compute_region();
      set3(lo, box.lo);
      set3(hi, box.hi);
      const sb_pitched aux = aq < 0 ? sb_pitched{nullptr, 0, 0} : pick(f, size_t(aq), aw);
      sb_transfer_plan *p = nullptr;
      const int rc = face >= 0 ? sb_transfer_fplan_create(&p, f.gpu(), dtype, face, pick(dd, dq, dw), dacc, dd.raw_size().z, pick(sd, sq, sw), sacc,
                                                          sd.raw_size().z, lo, hi)
                               : sb_transfer_plan_create(&p, f.gpu(), dtype, prolong ? SB_TRANSFER_PROLONG : SB_TRANSFER_RESTRICT, pick(dd, dq, dw), dacc,
                                                         dd.raw_size().z, pick(sd, sq, sw), sacc, sd.raw_size().z, aux, lo, hi);
      if (SB_OK != rc) LOG_FATAL(name << ": " << sb_last_error());
      per_dom.push_back(p);
    }
    found = transferPlans_.emplace(key, std::move(per_dom)).first;
  }
  const std::vector<sb_transfer_plan *> &plans = found->second;
  const size_t per = split ? 2 : 1;
  if (prolong && xq) { // the coarse apply streams it waits for follow the legacy default stream (blocking streams)
    coarse.queue_exchange(xq);
    wait_exchange(coarse, true);
  }
  queued_schedule([&](size_t di, int part, cudaStream_t s) {
    if (SB_OK != sb_transfer_plan_launch(plans[per * di + size_t(part)], s)) LOG_FATAL(name << ": " << sb_last_error());
  }, split ? xq : 0);
}

std::vector<unsigned char> DistributedDomain::allgather_records(const std::vector<unsigned char> &mine) const {
  if (worldSize_ <= 1) return mine;
  const int count = int(mine.size());
  std::vector<int> counts(static_cast<size_t>(worldSize_)), displs(static_cast<size_t>(worldSize_));
  MPI_Allgather(&count, 1, MPI_INT, counts.data(), 1, MPI_INT, MPI_COMM_WORLD);
  int total = 0;
  for (int r = 0; r < worldSize_; ++r) {
    displs[size_t(r)] = total;
    total += counts[size_t(r)];
  }
  std::vector<unsigned char> all(size_t(total), 0);
  MPI_Allgatherv(mine.data(), count, MPI_BYTE, all.data(), counts.data(), displs.data(), MPI_BYTE, MPI_COMM_WORLD);
  return all;
}

std::vector<stencil::Reduction> DistributedDomain::reduce_many(const std::vector<stencil::ReduceItem> &items, stencil::Sum sum) {
  using stencil::Which;
  const bool exact = sum == stencil::Sum::exact;
  const size_t n = items.size();
  if (0 == n) return {};
  std::vector<int64_t> key;
  for (const stencil::ReduceItem &it : items) {
    const int ns = it.kind == SB_REDUCE_SCALAR ? 1 : it.kind == SB_REDUCE_DIFF ? 1 : 3;
    if (it.kind < SB_REDUCE_SCALAR || it.kind > SB_REDUCE_NORM3) LOG_FATAL("reduce: unknown kind " << int(it.kind));
    for (int s = 0; s < ns; ++s) {
      if (it.q[s] >= dataDtype_.size()) LOG_FATAL("reduce: unknown data handle " << it.q[s]);
      if (dataDtype_[it.q[s]] != SB_DTYPE_F32 && dataDtype_[it.q[s]] != SB_DTYPE_F64) LOG_FATAL("reduce: quantity " << it.q[s] << " is not float or double");
      if (dataDtype_[it.q[s]] != dataDtype_[it.q[0]]) LOG_FATAL("reduce: the sources of a norm must share one type");
    }
    key.insert(key.end(), {int64_t(it.kind), int64_t(it.q[0]), int64_t(ns == 3 ? it.q[1] : it.q[0]), int64_t(ns == 3 ? it.q[2] : it.q[0]),
                           int64_t(it.kind == SB_REDUCE_SCALAR && it.which == Which::next)});
  }
  key.push_back(parity_);
  key.push_back(int64_t(exact));
  auto found = reducePlans_.find(key);
  if (found == reducePlans_.end()) {
    ReduceCache c;
    for (LocalDomain &d : domains_) {
      const Rect3 cr = d.get_compute_region();
      const Dim3 ao = d.origin() - Dim3(radius_.x(-1), radius_.y(-1), radius_.z(-1));
      std::vector<sb_reduce_item> its(n);
      for (size_t i = 0; i < n; ++i) {
        const stencil::ReduceItem &it = items[i];
        sb_reduce_item &r = its[i];
        r.kind = it.kind;
        r.dtype = dataDtype_[it.q[0]];
        for (int s = 0; s < 3; ++s) {
          cudaPitchedPtr p = d.curr_data(it.kind == SB_REDUCE_NORM3 ? it.q[s] : it.q[0]);
          if ((it.kind == SB_REDUCE_SCALAR && it.which == Which::next) || (it.kind == SB_REDUCE_DIFF && s == 1)) p = d.next_data(it.q[0]);
          r.src[s] = sb_pitched{p.ptr, int64_t(p.pitch), int64_t(p.ysize)};
        }
        const int64_t acc[3] = {ao.x, ao.y, ao.z}, lo[3] = {cr.lo.x, cr.lo.y, cr.lo.z}, hi[3] = {cr.hi.x, cr.hi.y, cr.hi.z};
        for (int a = 0; a < 3; ++a) {
          r.acc_origin[a] = acc[a];
          r.lo[a] = lo[a];
          r.hi[a] = hi[a];
        }
      }
      if (exact) {
        sb_reduce_exact_plan *plan = nullptr;
        if (SB_OK != sb_reduce_exact_plan_create(&plan, d.gpu(), its.data(), int64_t(n))) LOG_FATAL("reduce: " << sb_last_error());
        sb_reduce_exact_part *out = nullptr;
        d.set_device();
        CUDA_RUNTIME(cudaMalloc(&out, n * sizeof(sb_reduce_exact_part)));
        c.xplans.push_back(plan);
        c.xout.push_back(out);
      } else {
        sb_reduce_plan *plan = nullptr;
        if (SB_OK != sb_reduce_plan_create(&plan, d.gpu(), its.data(), int64_t(n))) LOG_FATAL("reduce: " << sb_last_error());
        sb_reduce_result *out = nullptr;
        d.set_device();
        CUDA_RUNTIME(cudaMalloc(&out, n * sizeof(sb_reduce_result)));
        c.plans.push_back(plan);
        c.out.push_back(out);
      }
    }
    found = reducePlans_.emplace(key, std::move(c)).first;
  }
  const ReduceCache &c = found->second;
  // 1. all work already queued on the local devices
  for (const int dev : std::set<int>(gpus_.begin(), gpus_.end())) {
    CUDA_RUNTIME(cudaSetDevice(dev));
    CUDA_RUNTIME(cudaDeviceSynchronize());
  }
  // 2. one launch sequence per local subdomain on its exchange stream; records: global index, then n results
  const Dim3 dim = placement_->dim();
  //    (exact: n sb_reduce_exact_parts, gathered unrounded)
  const size_t res_size = exact ? sizeof(sb_reduce_exact_part) : sizeof(sb_reduce_result);
  const size_t rec = sizeof(int64_t) + n * res_size;
  std::vector<unsigned char> mine(domains_.size() * rec);
  for (size_t di = 0; di < domains_.size(); ++di) {
    domains_[di].set_device();
    const int rc = exact ? sb_reduce_exact_plan_launch(c.xplans[di], c.xout[di], streams_[di]) : sb_reduce_plan_launch(c.plans[di], c.out[di], streams_[di]);
    if (SB_OK != rc) LOG_FATAL("reduce: " << sb_last_error());
    const Dim3 &idx = domainIdx_[di];
    const int64_t lin = idx.x + dim.x * (idx.y + dim.y * idx.z);
    std::memcpy(&mine[di * rec], &lin, sizeof(lin));
    const void *src = exact ? static_cast<const void *>(c.xout[di]) : static_cast<const void *>(c.out[di]);
    CUDA_RUNTIME(cudaMemcpyAsync(&mine[di * rec + sizeof(int64_t)], src, n * res_size, cudaMemcpyDeviceToHost, streams_[di]));
  }
  for (size_t di = 0; di < domains_.size(); ++di) {
    domains_[di].set_device();
    CUDA_RUNTIME(cudaStreamSynchronize(streams_[di]));
  }
  // 3. every rank's records
  const std::vector<unsigned char> all = allgather_records(mine);
  // 4. merge in global subdomain-index order, the same on every rank
  const size_t nrec = all.size() / rec;
  std::vector<std::pair<int64_t, size_t>> order(nrec);
  for (size_t k = 0; k < nrec; ++k) {
    std::memcpy(&order[k].first, &all[k * rec], sizeof(int64_t));
    order[k].second = k;
  }
  std::sort(order.begin(), order.end());
  std::vector<stencil::Reduction> result(n);
  if (exact) { // combined (in any order: the sums are exact), then rounded once
    std::vector<sb_reduce_exact_part> xparts(nrec);
    for (size_t i = 0; i < n; ++i) {
      for (size_t k = 0; k < nrec; ++k)
        std::memcpy(&xparts[k], &all[order[k].second * rec + sizeof(int64_t) + i * res_size], sizeof(sb_reduce_exact_part));
      sb_reduce_exact_part tot;
      sb_reduce_result r;
      if (SB_OK != sb_reduce_exact_combine(xparts.data(), int64_t(nrec), &tot) || SB_OK != sb_reduce_exact_round(&tot, &r))
        LOG_FATAL("reduce: " << sb_last_error());
      result[i] = stencil::Reduction{r.min, r.max, r.sum, r.sumsq, r.count};
    }
    return result;
  }
  std::vector<sb_reduce_result> parts(nrec);
  for (size_t i = 0; i < n; ++i) {
    for (size_t k = 0; k < nrec; ++k)
      std::memcpy(&parts[k], &all[order[k].second * rec + sizeof(int64_t) + i * sizeof(sb_reduce_result)], sizeof(sb_reduce_result));
    sb_reduce_result r;
    if (SB_OK != sb_reduce_combine(parts.data(), int64_t(nrec), &r)) LOG_FATAL("reduce: " << sb_last_error());
    result[i] = stencil::Reduction{r.min, r.max, r.sum, r.sumsq, r.count};
  }
  return result;
}

// ---- Krylov vector passes (DESIGN.md section 2.13) -----------------------------------------------------------------------
void DistributedDomain::destroy_krylov_plans() {
  for (auto &kv : krylovPlans_)
    for (size_t di = 0; di < kv.second.plans.size(); ++di) {
      sb_krylov_plan_destroy(kv.second.plans[di]);
      cudaSetDevice(domains_[di].gpu());
      if (kv.second.out[di]) cudaFree(kv.second.out[di]);
    }
  krylovPlans_.clear();
}

DistributedDomain::KrylovCache &DistributedDomain::krylov_plans(int mode, const std::vector<size_t> &qs) {
  if (domains_.empty()) LOG_FATAL("krylov: call realize() first");
  std::vector<int64_t> key{int64_t(mode)};
  for (size_t q : qs) {
    if (q >= dataDtype_.size()) LOG_FATAL("krylov: unknown data handle " << q);
    if (dataDtype_[q] != SB_DTYPE_F32 && dataDtype_[q] != SB_DTYPE_F64) LOG_FATAL("krylov: quantity " << q << " is not float or double");
    if (dataDtype_[q] != dataDtype_[qs[0]]) LOG_FATAL("krylov: the quantities must share one type");
    key.push_back(int64_t(q));
  }
  key.push_back(parity_);
  auto found = krylovPlans_.find(key);
  if (found != krylovPlans_.end()) return found->second;
  KrylovCache c;
  c.nparts = mode == SB_KRYLOV_DOT ? int(qs.size()) - 1 : mode == SB_KRYLOV_UPDATE ? int(qs.size()) - 3 : 0; // UPDATE with c: 2
  for (LocalDomain &d : domains_) {
    const Rect3 cr = d.get_compute_region();
    const Dim3 ao = d.origin() - Dim3(radius_.x(-1), radius_.y(-1), radius_.z(-1));
    std::vector<sb_pitched> bufs;
    for (size_t q : qs) {
      const cudaPitchedPtr p = d.curr_data(q);
      bufs.push_back(sb_pitched{p.ptr, int64_t(p.pitch), int64_t(p.ysize)});
    }
    const int64_t acc[3] = {ao.x, ao.y, ao.z}, lo[3] = {cr.lo.x, cr.lo.y, cr.lo.z}, hi[3] = {cr.hi.x, cr.hi.y, cr.hi.z};
    sb_krylov_plan *plan = nullptr;
    if (SB_OK != sb_krylov_plan_create(&plan, d.gpu(), mode, dataDtype_[qs[0]], bufs.data(), int(bufs.size()), acc, lo, hi))
      LOG_FATAL("krylov: " << sb_last_error());
    sb_reduce_exact_part *out = nullptr;
    if (c.nparts) {
      d.set_device();
      CUDA_RUNTIME(cudaMalloc(&out, size_t(c.nparts) * sizeof(sb_reduce_exact_part)));
    }
    c.plans.push_back(plan);
    c.out.push_back(out);
  }
  return krylovPlans_.emplace(key, std::move(c)).first->second;
}

void DistributedDomain::krylov_launch(KrylovCache &c, double s, double t, bool queued) {
  if (queued) {
    create_apply_streams();
    queue_after_exterior();
  } else {
    for (const int dev : std::set<int>(gpus_.begin(), gpus_.end())) {
      CUDA_RUNTIME(cudaSetDevice(dev));
      CUDA_RUNTIME(cudaDeviceSynchronize());
    }
  }
  for (size_t di = 0; di < domains_.size(); ++di) {
    domains_[di].set_device();
    if (SB_OK != sb_krylov_plan_launch2(c.plans[di], s, t, c.out[di], queued ? applyStreams_[2 * di] : cudaStream_t(streams_[di])))
      LOG_FATAL("krylov: " << sb_last_error());
  }
}

std::vector<double> DistributedDomain::krylov_sums(const std::vector<KrylovCache *> &cs, bool queued) {
  size_t n = 0;
  for (const KrylovCache *c : cs) n += size_t(c->nparts);
  const size_t rec = sizeof(int64_t) + n * sizeof(sb_reduce_exact_part);
  const Dim3 dim = placement_->dim();
  std::vector<unsigned char> mine(domains_.size() * rec);
  for (size_t di = 0; di < domains_.size(); ++di) {
    domains_[di].set_device();
    const Dim3 &idx = domainIdx_[di];
    const int64_t lin = idx.x + dim.x * (idx.y + dim.y * idx.z);
    std::memcpy(&mine[di * rec], &lin, sizeof(lin));
    const cudaStream_t st = queued ? applyStreams_[2 * di] : cudaStream_t(streams_[di]);
    size_t at = di * rec + sizeof(int64_t);
    for (const KrylovCache *c : cs) { // each cache's parts after the previous one's
      const size_t bytes = size_t(c->nparts) * sizeof(sb_reduce_exact_part);
      CUDA_RUNTIME(cudaMemcpyAsync(&mine[at], c->out[di], bytes, cudaMemcpyDeviceToHost, st));
      at += bytes;
    }
  }
  for (size_t di = 0; di < domains_.size(); ++di) {
    domains_[di].set_device();
    CUDA_RUNTIME(cudaStreamSynchronize(queued ? applyStreams_[2 * di] : cudaStream_t(streams_[di])));
  }
  const std::vector<unsigned char> all = allgather_records(mine);
  // exact sums: combined in any order, then rounded once, the same on every rank
  const size_t nrec = all.size() / rec;
  std::vector<double> out(n);
  std::vector<sb_reduce_exact_part> parts(nrec);
  for (size_t i = 0; i < n; ++i) {
    for (size_t k = 0; k < nrec; ++k) std::memcpy(&parts[k], &all[k * rec + sizeof(int64_t) + i * sizeof(sb_reduce_exact_part)], sizeof(sb_reduce_exact_part));
    sb_reduce_exact_part tot;
    sb_reduce_result r;
    if (SB_OK != sb_reduce_exact_combine(parts.data(), int64_t(nrec), &tot) || SB_OK != sb_reduce_exact_round(&tot, &r))
      LOG_FATAL("krylov: " << sb_last_error());
    out[i] = r.sum;
  }
  return out;
}

std::vector<Rect3> DistributedDomain::get_interior() const {
  std::vector<Rect3> out;
  for (const LocalDomain &d : domains_) out.push_back(stencil::geom::interior(d.get_compute_region(), radius_));
  return out;
}

std::vector<std::vector<Rect3>> DistributedDomain::get_exterior() const {
  std::vector<std::vector<Rect3>> out;
  for (const LocalDomain &d : domains_) out.push_back(stencil::geom::exterior(d.get_compute_region(), radius_));
  return out;
}

const Rect3 DistributedDomain::get_compute_region() const noexcept { return Rect3(Dim3(0, 0, 0), size_); }

uint64_t DistributedDomain::quantity_set(const std::vector<size_t> &quantities) const {
  if (quantities.empty()) LOG_FATAL("exchange: the quantity list is empty (exchange() exchanges every quantity)");
  uint64_t set = 0;
  std::set<size_t> seen;
  for (const size_t q : quantities) {
    if (q >= dataElemSize_.size()) LOG_FATAL("exchange: quantity " << q << " is not one of the domain's " << dataElemSize_.size() << " quantities");
    if (!seen.insert(q).second) LOG_FATAL("exchange: quantity " << q << " is named twice");
  }
  if (seen.size() == dataElemSize_.size()) return stencil::kAllQuantities;
  for (const size_t q : seen) {
    if (q >= 64) LOG_FATAL("exchange: quantity " << q << ": a subset names quantities 0..63 only");
    set |= uint64_t(1) << q;
  }
  return set;
}

void DistributedDomain::exchange(const std::vector<size_t> &quantities) {
  exchange_async(quantities);
  exchange_wait();
}

void DistributedDomain::exchange_async(const std::vector<size_t> &quantities) {
  if (domains_.empty() || plans_[0].size() != domains_.size()) LOG_FATAL("exchange: call realize() first");
  exchange_async_set(quantity_set(quantities));
}

const DistributedDomain::SubsetPlans &DistributedDomain::subset_plans(uint64_t set) {
  const auto key = std::make_pair(parity_, set);
  auto found = subsetPlans_.find(key);
  if (found != subsetPlans_.end()) return found->second;
  if (!agreedSets_.count(set)) { // exchange() is collective: every rank must move the same quantities
    uint64_t lo = set, hi = set;
    MPI_Allreduce(MPI_IN_PLACE, &lo, 1, MPI_UINT64_T, MPI_MIN, MPI_COMM_WORLD);
    MPI_Allreduce(MPI_IN_PLACE, &hi, 1, MPI_UINT64_T, MPI_MAX, MPI_COMM_WORLD);
    if (lo != set || hi != set)
      LOG_FATAL("exchange: rank " << rank_ << " exchanges the quantity set 0x" << std::hex << set << ", another rank 0x" << (lo != set ? lo : hi)
                                  << std::dec << ": every rank must pass the same subset");
    agreedSets_.insert(set);
  }
  SubsetPlans sp;
  for (size_t di = 0; di < domains_.size(); ++di) {
    const int dev = domains_[di].gpu();
    std::vector<sb_box_copy> copies, scatter;
    for (const TaggedCopy &t : fullCopies_[parity_][di])
      if (stencil::in_set(set, t.q)) copies.push_back(t.c);
    for (const TaggedCopy &t : fullScatter_[parity_][di])
      if (stencil::in_set(set, t.q)) scatter.push_back(t.c);
    sb_copy_plan *p = nullptr, *u = nullptr;
    if (SB_OK != sb_copy_plan_create(&p, dev, copies.data(), int64_t(copies.size()))) LOG_FATAL("exchange plan: " << sb_last_error());
    if (!scatter.empty() && SB_OK != sb_copy_plan_create(&u, dev, scatter.data(), int64_t(scatter.size())))
      LOG_FATAL("exchange scatter plan: " << sb_last_error());
    sp.copy.push_back(p);
    sp.scatter.push_back(u);
    if (!bcPlans_[parity_].empty()) {
      std::vector<sb_bc_quantity> qs;
      for (size_t q = 0; q < bcQuantities_[parity_][di].size(); ++q)
        if (stencil::in_set(set, q)) qs.push_back(bcQuantities_[parity_][di][q]);
      int64_t sz[3], r27[27];
      set3(sz, domains_[di].size());
      for (int z = -1, i = 0; z <= 1; ++z)
        for (int y = -1; y <= 1; ++y)
          for (int x = -1; x <= 1; ++x) r27[i++] = int64_t(radius_.dir(x, y, z));
      sb_bc_plan *b = nullptr;
      if (SB_OK != sb_bc_plan_create(&b, dev, qs.data(), int64_t(qs.size()), sz, r27)) LOG_FATAL("boundary conditions: " << sb_last_error());
      if (0 == sb_bc_plan_bytes(b)) {
        sb_bc_plan_destroy(b);
        b = nullptr;
      }
      sp.bc.push_back(b);
    }
  }
  return subsetPlans_.emplace(key, std::move(sp)).first->second;
}

void DistributedDomain::exchange_async() { exchange_async_set(stencil::kAllQuantities); }

void DistributedDomain::exchange_async_set(uint64_t set) {
  nvtxRangePush("DD::exchange_async");
  const SubsetPlans *sub = set == stencil::kAllQuantities ? nullptr : &subset_plans(set);
  const std::vector<sb_copy_plan *> &plans = sub ? sub->copy : plans_[parity_];
  const std::vector<sb_copy_plan *> &scatter = sub ? sub->scatter : unpackPlans_[parity_];
  const bool ranks = !nbrRanks_.empty();
  if (ranks) {
    ++epoch_;
    flags_begin();
  }
  bool anyStaged = false;
  for (size_t di = 0; di < plans.size(); ++di) {
    if (SB_OK != sb_copy_plan_launch(plans[di], streams_[di])) {
      LOG_FATAL("exchange: " << sb_last_error());
    }
    anyStaged = anyStaged || (scatter[di] != nullptr);
  }
  if (ranks) flags_finish(); // every remote sender's phase 1 has landed (and stream order covers the local ones below)
  const std::vector<sb_bc_plan *> &bc = sub ? sub->bc : bcPlans_[parity_];
  if (!ranks && (anyStaged || !bc.empty())) {
    for (size_t di = 0; di < plans.size(); ++di) {
      CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
      CUDA_RUNTIME(cudaEventRecord(phase1Done_[di], streams_[di]));
    }
  }
  if (anyStaged) {
    for (size_t di = 0; di < plans.size(); ++di) {
      if (!scatter[di]) continue;
      CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
      if (!ranks) // (with ranks, flags_finish already made every stream wait for every local phase 1)
        for (size_t sj : stageSenders_[di]) CUDA_RUNTIME(cudaStreamWaitEvent(streams_[di], phase1Done_[sj], 0));
      if (SB_OK != sb_copy_plan_launch(scatter[di], streams_[di])) {
        LOG_FATAL("exchange scatter: " << sb_last_error());
      }
    }
  }
  // boundary conditions: after this subdomain's phase 2 (stream order), the phase 1 of its local senders (events) and,
  // with ranks, every remote sender's phase 1 (flags_finish made every stream wait for it)
  for (size_t di = 0; di < bc.size(); ++di) {
    if (!bc[di]) continue;
    CUDA_RUNTIME(cudaSetDevice(domains_[di].gpu()));
    if (!ranks)
      for (size_t sj : bcSenders_[di])
        if (sj != di) CUDA_RUNTIME(cudaStreamWaitEvent(streams_[di], phase1Done_[sj], 0));
    if (SB_OK != sb_bc_plan_launch(bc[di], streams_[di])) LOG_FATAL("exchange boundary conditions: " << sb_last_error());
  }
  nvtxRangePop();
}

void DistributedDomain::exchange_wait() {
  for (size_t di = 0; di < streams_.size(); ++di) {
    CUDA_RUNTIME(cudaSetDevice(streams_[di].device()));
    CUDA_RUNTIME(cudaStreamSynchronize(streams_[di]));
  }
}

void DistributedDomain::exchange() {
  nvtxRangePush("DD::exchange()");
#ifdef STENCIL_EXCHANGE_STATS
  MPI_Barrier(MPI_COMM_WORLD);
  const double start = MPI_Wtime();
#endif
  exchange_async();
  exchange_wait();
#ifdef STENCIL_EXCHANGE_STATS
  double elapsed = MPI_Wtime() - start, maxElapsed = -1;
  MPI_Reduce(&elapsed, &maxElapsed, 1, MPI_DOUBLE, MPI_MAX, 0, MPI_COMM_WORLD);
  if (0 == rank_) timeExchange_ += maxElapsed;
#endif
  nvtxRangePop();
}

void DistributedDomain::write_paraview(const std::string &prefix, bool zeroNaNs) {
  nvtxRangePush("write_paraview");
  for (size_t di = 0; di < domains_.size(); ++di) {
    const LocalDomain &dom = domains_[di];
    const std::string path = prefix + "_" + std::to_string(size_t(rank_) * domains_.size() + di) + ".txt";
    LOG_INFO("write paraview file " << path);
    std::vector<std::vector<unsigned char>> host;
    for (int64_t q = 0; q < dom.num_data(); ++q) host.push_back(dom.interior_to_host(size_t(q)));

    FILE *f = std::fopen(path.c_str(), "w");
    if (!f) {
      LOG_ERROR("unable to open \"" << path << "\" for writing");
      nvtxRangePop();
      return;
    }
    std::fprintf(f, "Z,Y,X");
    for (int64_t q = 0; q < dom.num_data(); ++q) {
      const std::string &nm = dom.dataName_[size_t(q)];
      std::fprintf(f, ",%s", nm.empty() ? ("data" + std::to_string(q)).c_str() : nm.c_str());
    }
    std::fprintf(f, "\n");
    const Dim3 sz = dom.size(), org = dom.origin();
    size_t cell = 0;
    for (int64_t lz = 0; lz < sz.z; ++lz)
      for (int64_t ly = 0; ly < sz.y; ++ly)
        for (int64_t lx = 0; lx < sz.x; ++lx, ++cell) {
          std::fprintf(f, "%ld,%ld,%ld", long(org.z + lz), long(org.y + ly), long(org.x + lx));
          for (int64_t q = 0; q < dom.num_data(); ++q) {
            if (8 == dom.elem_size(size_t(q))) {
              double v = reinterpret_cast<const double *>(host[size_t(q)].data())[cell];
              if (zeroNaNs && std::isnan(v)) v = 0.0;
              std::fprintf(f, ",%.17f", v);
            } else if (4 == dom.elem_size(size_t(q))) {
              float v = reinterpret_cast<const float *>(host[size_t(q)].data())[cell];
              if (zeroNaNs && std::isnan(v)) v = 0.0f;
              std::fprintf(f, ",%.9f", v);
            }
          }
          std::fprintf(f, "\n");
        }
    std::fclose(f);
  }
  nvtxRangePop();
}
