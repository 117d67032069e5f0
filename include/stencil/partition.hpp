#pragma once
// Placement: which (rank, local GPU) owns each subdomain of the partition.
//   Trivial          RankPartition, subdomains dealt to ranks/GPUs in linear order
//   NodeAware        NodePartition + a QAP per node matching halo traffic to GPU-GPU bandwidth
//   IntraNodeRandom  NodePartition, random GPU assignment inside each node (placement_intranoderandom.hpp)
// On an H100 NVSwitch node gpu_topo::bandwidth() is uniform for all distinct pairs, so the QAP cost is
// permutation invariant and NodeAware degenerates to the identity assignment (still solved, so the
// code path and its tests stay alive for non-uniform hosts).

#include <cassert>
#include <cmath>
#include <iostream>
#include <map>
#include <numeric>
#include <sstream>
#include <string>
#include <vector>

#include "stencil/dim3.hpp"
#include "stencil/gpu_topology.hpp"
#include "stencil/local_domain.cuh"
#include "stencil/logging.hpp"
#include "stencil/mat2d.hpp"
#include "stencil/mpi_topology.hpp"
#include "stencil/numeric.hpp"
#include "stencil/partition_core.hpp"
#include "stencil/qap.hpp"
#include "stencil/radius.hpp"

enum class PlacementStrategy {
  NodeAware,
  Trivial,
  IntraNodeRandom // grouped by node, random inside a node
};

class Placement {
public:
  virtual ~Placement() {}
  virtual Dim3 get_idx(const int rank, const int i) = 0;  // index of subdomain i of `rank`
  virtual int get_rank(const Dim3 &idx) = 0;              // owning rank
  virtual int get_subdomain_id(const Dim3 &idx) = 0;      // id within the owning rank
  virtual int get_cuda(const Dim3 &idx) = 0;              // CUDA device
  virtual Dim3 subdomain_size(const Dim3 &idx) = 0;
  virtual Dim3 subdomain_origin(const Dim3 &idx) = 0;
  virtual Dim3 dim() = 0; // exclusive upper bound of idx
};

namespace stencil {
namespace detail {

// idx <-> (rank, id, cuda) tables shared by the placements
class OwnerTable {
  std::map<Dim3, int> rank_, id_, cuda_;
  std::vector<std::vector<Dim3>> idx_; // [rank][id]

public:
  void assign(const Dim3 &idx, int rank, int id, int cuda) {
    assert(rank >= 0 && id >= 0);
    rank_[idx] = rank;
    id_[idx] = id;
    cuda_[idx] = cuda;
    if (idx_.size() <= size_t(rank)) idx_.resize(size_t(rank) + 1);
    if (idx_[rank].size() <= size_t(id)) idx_[rank].resize(size_t(id) + 1);
    idx_[rank][id] = idx;
  }
  Dim3 idx(int rank, int id) const {
    assert(size_t(rank) < idx_.size() && size_t(id) < idx_[rank].size());
    return idx_[rank][id];
  }
  int rank(const Dim3 &i) { return rank_[i]; }
  int id(const Dim3 &i) { return id_[i]; }
  int cuda(const Dim3 &i) { return cuda_[i]; }
};

} // namespace detail
} // namespace stencil

class Trivial : public Placement {
  RankPartition partition_;
  stencil::detail::OwnerTable owners_;

public:
  Dim3 get_idx(int rank, int domId) override { return owners_.idx(rank, domId); }
  int get_rank(const Dim3 &idx) override { return owners_.rank(idx); }
  int get_subdomain_id(const Dim3 &idx) override { return owners_.id(idx); }
  int get_cuda(const Dim3 &idx) override { return owners_.cuda(idx); }
  Dim3 subdomain_size(const Dim3 &idx) override { return partition_.subdomain_size(idx); }
  Dim3 subdomain_origin(const Dim3 &idx) override { return partition_.subdomain_origin(idx); }
  Dim3 dim() override { return partition_.dim(); }

  // collective: every rank contributes the CUDA devices it will drive
  Trivial(const Dim3 &size, MpiTopology &mpiTopo, const std::vector<int> &rankCudaIds) {
    MPI_Barrier(MPI_COMM_WORLD);
    const int mine = int(rankCudaIds.size());
    std::vector<int> counts(mpiTopo.size());
    MPI_Allgather(&mine, 1, MPI_INT, counts.data(), 1, MPI_INT, MPI_COMM_WORLD);
    const int total = std::accumulate(counts.begin(), counts.end(), 0);
    partition_ = RankPartition(size, total);

    std::vector<int> offsets(counts.size(), 0);
    for (size_t r = 1; r < counts.size(); ++r) offsets[r] = offsets[r - 1] + counts[r - 1];
    std::vector<int> cudaOf(total);
    MPI_Allgatherv(rankCudaIds.data(), mine, MPI_INT, cudaOf.data(), counts.data(), offsets.data(), MPI_INT, MPI_COMM_WORLD);

    // subdomain k (linear order) goes to the k-th contributed GPU
    int k = 0;
    for (int rank = 0; rank < int(counts.size()); ++rank) {
      for (int id = 0; id < counts[rank]; ++id, ++k) {
        owners_.assign(partition_.dimensionize(k), rank, id, cudaOf[k]);
      }
    }
    MPI_Barrier(MPI_COMM_WORLD);
  }
};

inline double avg(const std::vector<double> &x) {
  assert(!x.empty());
  return std::accumulate(x.begin(), x.end(), 0.0) / double(x.size());
}

// population standard deviation
inline double cssd(const std::vector<double> &x) {
  const double m = avg(x);
  double acc = 0;
  for (double e : x) acc += (e - m) * (e - m);
  return std::sqrt(acc / double(x.size()));
}

// sample correlation coefficient (1 when both series are constant)
inline double scc(const std::vector<double> &x, const std::vector<double> &y) {
  assert(x.size() == y.size());
  const double mx = avg(x), my = avg(y);
  double num = 0;
  for (size_t i = 0; i < x.size(); ++i) num += (x[i] - mx) * (y[i] - my);
  const double den = double(x.size() - 1) * cssd(x) * cssd(y);
  if (0 == num && 0 == den) return 1;
  assert(0 != den);
  return num / den;
}

class NodeAware : public Placement {
  NodePartition partition_;
  stencil::detail::OwnerTable owners_;

public:
  Dim3 get_idx(int rank, int domId) override { return owners_.idx(rank, domId); }
  int get_rank(const Dim3 &idx) override { return owners_.rank(idx); }
  int get_subdomain_id(const Dim3 &idx) override { return owners_.id(idx); }
  int get_cuda(const Dim3 &idx) override { return owners_.cuda(idx); }
  Dim3 subdomain_size(const Dim3 &idx) override { return partition_.subdomain_size(idx); }
  Dim3 subdomain_origin(const Dim3 &idx) override { return partition_.subdomain_origin(idx); }
  Dim3 dim() override { return partition_.dim(); }

  // collective.  Assumes every rank drives the same number of GPUs and every node hosts the same
  // number of ranks.
  NodeAware(const Dim3 &size, MpiTopology &mpiTopo, Radius radius, const std::vector<int> &rankCudaIds) {
    MPI_Barrier(MPI_COMM_WORLD);
    const int gpusPerRank = int(rankCudaIds.size());
    const int ranksPerNode = mpiTopo.colocated_size();
    const int gpusPerNode = gpusPerRank * ranksPerNode;
    const int numNodes = mpiTopo.size() / ranksPerNode;
    const int numSubdomains = numNodes * gpusPerNode;
    partition_ = NodePartition(size, radius, numNodes, gpusPerNode);
    if (0 == mpi::world_rank()) {
      LOG_INFO("NodeAware: " << partition_.sys_dim() << "x" << partition_.node_dim());
    }

    // node number of every rank, numbered in order of first appearance of the processor name
    char name[MPI_MAX_PROCESSOR_NAME] = {0};
    int nameLen = 0;
    MPI_Get_processor_name(name, &nameLen);
    std::vector<char> names;
    if (0 == mpiTopo.rank()) names.resize(size_t(MPI_MAX_PROCESSOR_NAME) * mpiTopo.size());
    MPI_Gather(name, MPI_MAX_PROCESSOR_NAME, MPI_CHAR, names.data(), MPI_MAX_PROCESSOR_NAME, MPI_CHAR, 0, MPI_COMM_WORLD);

    std::vector<int> globalCudaIds(numSubdomains);
    MPI_Allgather(rankCudaIds.data(), gpusPerRank, MPI_INT, globalCudaIds.data(), gpusPerRank, MPI_INT, mpiTopo.comm());

    std::vector<int> rankOf(numSubdomains), idOf(numSubdomains), cudaOf(numSubdomains);
    if (0 == mpiTopo.rank()) {
      std::map<std::string, int> nodeOfName;
      std::vector<std::vector<int>> nodeRanks;
      for (int r = 0; r < mpiTopo.size(); ++r) {
        const std::string nm(names.data() + size_t(r) * MPI_MAX_PROCESSOR_NAME);
        auto it = nodeOfName.find(nm);
        if (it == nodeOfName.end()) {
          it = nodeOfName.emplace(nm, int(nodeRanks.size())).first;
          nodeRanks.emplace_back();
        }
        nodeRanks[it->second].push_back(r);
      }

      const Dim3 nodeDim = partition_.node_dim();
      const Dim3 globalDim = partition_.dim();
      for (int node = 0; node < numNodes; ++node) {
        const Dim3 sysIdx = partition_.sys_idx(node);
        const std::vector<int> &ranks = nodeRanks[node];
        assert(int(ranks.size()) == ranksPerNode);

        // component c = (rank slot, gpu slot) of this node
        auto cuda_of_component = [&](int c) { return globalCudaIds[ranks[c / gpusPerRank] * gpusPerRank + c % gpusPerRank]; };
        Mat2D<double> bw(gpusPerNode, gpusPerNode, 0.0);
        for (int a = 0; a < gpusPerNode; ++a)
          for (int b = 0; b < gpusPerNode; ++b) bw[a][b] = gpu_topo::bandwidth(cuda_of_component(a), cuda_of_component(b));

        // halo elements exchanged between the subdomains of this node (periodic adjacency)
        Mat2D<double> traffic(gpusPerNode, gpusPerNode, 0.0);
        for (int i = 0; i < gpusPerNode; ++i) {
          const Dim3 src = sysIdx * nodeDim + partition_.node_idx(i);
          for (int j = 0; j < gpusPerNode; ++j) {
            const Dim3 dst = sysIdx * nodeDim + partition_.node_idx(j);
            Dim3 dir = dst - src;
            for (int a = 0; a < 3; ++a) {
              if (dir[a] != 0 && dir[a] == globalDim[a] - 1) dir[a] = -1;
              if (dir[a] != 0 && dir[a] == 1 - globalDim[a]) dir[a] = 1;
            }
            if (Dim3(0, 0, 0) == dir || dir.any_gt(1) || dir.any_lt(-1)) continue;
            traffic[i][j] = double(LocalDomain::halo_extent(dir, partition_.subdomain_size(src), radius).flatten());
          }
        }

        Mat2D<double> distance = make_reciprocal(bw);
        const std::vector<size_t> component = qap::solve(traffic, distance);
        for (int id = 0; id < gpusPerNode; ++id) {
          const int c = int(component[id]);
          const int rank = ranks[c / gpusPerRank];
          const size_t gi = size_t(node) * gpusPerNode + id;
          rankOf[gi] = rank;
          idOf[gi] = c % gpusPerRank;
          cudaOf[gi] = globalCudaIds[rank * gpusPerRank + c % gpusPerRank];
        }
      }
    }
    MPI_Bcast(rankOf.data(), int(rankOf.size()), MPI_INT, 0, MPI_COMM_WORLD);
    MPI_Bcast(idOf.data(), int(idOf.size()), MPI_INT, 0, MPI_COMM_WORLD);
    MPI_Bcast(cudaOf.data(), int(cudaOf.size()), MPI_INT, 0, MPI_COMM_WORLD);

    // global id = node * gpusPerNode + in-node id
    for (size_t gi = 0; gi < rankOf.size(); ++gi) {
      const Dim3 idx = partition_.sys_idx(int64_t(gi / gpusPerNode)) * partition_.node_dim() + partition_.node_idx(int64_t(gi % gpusPerNode));
      owners_.assign(idx, rankOf[gi], idOf[gi], cudaOf[gi]);
    }
  }
};
