#pragma once
// The exchange plan: which boxes a subdomain sends to which neighbour, and how the thin ones are packed into the
// receiver's staging buffer.  A sender and a receiver (possibly in different processes) derive both independently, so
// this header is the one definition of each rule; DistributedDomain (C++) and the C ABI (sb_exchange_messages,
// sb_staging_layout, used by the Python host) both call it.  Host-only integer math.

#include <cstdint>
#include <vector>

#include "stencil/dim3.hpp"
#include "stencil/geometry.hpp"
#include "stencil/radius.hpp"
#include "stencil/topology.hpp"

namespace stencil {

// One halo message: the outermost compute cells of `srcIdx` on side `dir` (at srcPos) go to the ghost cells of
// `dstIdx` on side -dir (at dstPos), `ext` elements.
struct Message {
  Dim3 srcIdx, dstIdx, dir, srcPos, dstPos, ext;
};

// Every message subdomain `src` sends, in the canonical order both ends rely on: direction z, then y, then x, each
// ascending.  A direction is skipped when the neighbour's stencil does not reach back (radius(-dir) == 0), when the
// step crosses a wall, or when the box is empty.  sizeOf(idx) gives the compute size of subdomain idx.
template <typename SizeOf>
std::vector<Message> messages_from(const Dim3 &src, const Topology &topology, const Radius &radius, const SizeOf &sizeOf) {
  std::vector<Message> out;
  const Dim3 srcSz = sizeOf(src);
  for (int z = -1; z <= 1; ++z)
    for (int y = -1; y <= 1; ++y)
      for (int x = -1; x <= 1; ++x) {
        const Dim3 dir(x, y, z);
        if (Dim3(0, 0, 0) == dir) continue;
        if (0 == radius.dir(dir * -1)) continue;
        const Topology::OptionalNeighbor nbr = topology.get_neighbor(src, dir);
        if (!nbr.exists) continue;
        const Dim3 dstSz = sizeOf(nbr.index);
        const Dim3 ext = geom::halo_extent(dir * -1, dstSz, radius);
        if (0 == ext.flatten()) continue;
        out.push_back(Message{src, nbr.index, dir, geom::halo_pos(dir, srcSz, radius, false),
                              geom::halo_pos(dir * -1, dstSz, radius, true), ext});
      }
  return out;
}

// Rows shorter than this many bytes bound for another GPU are staged: storing them straight into the peer's ghost
// cells costs one small NVLink transaction per row, so the sender packs them into one dense buffer in the receiver's
// memory and the receiver scatters them locally.
constexpr int64_t kStageMaxRowBytes = 64;

// Quantity q of messagesFromSrc[msg] is packed at byte `offset` of the (src -> dst) staging buffer.
struct Staged {
  size_t msg;
  int64_t q, offset;
};

// A subset of a domain's quantities: bit q set = quantity q takes part.  An exchange of a subset moves only the boxes
// and fills only the BC regions of those quantities; kAllQuantities is the full exchange.  A subset names quantities
// 0..63 only (a domain with more quantities exchanges them all, or a subset of the first 64).
using QuantitySet = uint64_t;
constexpr QuantitySet kAllQuantities = ~QuantitySet(0);
inline bool in_set(QuantitySet set, size_t q) { return q >= 64 ? set == kAllQuantities : ((set >> q) & 1u) != 0; }

// The layout of the (src -> dst) staging buffer: the messages of messagesFromSrc (= messages_from(src, ...)) bound for
// dst in their order, the quantities of each in order; a (message, quantity) pair is staged when a row of it is
// shorter than kStageMaxRowBytes.  Each entry starts at a 16-byte boundary; *total is the end of the last one (0 when
// nothing is staged).  Whether staging applies at all (src and dst on different GPUs) is the caller's decision.
// quantities: only the entries of those quantities are returned, at the offsets the full layout gives them, and *total
// stays the full layout's, so an exchange of any subset uses the full exchange's staging buffers as they are.
inline std::vector<Staged> staging_layout(const std::vector<Message> &messagesFromSrc, const Dim3 &dst,
                                          const std::vector<int64_t> &elemSizes, int64_t *total,
                                          QuantitySet quantities = kAllQuantities) {
  std::vector<Staged> out;
  int64_t off = 0;
  for (size_t i = 0; i < messagesFromSrc.size(); ++i) {
    const Message &m = messagesFromSrc[i];
    if (!(m.dstIdx == dst)) continue;
    for (size_t q = 0; q < elemSizes.size(); ++q) {
      const int64_t es = elemSizes[q];
      if (m.ext.x * es >= kStageMaxRowBytes) continue;
      off = (off + 15) & ~int64_t(15);
      if (in_set(quantities, q)) out.push_back(Staged{i, int64_t(q), off});
      off += es * int64_t(m.ext.flatten());
    }
  }
  *total = off;
  return out;
}

} // namespace stencil
