#pragma once
// What the placement code needs to know about the GPUs of a node.  On an NVSwitch node (H100 HGX) every pair of
// GPUs is equally close, so bandwidth() only distinguishes same-device / peer / no-peer (src/gpu_topology.cpp).

namespace gpu_topo {

/* Can device `src` load and store device `dst`'s memory directly?  (true for src == dst) */
bool peer(const int src, const int dst);

/* Turn that on (idempotent; remembers what has been enabled). */
void enable_peer(const int src, const int dst);

/* A unitless figure of merit for src -> dst transfers, larger is faster; placement compares ratios only. */
double bandwidth(int src, int dst);

} // namespace gpu_topo
