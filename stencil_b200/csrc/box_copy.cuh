// Box-copy engine: strided 3-D box -> strided 3-D box, any number of boxes per launch.
//
// One kernel serves every data-movement role of the reference's halo path
//   pack      grid_pack / dev_packer_pack_domain      reference src/pack_kernel.cu:3-59, src/packer.cu:10-26
//   unpack    grid_unpack / dev_unpacker_unpack_domain           src/pack_kernel.cu:61-108, src/packer.cu:28-44
//   translate translate_grid / multi_translate                   src/copy.cu:34-85
//   exchange  PeerCopySender's pack -> cudaMemcpyPeerAsync -> unpack   include/stencil/tx_cuda.cuh:117-180
// by treating each (direction, quantity) message as a "segment": rows of `row_bytes` contiguous
// bytes, `ny` rows per plane, `nz` planes, with independent source and destination strides.  The
// destination may be a dense buffer (pack), a local allocation (translate/unpack) or a peer GPU's
// ghost cells mapped over NVLink (fused exchange: no send or receive buffer ever touches HBM).
//
// Work decomposition (sm_90a, 132 SMs on an H100): each segment is cut into tiles of consecutive rows sized
// to ~16 KiB of payload; a persistent grid (a multiple of the SM count) walks the tile table.
// Inside a tile a power-of-two group of lanes owns one row, so a 4 KiB z-face row is moved by a
// full warp with 16-byte accesses (512 B per warp instruction) while an 8-byte x-face "row" is
// one lane's single access and a warp covers 32 rows at once.  Four independent accesses are in
// flight per thread before the first store.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace sb {

struct Seg {
  const char *src; // address of the box's first byte
  char *dst;
  long long src_pitch, src_slice; // bytes between rows / planes
  long long dst_pitch, dst_slice;
  unsigned row_bytes;
  unsigned ny, nz;
  unsigned vec;      // access width in bytes (1,2,4,8,16): divides every address and stride
  unsigned lg_group; // log2 of lanes cooperating on one row
  unsigned ny_shift; // magic division by ny: q = (n * ny_magic) >> ny_shift, exact for n < 2^24
  unsigned long long ny_magic;
};

struct Tile {
  unsigned seg; // index into the Seg table
  unsigned row0;
  unsigned nrows;
};

constexpr int kCopyThreads = 256;
constexpr unsigned kTileBytes = 16384;
constexpr int kCopyCtasPerSm = 8; // persistent grid of a copy plan: CTAs per SM

void launch_box_copy(const Seg *segs_dev, const Tile *tiles_dev, unsigned ntiles, int grid, cudaStream_t stream);
void launch_box_copy_single(const Seg &seg, cudaStream_t stream);
unsigned rows_per_tile_for(unsigned row_bytes); // tile height for a segment
void preload_box_copy_kernels();

} // namespace sb
