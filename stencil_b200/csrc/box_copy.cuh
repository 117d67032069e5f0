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

// Opt-in (SB_TMA=1) TMA tile kinds for wide segments.  Constraints (probed with scripts/exp/tma_probe3.cu):
// a box's global START address must be 16-byte aligned (element-granular coordinates do NOT absorb an 8-byte row
// phase: UTMALDG/UTMASTG raise "illegal instruction"), and its shared-memory address must be 128-byte aligned.
//   kind 1  both sides TMA-legal (16-byte aligned base, strides and box start, e.g. r=2 FP64): cp.async.bulk.tensor
//           global -> shared (mbarrier complete_tx) then shared -> global (bulk_group), ONE elected thread per CTA,
//           4-stage shared-memory ring, a row cut into chunks of `bx` elements (box = bx x 1 x 1).
//   kind 2  source rows start off a 16-byte boundary (r=1 FP64): aligned-down TMA load, vector stores by all threads.
// Result on the B200 they were written on (not re-timed on the H100): for halo-sized messages (2-4 MB, <1 tile per
// SM) both kinds were slower than the LSU path below, which is why they are off by default.
constexpr int kMaxTmaMaps = 16;

// The CUtensorMap descriptors travel as a __grid_constant__ kernel parameter (the documented-safe home
// of a host-encoded tensor map); 128 bytes each, opaque here so that this header needs no <cuda.h>.
struct alignas(64) TmaMaps {
  unsigned long long m[kMaxTmaMaps][16];
};

struct TmaSeg {
  int smap; // index into TmaMaps: tensor map of the source allocation
  int dmap;
  int sx0, sy0, sz0; // region start inside the source tensor (elements / rows / planes)
  int dx0, dy0, dz0;
  unsigned bx;             // chunk width (elements)
  unsigned chunks_per_row; // ext.x / bx
  unsigned chunk_bytes;
  unsigned ny, nz;
  unsigned ny_shift;
  unsigned long long ny_magic;
  // kind 2 ("TMA load, vector store"): the halo rows of an FP64 r=1 subdomain start 8 bytes into a
  // 16-byte vector, and a TMA box must START on a 16-byte boundary (measured: UTMALDG raises an illegal
  // instruction otherwise).  The load therefore begins `pre` elements early (box = bxa elements, a
  // multiple of 16 bytes covering pre + bx), the payload sits `pre * es` bytes into each shared-memory
  // chunk, and all threads of the CTA store it to the destination -- 128-bit stores when source and
  // destination rows have the same phase (peeling the first / last element), else the widest aligned.
  char *dst;              // destination of the box's first payload byte
  long long dst_pitch, dst_slice;
  unsigned pre;           // elements loaded before the payload in every chunk
  unsigned bxa;           // box width (elements) of the source map
  unsigned cstride;       // bytes a chunk occupies in the ring (multiple of 128)
  unsigned es;            // element size
  unsigned vec;           // store width when the phases differ
  unsigned same_phase;    // 1: (dst - pre*es) is 16-byte aligned for every row
};

struct Tile {
  unsigned seg; // index into the Seg table (kind 0) or the TmaSeg table (kinds 1, 2)
  unsigned row0;
  unsigned nrows;
  unsigned kind;
};

constexpr int kCopyThreads = 256;
constexpr unsigned kTileBytes = 16384;

void launch_box_copy(const Seg *segs_dev, const TmaSeg *tsegs_dev, const TmaMaps *maps_host, const Tile *tiles_dev, unsigned ntiles, int grid,
                     cudaStream_t stream);
void launch_box_copy_single(const Seg &seg, cudaStream_t stream);
unsigned rows_per_tile_for(unsigned row_bytes); // tile height for a segment
void preload_box_copy_kernels();

} // namespace sb
