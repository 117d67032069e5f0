// Linear stencil systems: several outputs over several inputs in one launch (include/stencil_b200.h, sb_stencil_sys_*;
// DESIGN.md section 2.8).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "stencil_op.cuh"

namespace sb {

constexpr int kSysMaxInputs = 8, kSysMaxOutputs = 4, kSysMaxTerms = 128;

// Both kernels see the terms sorted by output (stable): output j owns terms [first[j], first[j + 1]).  Per term: the
// input it reads (in), the input it reads as a coefficient (cin, -1: none) and the weight rounded to each type.
struct SysTerms {
  char *out[kSysMaxOutputs];
  long long pitch, slice;
  int n, nout;
  int first[kSysMaxOutputs + 1];
  signed char in[kSysMaxTerms], cin[kSysMaxTerms];
  double w[kSysMaxTerms];
  float wf[kSysMaxTerms];
};

// z-marching tile kernel over one box [lo, lo + ext) (allocation coordinates); a CTA owns kOpTileX x kOpTileY cells and
// a z chunk.  Every input the system reads has its own ring of ns[r] = rm[r][2] + rp[r][2] + 2 planes of kOpTileY +
// rm[r][1] + rp[r][1] rows of sw elements at shared element base[r], filled by cp.async one plane ahead, each plane's
// window cut to that input's reach (rm / rp below / above per axis).  Element x of a ring row sits at column
// x - x0 + rm[r][0] + shift[r]: shift[r] puts the 16-byte chunks of the allocation on 16-byte shared addresses, so
// vec[r] inputs (pitch a multiple of 16 bytes) are copied in 16-byte pieces wherever a chunk lies inside the window, and
// elements one by one at the window's two ends (no cell outside the window is read) or where the pitch gives rows of two
// phases.
// Per term: oz / coz the z offset of its reads, inpl / cinpl the rest of their shared offset from the cell's own slot
// position wy * sw + lane.  in / cin of SysTerms index the rings here.
struct SysTileParams {
  SysTerms c;
  const char *in[kSysMaxInputs];
  int nr; // rings (inputs the system reads)
  int rm[kSysMaxInputs][3], rp[kSysMaxInputs][3];
  int ns[kSysMaxInputs], base[kSysMaxInputs], shift[kSysMaxInputs], vec[kSysMaxInputs];
  int lo[3], ext[3];
  int zchunk, tiles_x, tiles_y, sw;
  signed char oz[kSysMaxTerms], coz[kSysMaxTerms];
  int inpl[kSysMaxTerms], cinpl[kSysMaxTerms];
};
static_assert(sizeof(SysTileParams) <= 4096, "the system tile kernel's parameters fit the classic 4 KB limit");

// one thread per cell over up to kOpMaxBoxes thin boxes; o / co: the offsets of a term's reads
struct SysCellParams {
  SysTerms c;
  const char *in[kSysMaxInputs];
  signed char o[kSysMaxTerms][3], co[kSysMaxTerms][3];
  int nb;
  int lo[kOpMaxBoxes][3], ext[kOpMaxBoxes][3];
  long long first[kOpMaxBoxes + 1];
};
static_assert(sizeof(SysCellParams) <= 4096, "the system cell kernel's parameters fit the classic 4 KB limit");

// shared memory of the tile kernel ahead of the rings: each term's read offsets for two planes
constexpr int kSysTableBytes = 2 * 2 * kSysMaxTerms * int(sizeof(int));

// Host: one-time attribute setup and the number of tile CTAs of `smem` bytes that fit on one SM (0 on error); launch_*
// return the number of launches issued.
int sys_tile_prepare(int es, int device, size_t smem);
int launch_sys_tile(const SysTileParams &p, int es, size_t smem, int grid, cudaStream_t stream);
int launch_sys_cells(const SysCellParams &p, int es, int grid, cudaStream_t stream);

} // namespace sb
