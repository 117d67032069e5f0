// Constant-coefficient linear stencil operators (include/stencil_b200.h, sb_stencil_*; DESIGN.md section 2.7).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace sb {

constexpr int kOpMaxTerms = 64;
constexpr int kOpMaxReach = 4;
// tile kernel: a CTA of 256 threads owns kOpTileX x kOpTileY cells of a plane (8 warps, one row each, two cells per lane)
constexpr int kOpTileX = 64, kOpTileY = 8, kOpThreads = 256;
constexpr int kOpMaxBoxes = 16; // thin boxes per cell-kernel launch

// What both kernels share.  dst / src / aux are allocation bases (element (0,0,0)); the three share pitch and slice.
struct OpCommon {
  char *dst;
  const char *src;
  const char *aux;
  long long pitch, slice;
  int n;         // terms
  int has_aux;   // any term on aux
  signed char source[kOpMaxTerms];
  double w[kOpMaxTerms];   // T(w) for T = double
  float wf[kOpMaxTerms];   // T(w) for T = float
};

// z-marching tile kernel over one box [lo, lo + ext) (allocation coordinates).  The halo'd planes of a tile live in a ring
// of 2R + 1 slots of (kOpTileX + 2R) x (kOpTileY + 2R) elements.  toff[c][t]: the shared-memory element offset of term t,
// relative to the cell's own position in the tile, while the centre plane occupies ring slot c (precomputed by the plan).
struct OpTileParams {
  OpCommon c;
  const char *src_end; // end of the src allocation: a 16-byte load never reaches it
  int lo[3], ext[3];
  int rm[3], rp[3];    // reach of the op below / above a cell on each axis
  int zchunk, tiles_x, tiles_y;
  int toff[2 * kOpMaxReach + 1][kOpMaxTerms];
};

// one thread per cell over up to kOpMaxBoxes thin boxes; goff[t]: byte offset of term t from the cell
struct OpCellParams {
  OpCommon c;
  long long goff[kOpMaxTerms];
  int n;
  int lo[kOpMaxBoxes][3], ext[kOpMaxBoxes][3];
  long long first[kOpMaxBoxes + 1];
};

// shared-memory row width / plane size of the tile kernel for reach R
__host__ __device__ constexpr int op_tile_sw(int R) { return kOpTileX + 2 * R; }
__host__ __device__ constexpr int op_tile_plane(int R) { return (kOpTileX + 2 * R) * (kOpTileY + 2 * R); }

// Host: dynamic shared memory of the tile kernel; one-time attribute setup; the number of CTAs of the tile kernel that
// fit on one SM (0 on error).  launch_* return the number of launches issued.
size_t op_tile_smem(int R, int es);
int op_tile_prepare(int R, int es, int device);
int launch_op_tile(const OpTileParams &p, int R, int es, int grid, cudaStream_t stream);
int launch_op_cells(const OpCellParams &p, int es, int grid, cudaStream_t stream);

} // namespace sb
