// Linear stencil operators, constant and variable coefficients (include/stencil_b200.h, sb_stencil_*; DESIGN.md
// section 2.7).
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

// Coefficient fields (sb_stencil_vplan_create).  The plan numbers the fields the op references 0 .. nf - 1 (in order of
// their C ABI index).  In the tile kernel each one has a ring of kOpCoefSlots planes of op_tile_plane(1) elements after
// the src ring, filled by cp.async one plane ahead (slot of plane z: (z - z0 + 1) % kOpCoefSlots), each field's window
// limited to its own reach crm / crp.  cfield[t]: the field of term t, or -1.
constexpr int kOpMaxCoefs = 4;
constexpr int kOpCoefSlots = 4; // planes z - 1 .. z + 1 being read, and z + 2 landing
struct OpCoefTile {
  const char *coef[kOpMaxCoefs];
  int nf;
  int crm[kOpMaxCoefs][3], crp[kOpMaxCoefs][3];
  signed char cfield[kOpMaxTerms];
  short coff[kOpCoefSlots][kOpMaxTerms]; // shared-memory element offset of term t's coefficient from the cell's own
                                         // position in field 0's ring, while the centre plane sits in slot c
};
struct OpVTileParams : OpTileParams {
  OpCoefTile k;
};
static_assert(sizeof(OpVTileParams) <= 4096, "the tile kernel's parameters fit the classic 4 KB limit");

// the cell kernel's coefficient reads: field cfield[t] (-1: none) at byte offset cgoff[t] from the cell
struct OpVCellParams : OpCellParams {
  const char *coef[kOpMaxCoefs];
  signed char cfield[kOpMaxTerms];
  long long cgoff[kOpMaxTerms];
};

// Coloured application (sb_stencil_cplan_create; DESIGN.md section 2.9): only the cells of colour c under the colouring
// m (1, 2 or 8) are written.  par[a]: the parity of the global coordinate of allocation element 0 on axis a, so a cell's
// colour follows from its allocation coordinates.  m = 1 launches the uncoloured kernels, which take the base parameters.
struct OpColour {
  int m, c;
  int par[3];
};
struct OpCTileParams : OpVTileParams {
  OpColour col;
};
static_assert(sizeof(OpCTileParams) <= 4096, "the coloured tile kernel's parameters fit the classic 4 KB limit");
struct OpCCellParams : OpVCellParams {
  OpColour col;
};

// Diagonal relaxation (sb_stencil_dplan_create; DESIGN.md section 2.12): the op is A (src terms only), aux holds f, and
// a cell of the colour gets u + T(omega) * ((f - A u) / d), d the sum of the factors T(w) (times C) of the terms at
// offset 0 (bit t of centre: term t is one).  The diagonal kernels are the coloured ones with this flag (DIAG, a
// compile-time switch); with m = 1 they write every cell of the boxes.
struct OpDiag {
  int on;
  unsigned long long centre;
  double omega;
  float omegaf;
};
struct OpDTileParams : OpCTileParams {
  OpDiag dg;
};
static_assert(sizeof(OpDTileParams) <= 4096, "the diagonal tile kernel's parameters fit the classic 4 KB limit");
struct OpDCellParams : OpCCellParams {
  OpDiag dg;
};

// Host: dynamic shared memory of the tile kernel; one-time attribute setup; the number of CTAs of the tile kernel that
// fit on one SM (0 on error).  launch_* return the number of launches issued.  nf: coefficient fields (0: the plain
// kernel); col: the coloured kernel; diag: the diagonal one (p.dg.on in the launches).
size_t op_tile_smem(int R, int es, int nf = 0);
int op_tile_prepare(int R, int es, int device, int nf = 0, bool col = false, bool diag = false);
int launch_op_tile(const OpDTileParams &p, int R, int es, int grid, cudaStream_t stream);
int launch_op_cells(const OpDCellParams &p, int es, bool has_coef, int grid, cudaStream_t stream);

} // namespace sb
