// Multigrid transfers between a cell-centred grid and its coarsening by 2 (include/stencil_b200.h, sb_transfer_*;
// DESIGN.md section 2.10).
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace sb {

// restriction: a CTA of kRestrictX x kRestrictY threads, one coarse cell each (a warp reads 64 contiguous fine elements
// per row); prolongation: a CTA owns kProlongX x kProlongY coarse cells of a z chunk and writes their 2 x 2 x 2 children
constexpr int kRestrictX = 32, kRestrictY = 8;
constexpr int kProlongX = 32, kProlongY = 8, kProlongThreads = kProlongX * kProlongY;
constexpr int kProlongSW = kProlongX + 2, kProlongPlane = kProlongSW * (kProlongY + 2); // a ring slot: the tile and its ring

// Allocation coordinates throughout: element (x, y, z) of an allocation at byte (z * ysize + y) * pitch + x * es.
struct RestrictParams {
  char *dst;                  // coarse
  const char *src;            // fine
  long long dpitch, dslice;   // dst
  long long spitch, sslice;   // src
  int lo[3], ext[3];          // the coarse box in dst's allocation coordinates
  int flo[3];                 // the fine cell 2 * (global lo) in src's allocation coordinates
};
static_assert(sizeof(RestrictParams) <= 4096, "the restriction's parameters fit the classic 4 KB limit");

struct ProlongParams {
  char *dst;                  // fine
  const char *aux;            // fine, dst's pitch and rows; NULL: dst = P e
  const char *src;            // coarse
  long long dpitch, dslice;   // dst and aux
  long long spitch, sslice;   // src
  int lo[3], ext[3];          // the fine box in dst's allocation coordinates
  int off[3];                 // child d of the parent at src allocation coordinate c sits at dst coordinate 2c + d + off
  int plo[3], pext[3];        // the parents' box in src's allocation coordinates
  int rlo[3], rhi[3];         // the coarse cells the rule reads, [rlo, rhi), in src's allocation coordinates
  int zchunk, tiles_x, tiles_y;
};
static_assert(sizeof(ProlongParams) <= 4096, "the prolongation's parameters fit the classic 4 KB limit");

// Fused residual-restriction (sb_transfer_oplan_create): a plain op of reach <= 1 evaluated on the eight fine cells of
// each coarse cell and restricted, the fine values never stored.  Weights already rounded to T; off[t]: term t's offset.
constexpr int kRopMaxTerms = 64;
constexpr int kRopMaxBoxes = 16; // thin boxes per cell-kernel launch
// tile kernel: a CTA of kRestrictX x kRestrictY threads owns as many coarse cells of a z chunk; the fine planes of its
// 2kRestrictX x 2kRestrictY footprint and a one-cell ring pass through a 3-slot shared ring
constexpr int kRopSW = 2 * kRestrictX + 2, kRopPlane = kRopSW * (2 * kRestrictY + 2);
struct RopCommon {
  char *dst;                  // coarse
  const char *src, *aux;      // fine; aux shares src's pitch and rows (NULL: no aux term)
  long long dpitch, dslice;   // dst
  long long spitch, sslice;   // src and aux
  int n;
  signed char source[kRopMaxTerms];
  signed char off[kRopMaxTerms][3];
  double w[kRopMaxTerms];     // T(w) for T = double
  float wf[kRopMaxTerms];     // T(w) for T = float
};
struct RopTileParams {
  RopCommon c;
  int lo[3], ext[3];          // the coarse box in dst's allocation coordinates
  int flo[3];                 // the fine cell 2 * (global lo) in src's allocation coordinates
  int rlo[3], rhi[3];         // the fine cells the plan checked, [flo - 1, flo + 2 ext + 1), in src's allocation coordinates
  int zchunk, tiles_x, tiles_y;
  int toff[3][kRopMaxTerms];  // shared-memory element offset of term t's src cell from the ring base, relative to the
                              // cell's place in a slot, while the centre plane occupies ring slot c (precomputed by the plan)
};
static_assert(sizeof(RopTileParams) <= 4096, "the fused restriction's tile parameters fit the classic 4 KB limit");
struct RopCellParams {
  RopCommon c;
  int n;                      // boxes
  int lo[kRopMaxBoxes][3], ext[kRopMaxBoxes][3], flo[kRopMaxBoxes][3];
  long long first[kRopMaxBoxes + 1];
};
static_assert(sizeof(RopCellParams) <= 4096, "the fused restriction's cell parameters fit the classic 4 KB limit");
// With coefficient terms (sb_transfer_voplan_create): term t's factor is T(w) * C_f(p + coff[t]), f = cfield[t] (-1:
// none); the fields share src's pitch and rows.  The tile kernel reads them through the read-only path at the byte
// offset cgoff[t] from the fine cell.
constexpr int kRopMaxCoefs = 4;
struct RopVTileParams : RopTileParams {
  const char *coef[kRopMaxCoefs];
  signed char cfield[kRopMaxTerms];
  long long cgoff[kRopMaxTerms];
};
static_assert(sizeof(RopVTileParams) <= 4096, "the coefficient fused restriction's tile parameters fit the classic 4 KB limit");
struct RopVCellParams : RopCellParams {
  const char *coef[kRopMaxCoefs];
  signed char cfield[kRopMaxTerms];
  signed char coff[kRopMaxTerms][3];
};
static_assert(sizeof(RopVCellParams) <= 4096, "the coefficient fused restriction's cell parameters fit the classic 4 KB limit");

// Host: launch_* return the number of launches issued (0 on an empty box or an unknown element size).
int launch_restrict(const RestrictParams &p, int es, cudaStream_t stream);
// face-coefficient restriction (sb_transfer_fplan_create) of the faces normal to axis 0, 1 or 2: RestrictParams' box
// and allocations, the same grid
int launch_face_restrict(const RestrictParams &p, int es, int axis, cudaStream_t stream);
int prolong_ctas_per_sm(int es);
int launch_prolong(const ProlongParams &p, int es, int grid, cudaStream_t stream);
int rop_tile_ctas_per_sm(int es, bool coef = false);
int launch_rop_tile(const RopTileParams &p, int es, int grid, cudaStream_t stream);
int launch_rop_cells(const RopCellParams &p, int es, int grid, cudaStream_t stream);
int launch_rop_vcells(const RopVCellParams &p, int es, int grid, cudaStream_t stream);
int launch_rop_vtile(const RopVTileParams &p, int es, int grid, cudaStream_t stream);

} // namespace sb
