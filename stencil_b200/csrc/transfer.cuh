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

// Host: launch_* return the number of launches issued (0 on an empty box or an unknown element size).
int launch_restrict(const RestrictParams &p, int es, cudaStream_t stream);
int prolong_ctas_per_sm(int es);
int launch_prolong(const ProlongParams &p, int es, int grid, cudaStream_t stream);

} // namespace sb
