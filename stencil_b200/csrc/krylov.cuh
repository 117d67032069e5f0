// Krylov vector kernels (sb_krylov_plan_* of include/stencil_b200.h; DESIGN.md section 2.13): one elementwise pass over a
// box with each buffer read once and each output written once, with up to two exact dot products on the way.
//
// The box is cut into tiles of whole x rows.  A persistent grid walks the tile table: inside a tile a power-of-two group
// of G lanes owns a row and reads it with 16-byte vectors when every buffer has the same address modulo 16 (after
// peeling a head and a tail of at most 3 cells per row), four vectors per buffer in flight per lane.  Dot terms go to the
// exact accumulator of exact_acc.cuh; each tile writes one KryPartial, and a combine launch (one block per dot) adds the
// tiles' digit counters, carries them into an sb_exact_sum and merges min / max by sb_reduce_exact_combine's
// order-independent rule.  Exact sums do not depend on the order of their terms, so the result bits are a function of
// the multiset of per-cell terms alone, whatever the tiling, the grid or the allocation layout.
#pragma once

#include <cuda_runtime.h>

#include "reduce.cuh"
#include "stencil_b200.h"

namespace sb {

// kernel modes: the public SB_KRYLOV_DOT with one or two pairs, SB_KRYLOV_XPBY with T(s) = +-0 (a copy) or not, UPDATE
// without and with c, BICG_P (DESIGN.md section 2.14)
enum KryMode { kKryDot1 = 0, kKryDot2 = 1, kKryCopy = 2, kKryXpby = 3, kKryUpdate = 4, kKryBicgP = 5, kKryUpdateC = 6 };
constexpr int kKryModes = 7;

struct KryParams {
  char *buf[5];           // address of the box's cell lo in each buffer: DOT a, b[, c]; XPBY p, z; UPDATE x, p, r, q[, c];
                          // BICG_P p, r, v
  long long pitch, slice; // bytes between rows / planes (the same for every buffer)
  int ext[3];             // box extent
  int lg_group;           // log2 of the lanes that share a row
  unsigned rows_per_tile, ntiles;
  long long count;        // cells of the box
};

struct KryPartial {
  double min[2], max[2];
  long long digit[2][kExDigits]; // per dot: uncarried counters of 32-bit digits
  unsigned flags[2];
  unsigned pad[2];
};

// dots written by a kernel mode
__host__ __device__ constexpr int kry_dots(int mode) {
  return mode == kKryDot1 || mode == kKryUpdate ? 1 : mode == kKryDot2 || mode == kKryUpdateC ? 2 : 0;
}

// the persistent grid of (dtype, mode, wide) for ntiles tiles
int krylov_grid(int device, int dtype, int mode, bool wide, unsigned ntiles);
// the tile launch (none for an empty box) and, for a mode with dots, the combine launch into out[0 .. dots); returns the
// number of kernels launched.  t is BICG_P's second scalar (omega); the other modes ignore it.
int launch_krylov(const KryParams &p, int dtype, int mode, bool wide, int grid, double s, double t, KryPartial *scratch, sb_reduce_exact_part *out,
                  cudaStream_t stream);

} // namespace sb
