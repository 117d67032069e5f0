// Deterministic reductions: min, max, sum and sum of squares of a per-cell value over a box of compute cells.
//
// The host (capi.cu, sb_reduce_plan_create) turns each sb_reduce_item of include/stencil_b200.h into a RedItem and cuts
// its box into tiles of whole x rows.  Launch 1 is a persistent grid over that tile table (one kernel per class of
// items present: element type x kind x access width): inside a tile, a
// power-of-two group of G lanes owns a row and reads it with the widest access its addresses allow (16 bytes, after
// peeling a head and a tail of at most 3 cells per row), four accesses per source in flight per lane.  Each thread keeps
// one FP64 chain per statistic over the cells it reads; the block combines its 256 chains by a fixed tree and writes
// one partial per tile.  Launch 2 (one block per item) combines the item's tile partials by a pairwise tree in tile
// order.  Nothing depends on which CTA took which tile or how many CTAs ran, so the result bits are a function of the
// box and the allocation layout alone.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

#include "stencil_b200.h"

namespace sb {

struct RedItem {
  const char *src[3];     // address of the box's cell (lo.x, lo.y, lo.z) in each source
  long long pitch, slice; // bytes between rows / planes (the same for every source)
  int ext[3];             // box extent
  int kind;               // sb_reduce_kind
  int dtype;              // SB_DTYPE_F32 / SB_DTYPE_F64
  int vec;                // 16: 16-byte body with a peeled head and tail per row; else one element per access
  int lg_group;           // log2 of the lanes that share a row
  unsigned tile0, ntiles; // this item's tiles in the table (and its partials in the scratch)
  long long count;
};

struct RedTile {
  unsigned item;
  unsigned row0; // first row (rows = ext.y * ext.z, y fastest)
  unsigned nrows;
};

struct RedPartial {
  double min, max, sum, sumsq;
};

constexpr int kRedThreads = 256;
// A tile holds as many whole passes of the block over its rows as keep every thread's chain at or below kRedChain cells
// (rows wider than that per lane give one pass and a longer chain; see sb_reduce_plan_create).
constexpr int kRedChain = 256;

// min / max that propagate NaN: a NaN operand wins, otherwise the smaller (larger); for equal operands (+0 and -0) a.
__host__ __device__ inline double red_min(double a, double b) { return (a != a) ? a : ((b != b) || b < a) ? b : a; }
__host__ __device__ inline double red_max(double a, double b) { return (a != a) ? a : ((b != b) || b > a) ? b : a; }

// The one rule by which two results merge (device tile tree and sb_reduce_combine alike).
__host__ __device__ inline sb_reduce_result red_merge(const sb_reduce_result &a, const sb_reduce_result &b) {
  sb_reduce_result r;
  r.min = red_min(a.min, b.min);
  r.max = red_max(a.max, b.max);
  r.sum = a.sum + b.sum;
  r.sumsq = a.sumsq + b.sumsq;
  r.count = a.count + b.count;
  return r;
}

// One cell's v and its squared term q (include/stencil_b200.h), formed with separately rounded operations (no FMA
// contraction), for the exact kernels.  reduce.cu's add(Acc &) writes the same operations out: calling this from there
// swaps the operands of the min / max compares in the FP64 SCALAR ordered kernels' SASS.
template <int KIND> __device__ __forceinline__ void cell_terms(double x, double y, double z, double &v, double &q) {
  if (KIND == SB_REDUCE_SCALAR) {
    v = x;
    q = __dmul_rn(v, v);
  } else if (KIND == SB_REDUCE_DIFF) {
    v = __dadd_rn(x, -y);
    q = __dmul_rn(v, v);
  } else {
    q = __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
    v = __dsqrt_rn(q);
  }
}

// Launch 1 has one kernel instance per class (element type, kind, access width); the tile table holds the tiles of
// each class contiguously, class by class.
constexpr int kRedClasses = 12;
int reduce_class(const RedItem &it);
// persistent grid of class cls: resident blocks per SM times the SM count, at most ntiles
int reduce_grid(int device, int cls, unsigned ntiles);
// the same for any tile kernel of kRedThreads threads
int persistent_grid(int device, const void *kernel, unsigned ntiles);
// launch 1 (the classes with tiles) and launch 2 on `stream`; returns the number of kernels launched
int launch_reduce(const RedItem *items_dev, unsigned nitems, const RedTile *tiles_dev, const unsigned (*class_tiles)[2], const int *grids,
                  RedPartial *scratch, sb_reduce_result *out, cudaStream_t stream);

// ---- exact reductions (sb_reduce_exact_*; DESIGN.md section 2.6.1).  The same items, tile table, classes and row walk.
// Each thread keeps, per sum, a floating-point expansion of kExFpe doubles grown by TwoSum (error-free while no operand
// reaches 2^990); what does not fit (the expansion's last error term, a term of magnitude >= 2^990, inf and NaN) goes to
// the CTA's fixed-point accumulator in shared memory by 64-bit shared atomics.  The accumulator has one int64 counter
// per 32-bit digit (LSB weight 2^-1074) and receives unsigned chunks below 2^32, so it holds at least 2^31 additions: a
// tile never makes that many (sb_reduce_exact_plan_create refuses rows of more than 2^27 cells, so a tile holds at most
// 2^30 cells).  At the end of a tile each warp merges its 32 expansions, lane 0 adds its own to the accumulator, and the
// tile's counters, flags and min / max (by the plain kernel's tree) go to its partial.  Launch 2 adds an item's tile
// partials digit by digit, carries them to the canonical sb_exact_sum and merges min / max by the plain tile-order tree.
constexpr int kExDigits = 2 * SB_EXACT_WORDS; // 32-bit digits of the accumulator
constexpr int kExFpe = 3;                     // doubles per thread and sum
constexpr int kExCombineThreads = 1024;

struct RedExactPartial {
  double min, max;
  long long digit[2][kExDigits]; // [sum of v, sum of q]: uncarried counters of 32-bit digits
  unsigned flags[2];
  unsigned pad[2];
};

int reduce_exact_grid(int device, int cls, unsigned ntiles);
int launch_reduce_exact(const RedItem *items_dev, unsigned nitems, const RedTile *tiles_dev, const unsigned (*class_tiles)[2], const int *grids,
                        RedExactPartial *scratch, sb_reduce_exact_part *out, cudaStream_t stream);

} // namespace sb
