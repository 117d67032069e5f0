// Boundary-condition fill: the ghost cells behind the wall faces of a subdomain, for every quantity, in one launch.
//
// The host (capi.cu, sb_bc_plan_create) turns each (quantity, BC region) of include/stencil_b200.h into a segment: a
// box of ghost cells, its source map (a mirror on every wall axis) and the chain of operations the wall faces apply.
// A persistent grid walks a tile table of row ranges, like the copy engine (box_copy.cuh), in two shapes:
//   row segments     no mirror along x (y and z faces, their edges): a ghost row is another row of the same x range,
//                    so a power-of-two group of lanes moves it with the widest access its addresses allow (16 bytes on
//                    lead-aligned allocations) and four accesses in flight per lane;
//   mirrored rows    a wall on x: the row is reversed within itself, ghost widths are 1..3 cells, so one lane owns a row.
// Sources are never cells a BC writes, so no tile waits for another.
#pragma once

#include <cuda_runtime.h>

namespace sb {

struct BcSeg {
  char *base; // the allocation's element (0, 0, 0)
  long long pitch, slice;
  int pos[3];    // first ghost cell of the box (allocation coordinates)
  int ext[3];    // box extent
  int mirror[3]; // wall axis: source coordinate = mirror - p; else -1 (source = p)
  int read;      // 1: start from the source cell; 0: start from value0 (a VALUE face), nothing is read
  int nops;      // then, for k < nops: v = twoc[k] - v (the ODD faces after the last VALUE face)
  double value0; // exactly representable in the quantity's type (converted on the host)
  double twoc[3];
  unsigned es;       // element size in bytes
  unsigned dtype;    // sb_dtype: 0 raw (copy only), 1 float, 2 double
  unsigned vec;      // row segments: access width in bytes, divides every address, pitch and the row
  unsigned lg_group; // row segments: log2 of the lanes that share a row
};

struct BcTile {
  unsigned seg;
  unsigned row0; // first row (rows = ext.y * ext.z, y fastest)
  unsigned nrows;
};

constexpr int kBcThreads = 256;

void launch_bc_fill(const BcSeg *segs_dev, const BcTile *tiles_dev, unsigned ntiles, int grid, cudaStream_t stream);

} // namespace sb
