// 7-point jacobi step with hot/cold Dirichlet spheres -- H100 rewrite of the reference's user
// kernel (bin/jacobi3d.cu:40-85).  Bandwidth-bound pointwise stencil: no tensor cores.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace sb {

struct JacobiParams {
  char *dst;       // allocation base (element 0,0,0)
  const char *src; // allocation base
  long long pitch; // bytes between rows (same for src and dst)
  long long slice; // bytes between planes
  int raw[3];      // allocation size in elements (x,y,z)
  int lo[3];       // region to update, ALLOCATION-relative element coordinates
  int hi[3];
  int org[3];    // global coordinate of allocation element (0,0,0)
  int hot_x;     // sphere centres (global coordinates), shared y/z
  int cold_x;
  int cy, cz;
  int rad;       // sphere radius
  int zchunk;    // planes marched per CTA
  int prefetch;  // L2 prefetch distance in planes (0 = off)
  int x0a;       // first cell of the first strip: the largest x <= lo[0] whose address is vector aligned (set by the launcher)
  // fused halo push (launch_jacobi_push): for direction d = -x,+x,-y,+y,-z,+z the address, inside the NEIGHBOUR's
  // output allocation, of the ghost line/plane this subdomain's boundary cells belong to, already offset to the fixed
  // coordinate of that face; the two varying coordinates are this subdomain's own allocation coordinates times the
  // neighbour's pitch / slice.  nullptr = no push in that direction.
  char *push_ptr[6];
  long long push_pitch[6];
  long long push_slice[6];
  // periodic self-neighbour along x / y / z (fused launch only): the first / last column (row) takes its out-of-subdomain
  // neighbour from the OPPOSITE face of src instead of from the ghost cells -- a pointer set up before the marching loop,
  // so that axis needs no exchange and no push at all
  int xwrap, ywrap, zwrap;
  // dense x faces between ranks (fused launch, mode 3): xdense[d] != 0 means push_ptr[d] is not a ghost column but a
  // dense array [y][z] (z fastest, this subdomain's allocation coordinates; push_pitch[d] = bytes per row) in the
  // NEIGHBOUR's memory: the column is staged in shared memory and written out as one 256-byte line per row and chunk
  // instead of one 8-byte NVLink store per row and plane.  xghost_ptr[s]: the same kind of array received FROM the
  // neighbour on side s, read by the edge lanes instead of the ghost column of src.
  int xdense[2];
  const char *xghost_ptr[2];
  long long xghost_pitch[2];
};

// Mailbox rows of the fused kernel (see jacobi_fused_kernel): one word per boundary tile of a face -- (z chunks x tile rows)
// for x faces, (z chunks x strips) for y faces, (tile rows x strips) for z faces; 32 x 64 = 2048 at 512^3 FP64 with the
// default 16-plane chunks (launch_jacobi_fused falls back to 32-plane chunks where 16 would exceed the limit)
#ifndef SB_FUSED_MAX_GROUPS
#define SB_FUSED_MAX_GROUPS 4096
#endif

// Ordering between ranks inside the fused kernel.  All pointers are device addresses.
struct FusedSync {
  const uint32_t *wait_row[6];   // per face: this GPU's mailbox row [tile] written by the neighbour across that face (null: no wait)
  uint32_t *signal_row[6];       // per face: the neighbour's mailbox row [tile] for this subdomain (null: neighbour ordered by stream events)
  uint32_t wait_value, signal_value;
  int xrot, yrot, zrot;    // set by the launcher: where the walk over the tiles starts on each axis
  int any_wait, any_signal; // set by the launcher
  int col_cy, col_x;        // set by the launcher: tail-column tiles of phase-shifted rows (march_column): CTAs per z chunk (0: none), first cell
  int debug;                // timing experiments (SB_DEBUG_FUSED bits 16, 32; wrong results)
};

// Up to 8 thin regions (the exterior slabs of one subdomain) updated by ONE launch.
struct JacobiRegions {
  int n;
  int lo[8][3];  // allocation-relative
  int ext[8][3];
  long long first[9]; // prefix sum of cell counts
};

// returns the number of kernel launches issued (0 if the region is empty)
int launch_jacobi_regions(const JacobiParams &p, const JacobiRegions &r, int dtype_size, cudaStream_t stream);
int launch_jacobi(const JacobiParams &p, int dtype_size, cudaStream_t stream);
// the same update over the WHOLE compute region [lo, hi) of a subdomain; every boundary cell is also stored into the
// ghost cell of the face neighbour that needs it (p.push_*), so the next iteration needs no halo exchange
int launch_jacobi_fused(const JacobiParams &p, const FusedSync &sync, int dtype_size, cudaStream_t stream);
int launch_fill(char *dst, long long pitch, long long slice, const int lo[3], const int hi[3], int dtype_size, double value,
                cudaStream_t stream);
int launch_sqdiff(const char *a, const char *b, long long pitch, long long slice, const int lo[3], const int hi[3],
                  int dtype_size, double *out_dev, cudaStream_t stream);

} // namespace sb
