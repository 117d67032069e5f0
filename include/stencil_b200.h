/* stencil_b200.h -- C ABI of the H100-native halo-exchange / jacobi hot path.
 *
 * This is the drop-in boundary below the C++ API (include/stencil/*.hpp): plain pointers and
 * sizes, no C++ or torch types.  Each entry point names the interface of cwpearson/stencil it
 * replaces (paths relative to the reference checkout).  Device pointers are raw CUDA device
 * addresses (cudaMalloc, cudaIpcOpenMemHandle or peer-mapped); `stream` is a cudaStream_t passed
 * as void*.  All functions return 0 on success or a negative sb_status; sb_last_error() gives the
 * message.  Nothing here falls back to the CPU: without a CUDA device every launch fails loudly.
 *
 * Memory layout (reference src/local_domain.cu:187-203): quantity allocation = x fastest,
 * element (x,y,z) at byte offset (z*ysize + y)*pitch + x*elem_size, where (pitch, ysize) are the
 * cudaPitchedPtr fields the reference carries (pitch == xsize == row bytes, unpitched).
 */
#ifndef STENCIL_B200_H
#define STENCIL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_VERSION 2

typedef enum sb_status {
  SB_OK = 0,
  SB_ERR_INVALID = -1, /* bad argument */
  SB_ERR_CUDA = -2,    /* a CUDA runtime call failed */
  SB_ERR_NOGPU = -3,   /* no usable CUDA device */
  SB_ERR_ALLOC = -4
} sb_status;

/* Thread-local message for the last failing call on this thread. */
const char *sb_last_error(void);
int sb_version(void);
/* Number of kernel launches issued by this library since load (bench.py's gpu_launches). */
uint64_t sb_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Geometry.  radius27 is the reference's DirectionMap<size_t> storage order:
 * radius27[(dz+1)*9 + (dy+1)*3 + (dx+1)]  (include/stencil/direction_map.hpp:15,44-50).
 * ------------------------------------------------------------------------------------------- */

/* LocalDomain::halo_pos, src/local_domain.cu:86-125 */
int sb_halo_pos(const int64_t dir[3], const int64_t size[3], const int64_t radius27[27], int halo, int64_t out[3]);
/* LocalDomain::halo_extent, include/stencil/local_domain.cuh:212-222 */
int sb_halo_extent(const int64_t dir[3], const int64_t size[3], const int64_t radius27[27], int64_t out[3]);
/* LocalDomain::raw_size, local_domain.cuh:236-239 */
int sb_raw_size(const int64_t size[3], const int64_t radius27[27], int64_t out[3]);
/* prime_factors (descending), src/numeric.cpp:6-26.  Returns the count (<= cap) or <0. */
int sb_prime_factors(int64_t n, int64_t *out, int cap);
/* RankPartition, include/stencil/partition.hpp:20-116: dim, base subdomain size, remainder */
int sb_rank_partition(const int64_t size[3], int64_t n, int64_t dim[3], int64_t base[3], int64_t rem[3]);
/* NodePartition, partition.hpp:120-256 */
int sb_node_partition(const int64_t size[3], const int64_t radius27[27], int64_t nodes, int64_t gpus, int64_t sys_dim[3],
                      int64_t node_dim[3], int64_t base[3], int64_t rem[3]);
/* subdomain_size / subdomain_origin of either partition, partition.hpp:55-86 */
int sb_subdomain_size(const int64_t base[3], const int64_t rem[3], const int64_t idx[3], int64_t out[3]);
int sb_subdomain_origin(const int64_t base[3], const int64_t rem[3], const int64_t idx[3], int64_t out[3]);
/* DistributedDomain::get_interior / get_exterior for one subdomain, src/stencil.cu:878-977.
 * lo/hi = compute region of the subdomain (global coords).  Exterior: up to 6 boxes in the order
 * +x,+y,+z,-x,-y,-z; returns the number written to ext_lo/ext_hi (each 6*3 int64). */
int sb_interior(const int64_t lo[3], const int64_t hi[3], const int64_t radius27[27], int64_t int_lo[3], int64_t int_hi[3]);
int sb_exterior(const int64_t lo[3], const int64_t hi[3], const int64_t radius27[27], int64_t *ext_lo, int64_t *ext_hi);

/* ---------------------------------------------------------------------------------------------
 * Box copies: the one engine behind pack, unpack, translate and the fused direct halo write.
 * ------------------------------------------------------------------------------------------- */

/* A 3-D strided allocation, the cudaPitchedPtr the reference passes around. */
typedef struct sb_pitched {
  void *ptr;
  int64_t pitch; /* bytes between rows */
  int64_t ysize; /* rows per z-plane */
} sb_pitched;

/* One strided->strided copy of `extent` elements (x,y,z) from src@src_pos to dst@dst_pos.
 * Replaces translate() (src/copy.cu:34-77); with a dense dst it is pack_kernel
 * (src/pack_kernel.cu:3-59), with a dense src unpack_kernel (:61-108). */
typedef struct sb_box_copy {
  sb_pitched dst;
  int64_t dst_pos[3];
  sb_pitched src;
  int64_t src_pos[3];
  int64_t extent[3];
  int64_t elem_size;
} sb_box_copy;

/* pack_kernel / unpack_kernel / translate one-shots (tests launch these directly in the reference:
 * test/test_cuda_pack.cu:76, test/test_cuda_translate_kernel.cu). */
int sb_pack(void *dst, sb_pitched src, const int64_t pos[3], const int64_t extent[3], int64_t elem_size, void *stream);
int sb_unpack(sb_pitched dst, const void *src, const int64_t pos[3], const int64_t extent[3], int64_t elem_size,
              void *stream);
int sb_translate(sb_pitched dst, const int64_t dst_pos[3], sb_pitched src, const int64_t src_pos[3],
                 const int64_t extent[3], int64_t elem_size, void *stream);

/* A persistent plan: any number of box copies executed by ONE kernel launch on `device`.
 * This is what replaces, per source GPU, the reference's per-message launches of
 * dev_packer_pack_domain (src/packer.cu:10-26, 109-148), multi_translate (src/copy.cu:79-85,
 * tx_cuda.cuh:74-104), cudaMemcpyPeerAsync (tx_cuda.cuh:162) and dev_unpacker_unpack_domain
 * (src/packer.cu:28-44): destination pointers may be local, or a peer GPU's ghost cells
 * (peer-access or CUDA-IPC mapped), in which case the halo is written straight over NVLink. */
typedef struct sb_copy_plan sb_copy_plan;
int sb_copy_plan_create(sb_copy_plan **out, int device, const sb_box_copy *copies, int64_t n);
int sb_copy_plan_launch(sb_copy_plan *plan, void *stream);
int64_t sb_copy_plan_bytes(const sb_copy_plan *plan);     /* payload bytes per launch */
int64_t sb_copy_plan_num_tiles(const sb_copy_plan *plan); /* work items per launch */
int sb_copy_plan_destroy(sb_copy_plan *plan);

/* Cross-GPU completion flags for the fused exchange when source and destination GPUs are driven
 * by different processes (the reference's IPC event + 0-byte MPI notify, tx_cuda.cuh:225-315,
 * src/tx_ipc.cpp).  flags are uint32 slots in device memory that peers map via CUDA IPC.
 *  - sb_signal: after all prior work on `stream`, store `value` (release, system scope) to each
 *    of the n remote slots.
 *  - sb_wait:   make `stream` wait until each of n local slots is >= value (acquire). */
int sb_signal(uint32_t *const *remote_slots, int n, uint32_t value, int device, void *stream);
int sb_wait(const uint32_t *local_slots, int n, uint32_t value, int device, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Physical boundary conditions (BCs) on non-periodic grids (not in the reference, whose grids are periodic).
 * A wall face of a subdomain is a face across which the grid does not continue (an axis that does not wrap).  The
 * ghost cells behind it are filled after the halo exchange by ONE launch per subdomain.  Faces are numbered
 * 0..5 = -x, +x, -y, +y, -z, +z.  Each (quantity, face) has a kind and a value c:
 *   SB_BC_NONE   ghost cells untouched
 *   SB_BC_VALUE  ghost = c                                  (float / double quantities)
 *   SB_BC_EVEN   ghost = its mirror image about the face    (any element type: a plain copy)
 *   SB_BC_ODD    ghost = 2c - its mirror image              (float / double; c is the value AT the face, ODD(0) = antisymmetric)
 * Mirror along axis a in allocation coordinates, with ghost widths g- / g+ and compute cells [g-, g- + n): a low ghost
 * cell i reads 2 g- - 1 - i, a high ghost cell i reads 2 (g- + n) - 1 - i.  EVEN and ODD need g <= n on their side.
 * Regions: for each of the 26 directions d with radius27(d) > 0, the ghost box halo_pos(d, size, r, 1) of extent
 * halo_extent(d, size, r).  A region is written when a non-zero component of d points across a face whose kind is not
 * NONE; those are its wall axes A.  For a cell p of it: v = the allocation at p mirrored on every axis of A, then for each
 * a in A, in order x, y, z: VALUE v = c, EVEN v unchanged, ODD v = 2c - v, all in the quantity's type.  This equals the x
 * walls, then the y walls, then the z walls applied as separate passes, but every source cell is one no BC writes, so
 * the launch needs no ordering inside.  On non-wall axes the source is a ghost cell the exchange filled: launch after
 * every write of the exchange into this subdomain has completed.
 * ------------------------------------------------------------------------------------------- */
typedef enum sb_bc_kind { SB_BC_NONE = 0, SB_BC_VALUE = 1, SB_BC_EVEN = 2, SB_BC_ODD = 3 } sb_bc_kind;
typedef enum sb_dtype { SB_DTYPE_RAW = 0, SB_DTYPE_F32 = 1, SB_DTYPE_F64 = 2 } sb_dtype;

/* One BC region of a subdomain.  pos / extent: the ghost box in allocation coordinates.  mirror[a]: on a wall axis the
 * source coordinate is mirror[a] - p[a]; on the other axes mirror[a] = -1 and the source coordinate is p[a].
 * faces: bit f set when face f (numbered as above) is applied to this region; they are applied in order x, y, z. */
typedef struct sb_bc_region {
  int64_t dir[3];
  int64_t pos[3];
  int64_t extent[3];
  int64_t mirror[3];
  int32_t faces;
  int32_t reserved;
} sb_bc_region;

/* Host only.  The BC regions of a subdomain of compute size `size` whose faces carry `kinds` (sb_bc_kind, per face;
 * NONE on every face that is not a wall of this subdomain), in direction order z, y, x ascending (dir -1 first).
 * Writes at most cap regions to out (out may be NULL with cap 0) and returns their total number (<= 26), or
 * SB_ERR_INVALID when a kind is unknown or an EVEN / ODD face has a ghost width larger than the subdomain on its axis. */
int sb_bc_regions(const int64_t size[3], const int64_t radius27[27], const int32_t kinds[6], sb_bc_region *out, int cap);

/* ---------------------------------------------------------------------------------------------
 * The exchange plan (include/stencil/exchange_plan.hpp), host only.  A grid of dim subdomains cut as (base, rem) --
 * the pair sb_node_partition / sb_rank_partition return -- closed per axis by boundary[a] = 1 (PERIODIC: wraps) or
 * 2 (FIXED: a wall), the values of Topology::Boundary.  Errors (SB_ERR_INVALID with a message): dim < 1 on an axis, an
 * index outside the grid, another boundary value, an elem_size <= 0, an output capacity below the count.
 * ------------------------------------------------------------------------------------------- */
/* One message: the outermost compute cells of the source on side dir, at src_pos, go to the ghost cells of subdomain
 * dst_idx on side -dir, at dst_pos; extent elements. */
typedef struct sb_message {
  int64_t dir[3];
  int64_t dst_idx[3];
  int64_t src_pos[3];
  int64_t dst_pos[3];
  int64_t extent[3];
} sb_message;
/* Every message subdomain src_idx sends, in direction order z, y, x ascending: a direction is skipped when
 * radius27(-dir) == 0, when the step crosses a wall, or when the box is empty.  Returns the count (<= 26). */
int sb_exchange_messages(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                         const int64_t radius27[27], const int64_t src_idx[3], sb_message *out, int cap);

/* Rows shorter than SB_STAGE_MAX_ROW_BYTES bound for another GPU travel through one dense staging buffer per
 * (src, dst) pair in the receiver's memory.  Entry: quantity q of message msg (an index into src_idx's
 * sb_exchange_messages list) sits at byte offset of that buffer. */
#define SB_STAGE_MAX_ROW_BYTES 64
typedef struct sb_staged {
  int64_t msg;
  int64_t q;
  int64_t offset;
} sb_staged;
/* The layout of the (src_idx -> dst_idx) staging buffer for quantities of elem_sizes[0..nq): src_idx's messages to
 * dst_idx in order, each one's quantities in order; a pair is staged when extent[0] * elem_size < SB_STAGE_MAX_ROW_BYTES.
 * Each entry starts at a 16-byte boundary; *total = the end of the last one (0: nothing staged).  Returns the count.
 * Whether staging applies at all (the two subdomains live on different GPUs) is the caller's decision. */
int sb_staging_layout(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                      const int64_t radius27[27], const int64_t src_idx[3], const int64_t dst_idx[3],
                      const int64_t *elem_sizes, int nq, sb_staged *out, int cap, int64_t *total);
/* sb_staging_layout of an exchange of a subset of the quantities: bit q of quantities set = quantity q is exchanged.
 * Returns the full layout's entries of those quantities only, at the same offsets, and the same *total, so a subset
 * exchange packs into the full exchange's staging buffers.  quantities ~0 is sb_staging_layout.  Errors besides
 * sb_staging_layout's: an empty set, and a bit q >= nq ("quantity q is not one of the nq quantities"). */
int sb_staging_layout_subset(const int64_t dim[3], const int64_t base[3], const int64_t rem[3], const int32_t boundary[3],
                             const int64_t radius27[27], const int64_t src_idx[3], const int64_t dst_idx[3],
                             const int64_t *elem_sizes, int nq, uint64_t quantities, sb_staged *out, int cap, int64_t *total);

/* One quantity of a BC plan: its allocation (the CURRENT buffer the plan will read and write), element type, and
 * per-face kind and value.  dtype RAW takes elem_size 1, 2, 4, 8 or 16 and allows NONE and EVEN only; F32 needs
 * elem_size 4, F64 elem_size 8.  value[f] is converted to the quantity's type. */
typedef struct sb_bc_quantity {
  sb_pitched data;
  int64_t elem_size;
  double value[6];
  int32_t dtype;
  int32_t kind[6];
} sb_bc_quantity;

/* A persistent plan: every BC region of every quantity of one subdomain, filled by ONE launch on `device`.  The tile
 * table is uploaded here; size / radius27 describe the subdomain (every quantity has the same geometry).  Errors
 * (SB_ERR_INVALID with a message): a kind outside sb_bc_kind, VALUE or ODD on a RAW quantity, a mismatched elem_size,
 * EVEN or ODD with a ghost width larger than the subdomain.  A plan with nothing to write launches nothing. */
typedef struct sb_bc_plan sb_bc_plan;
int sb_bc_plan_create(sb_bc_plan **out, int device, const sb_bc_quantity *quantities, int64_t n, const int64_t size[3],
                      const int64_t radius27[27]);
int sb_bc_plan_launch(sb_bc_plan *plan, void *stream);
int64_t sb_bc_plan_bytes(const sb_bc_plan *plan); /* ghost-cell bytes written per launch */
int sb_bc_plan_destroy(sb_bc_plan *plan);

/* ---------------------------------------------------------------------------------------------
 * Deterministic reductions over a box of compute cells (the reference's astaroth reductions, astaroth/reductions.cuh,
 * RTYPE_MIN / MAX / SUM / RMS of astaroth/user_defines.h:161-169; its jacobi driver has none).
 * An item is a source evaluated at every cell of the box [lo, hi) (global coordinates; acc_origin = global coordinate
 * of allocation element (0,0,0), as for sb_jacobi3d).  Ghost cells are never read.  Per cell, in FP64 with separately
 * rounded operations (no FMA):
 *   SB_REDUCE_SCALAR  v = a                                   q = v*v
 *   SB_REDUCE_DIFF    v = a - b                               q = v*v
 *   SB_REDUCE_NORM3   s = ((a*a + b*b) + c*c), v = sqrt(s)    q = s
 * with a, b, c = src[0..2] widened to double.  Result: min and max of v (a NaN v makes both NaN), sum = sum of v,
 * sumsq = sum of q, count = cells.  An empty box gives min = +inf, max = -inf, sum = sumsq = 0, count = 0.
 * Determinism: the order of every sum is a function of the box and the allocation layout only (not of the SM count or
 * of which CTA took which tile), so a plan gives the same bits on every launch, in a CUDA graph, and on every rank.
 * ------------------------------------------------------------------------------------------- */
typedef enum sb_reduce_kind { SB_REDUCE_SCALAR = 0, SB_REDUCE_DIFF = 1, SB_REDUCE_NORM3 = 2 } sb_reduce_kind;

/* One item.  dtype: SB_DTYPE_F32 or SB_DTYPE_F64, shared by its sources, which also share pitch and ysize.  SCALAR reads
 * src[0], DIFF src[0] - src[1], NORM3 src[0..2]; unused sources are ignored. */
typedef struct sb_reduce_item {
  int32_t kind, dtype;
  sb_pitched src[3];
  int64_t acc_origin[3], lo[3], hi[3];
} sb_reduce_item;

typedef struct sb_reduce_result {
  double min, max, sum, sumsq;
  int64_t count;
} sb_reduce_result;

/* A persistent plan: n >= 1 items, reduced by one launch sequence on `device` (a tile kernel and a small per-item
 * combine).  Errors (SB_ERR_INVALID with a message, before anything is allocated): n < 1, an unknown kind or dtype,
 * sources of one item with different pitches or row counts, a pointer or pitch that is not a multiple of the element
 * size, lo > hi on an axis, a box outside the allocation.
 * sb_reduce_plan_launch writes one sb_reduce_result per item, in item order, to out_dev (device memory, n results)
 * in the order of `stream`.  It allocates nothing and never synchronises the host, so it may be captured in a CUDA
 * graph.  The plan owns the scratch memory the launch uses: at most ONE launch of a plan may be in flight at a time
 * (order launches of the same plan on one stream, or wait for the previous one). */
typedef struct sb_reduce_plan sb_reduce_plan;
int sb_reduce_plan_create(sb_reduce_plan **out, int device, const sb_reduce_item *items, int64_t n);
int sb_reduce_plan_launch(sb_reduce_plan *plan, sb_reduce_result *out_dev, void *stream);
int64_t sb_reduce_plan_bytes(const sb_reduce_plan *plan); /* source bytes read per launch */
int sb_reduce_plan_destroy(sb_reduce_plan *plan);
/* Host only.  The one place that defines how results merge: parts[0..n) (n >= 1) combined by the pairwise tree
 * "parts[i] = merge(parts[i], parts[i + s]) for every i % 2s == 0, i + s < n" for s = 1, 2, 4, ..., result parts[0];
 * merge takes the NaN-propagating min and max and adds sum, sumsq and count.  Callers pass per-subdomain results in
 * global subdomain-index order (partition index (i, j, k), x fastest). */
int sb_reduce_combine(const sb_reduce_result *parts, int64_t n, sb_reduce_result *out);

/* ---------------------------------------------------------------------------------------------
 * Exact reductions (DESIGN.md section 2.6.1): the same items and per-cell v and q as above, with
 *   min, max, count  the plain plan's, bit for bit (the same NaN rule and empty-box values); across parts,
 *                    sb_reduce_exact_combine's order-independent rule below, which may pick other bits than
 *                    sb_reduce_combine's tree only between +0 and -0 or between two NaNs;
 *   sum (sumsq)      the exact real sum of every v (q), rounded once to double, to nearest, ties to even.
 * Special values, for both sums: a NaN term gives NaN; +inf and -inf among the terms give NaN; otherwise an infinite
 * term gives that infinity; an exact sum beyond the double range rounds to +-inf as IEEE round-to-nearest does; an
 * exact zero is +0.0.  A q that overflowed to inf when it was formed is an infinite term.
 * The sums depend only on the multiset of per-cell terms: not on the partition, the tiling, the allocation layout, the
 * SM count or the order in which parts are combined.
 *
 * sb_exact_sum is the canonical accumulator: the exact sum of the finite terms as a 2176-bit two's complement integer
 * in units of 2^-1074, word[0] least significant, fully carried (equal multisets give byte-identical accumulators),
 * plus the flags of the non-finite terms.  A finite term is below 2^1024 = 2^2098 units, so any sum of fewer than 2^77
 * terms (every cell count the library can form, and any combine of such parts) fits without overflow.
 * ------------------------------------------------------------------------------------------- */
#define SB_EXACT_WORDS 34
#define SB_EXACT_NAN 1u     /* some term is NaN */
#define SB_EXACT_POS_INF 2u /* some term is +inf */
#define SB_EXACT_NEG_INF 4u /* some term is -inf */
typedef struct sb_exact_sum {
  uint64_t word[SB_EXACT_WORDS];
  uint64_t flags;
} sb_exact_sum;

typedef struct sb_reduce_exact_part {
  double min, max;
  int64_t count;
  sb_exact_sum sum, sumsq;
} sb_reduce_exact_part;

/* A persistent plan with the contract of sb_reduce_plan_*: the same items and the same errors and messages, plus one:
 * a box with rows of more than 2^27 cells.  sb_reduce_exact_plan_launch writes one sb_reduce_exact_part per item, in
 * item order, to out_dev (device memory); it allocates nothing, never synchronises the host, may be captured in a CUDA
 * graph, and at most one launch of a plan may be in flight at a time. */
typedef struct sb_reduce_exact_plan sb_reduce_exact_plan;
int sb_reduce_exact_plan_create(sb_reduce_exact_plan **out, int device, const sb_reduce_item *items, int64_t n);
int sb_reduce_exact_plan_launch(sb_reduce_exact_plan *plan, sb_reduce_exact_part *out_dev, void *stream);
int64_t sb_reduce_exact_plan_bytes(const sb_reduce_exact_plan *plan); /* source bytes read per launch */
int sb_reduce_exact_plan_destroy(sb_reduce_exact_plan *plan);
/* Host only.  parts[0..n) (n >= 1, e.g. one per subdomain) merged: accumulators added, flags or-ed, counts added, min
 * and max by a rule that does not depend on the order of parts (a NaN operand wins, the larger bit pattern of two
 * NaNs; of +0 and -0 min takes -0 and max +0).  Combine parts, then round: rounding each part first would make the
 * result depend on the partition again. */
int sb_reduce_exact_combine(const sb_reduce_exact_part *parts, int64_t n, sb_reduce_exact_part *out);
/* Host only.  The one place that rounds: min, max and count copied, sum and sumsq rounded by the rule above. */
int sb_reduce_exact_round(const sb_reduce_exact_part *part, sb_reduce_result *out);

/* ---------------------------------------------------------------------------------------------
 * Krylov vector kernels (DESIGN.md section 2.13): the vector algebra between operator applications of a conjugate-gradient
 * iteration, one elementwise pass over a box [lo, hi) (global coordinates) of buffers that share dtype, pitch and row
 * count.  T(s) is the double s rounded to the buffers' type; every per-cell multiply and add is rounded to nearest on
 * its own (no FMA contraction).  An exact dot <a, b> is the exact real sum over the cells of v = fl64(double(a) *
 * double(b)) (exact for float; one rounded multiply for double), written as an sb_reduce_exact_part with sum = the
 * exact sum of v, sumsq = an exact zero, count = the cells and min / max of v by sb_reduce_exact_combine's
 * order-independent rule; so parts of several boxes, subdomains or ranks merge by sb_reduce_exact_combine and round once
 * by sb_reduce_exact_round, and the result does not depend on the partition.
 *   SB_KRYLOV_DOT     buffers a, b[, c]: part 0 = <a, b>, part 1 = <a, c> (with c).  Sources may alias.
 *   SB_KRYLOV_XPBY    buffers p, z:      p = z + T(s) * p; where T(s) is +0 or -0, p = z without reading p.  p and z
 *                                      must not overlap.
 *   SB_KRYLOV_UPDATE  buffers x, p, r, q[, c]: x = x + T(s) * p, r = r - T(s) * q, part 0 = <r, r> of the stored new
 *                     r and, with c, part 1 = <c, r> of the stored new r.  x, p, r and q are four buffers, no two
 *                     overlapping; c must not overlap x or r, and may be p or q (DESIGN.md section 2.14).
 *   SB_KRYLOV_BICG_P  buffers p, r, v:   p = r + T(s) * (p - T(t) * v), the BiCGStab direction with s = beta and
 *                     t = omega (section 2.14).  p must not overlap r or v; r and v may alias.
 * Cells outside the box are neither read nor written.
 * ------------------------------------------------------------------------------------------- */
typedef enum sb_krylov_mode { SB_KRYLOV_DOT = 0, SB_KRYLOV_XPBY = 1, SB_KRYLOV_UPDATE = 2, SB_KRYLOV_BICG_P = 4 } sb_krylov_mode;

/* A persistent plan of one mode over one box.  bufs: nbuf buffers in the order above (DOT 2 or 3, XPBY 2, UPDATE 4 or
 * 5, BICG_P 3), acc_origin the global coordinate of their element (0,0,0).  dtype SB_DTYPE_F32 or SB_DTYPE_F64.  Errors
 * (SB_ERR_INVALID with a message, before anything is allocated): an unknown mode or dtype, a wrong buffer count, a NULL
 * buffer, buffers with different pitches or row counts, a pointer or pitch that is not a multiple of the element size,
 * lo > hi, a box outside the allocation, rows of more than 2^27 cells or more than 2^31 rows, and forbidden aliasing:
 * XPBY's p equal to z, UPDATE's x, p, r, q not distinct, UPDATE's c equal to x or r, BICG_P's p equal to r or v, and
 * for XPBY, UPDATE and BICG_P any two buffers whose bytes from the box's first cell to its last overlap where one of
 * them is written or both are among UPDATE's x, p, r, q (DOT sources may alias; so may BICG_P's r and v and UPDATE's c
 * with p or q).  16-byte accesses are used when every buffer has the same address modulo 16.
 * sb_krylov_plan_launch runs the mode with the scalar s (ignored by DOT) and writes its parts (DOT: nbuf - 1, UPDATE: 1,
 * or 2 with c, XPBY and BICG_P: none, parts_dev may be NULL) to parts_dev (device memory) in the order of `stream`; it
 * allocates nothing, never synchronises the host, may be captured in a CUDA graph, and at most one launch of a plan may
 * be in flight at a time.  It refuses a BICG_P plan, which takes two scalars: sb_krylov_plan_launch2 passes s and t to
 * any mode (the modes other than BICG_P ignore t).
 * sb_krylov_plan_bytes: the algorithmic bytes of a launch, per cell one element per distinct buffer read (XPBY counts p)
 * and one per buffer written. */
typedef struct sb_krylov_plan sb_krylov_plan;
int sb_krylov_plan_create(sb_krylov_plan **out, int device, int mode, int dtype, const sb_pitched *bufs, int nbuf, const int64_t acc_origin[3],
                          const int64_t lo[3], const int64_t hi[3]);
int sb_krylov_plan_launch(sb_krylov_plan *plan, double s, sb_reduce_exact_part *parts_dev, void *stream);
int sb_krylov_plan_launch2(sb_krylov_plan *plan, double s, double t, sb_reduce_exact_part *parts_dev, void *stream);
int64_t sb_krylov_plan_bytes(const sb_krylov_plan *plan);
int sb_krylov_plan_destroy(sb_krylov_plan *plan);

/* ---------------------------------------------------------------------------------------------
 * Constant-coefficient linear stencil operators (not in the reference; DESIGN.md section 2.7).
 * An operator is a list of 1 <= n <= SB_STENCIL_MAX_TERMS terms (source s, offset o, weight w): s = 0 reads src at
 * p + o, s = 1 reads aux at p (aux terms have offset 0: a previous time level, a right-hand side, a blend);
 * |o_a| <= SB_STENCIL_MAX_REACH.  For every cell p of a box, in the quantity's type T with every multiply and add
 * rounded to nearest separately (no FMA contraction), T(w) = w rounded to T:
 *   acc = T(w_0) * S_0(p + o_0);  acc = acc + T(w_k) * S_k(p + o_k) for k = 1 .. n-1 in list order;  dst[p] = acc
 * dst may be aux (each cell's aux value is read before that cell is written, by the same thread); dst must not be src.
 * Reads stay inside the allocation; cells of dst outside the boxes are not written.  The result does not depend on the
 * launch shape.
 * ------------------------------------------------------------------------------------------- */
#define SB_STENCIL_MAX_TERMS 64
#define SB_STENCIL_MAX_REACH 4
typedef struct sb_stencil_term {
  int32_t source;    /* 0 = src, 1 = aux */
  int32_t offset[3]; /* dx, dy, dz */
  double weight;
} sb_stencil_term;

/* Host only.  Whether a subdomain with ghost widths radius27 can apply the op: every term with o != 0 needs
 * radius27(sign(o)) > 0 (that ghost box is exchanged) and |o_a| <= the face radius on side sign(o_a) of every axis a with
 * o_a != 0.  SB_ERR_INVALID, with a message naming the term, for a term that breaks either condition or a list outside
 * the limits above (n, source, |o_a|, an aux term with an offset).  A wall face passes like any other face. */
int sb_stencil_check(const sb_stencil_term *terms, int n, const int64_t radius27[27]);
/* Host only.  The central-difference Laplacian of order 2, 4, 6 or 8 (radius 1 to 4) on a grid of spacing[3]: the centre
 * term, then for k = 1..R the axes x, y, z, side - then side +.  In double with i_a = 1 / (h_a * h_a): an axis term is
 * c_k * i_a, the centre (c_0 * i_x + c_0 * i_y) + c_0 * i_z, with c = (-2, 1), (-5/2, 4/3, -1/12),
 * (-49/18, 3/2, -3/20, 1/90), (-205/72, 8/5, -1/5, 8/315, -1/560).  Writes at most cap terms (out may be NULL with cap 0)
 * and returns their total number 1 + 6R, or SB_ERR_INVALID for another order or a spacing that is not finite and > 0. */
int sb_stencil_laplacian(int order, const double spacing[3], sb_stencil_term *out, int cap);

/* A persistent plan: the op over nbox boxes [lo, hi) (global coordinates, nbox*3 int64 each; acc_origin = global
 * coordinate of allocation element (0,0,0), as for sb_jacobi3d) of three allocations of zsize planes that share pitch and
 * ysize.  dtype SB_DTYPE_F32 or SB_DTYPE_F64; aux.ptr may be NULL when no term reads aux.  Boxes of at least 8 cells on
 * every axis go to the z-marching tile kernel, one launch each; thinner boxes (exterior slabs) share one-thread-per-cell
 * launches of up to 16 boxes.  Errors (SB_ERR_INVALID with a message, checked before anything is allocated): an unknown
 * dtype, an invalid term list, an aux term without aux, dst == src, mismatched pitches or row counts, a pointer or pitch
 * that is not a multiple of the element size, lo > hi, and a box whose reads leave the allocation.  The kernels take
 * allocation coordinates as 32-bit int, so a box whose read window (reach included) ends past 2^31 - 1 on some axis, or
 * that has 2^32 cells or more, is SB_ERR_INVALID too, with a message naming the box and axis; this holds for every
 * operator, coloured, diagonal and system plan.  Empty boxes keep their place in the numbering of the messages.
 * sb_stencil_plan_launch allocates nothing and never synchronises the host. */
typedef struct sb_stencil_plan sb_stencil_plan;
int sb_stencil_plan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_term *terms, int n, sb_pitched dst,
                           sb_pitched src, sb_pitched aux, const int64_t acc_origin[3], int64_t zsize, int nbox,
                           const int64_t *lo, const int64_t *hi);
int sb_stencil_plan_launch(sb_stencil_plan *plan, void *stream);
/* algorithmic bytes per launch: per cell, one element read of src, one of aux if a term reads it, one of each coefficient
 * field the op references (sb_stencil_vplan_create), one written */
int64_t sb_stencil_plan_bytes(const sb_stencil_plan *plan);
int sb_stencil_plan_destroy(sb_stencil_plan *plan);

/* ---------------------------------------------------------------------------------------------
 * Variable-coefficient linear stencil operators: the rule above, where a term may also name a coefficient field k
 * (0 <= k < SB_STENCIL_MAX_COEFS) read at p + c, |c_a| <= SB_STENCIL_COEF_REACH.  Per cell, in T, no FMA contraction:
 *   coefficient term  m_t = (T(w_t) * C_k(p + c_t)) * S_t(p + o_t)      (two multiplies, each rounded)
 *   plain term        m_t = T(w_t) * S_t(p + o_t)
 *   acc = m_0;  acc = acc + m_t for t = 1 .. n-1 in list order;  dst[p] = acc
 * With every C = 1 the result is the plain op's, bit for bit (T(w) * 1 is exact).  Coefficient fields are read only:
 * they must not be dst, may alias src, aux or each other, and share pitch and row count with src.  Aux terms keep offset
 * 0 and may carry a coefficient.
 * ------------------------------------------------------------------------------------------- */
#define SB_STENCIL_MAX_COEFS 4
#define SB_STENCIL_COEF_REACH 1
typedef struct sb_stencil_vterm {
  int32_t source;         /* 0 = src, 1 = aux */
  int32_t offset[3];      /* dx, dy, dz of the source read */
  int32_t coef;           /* coefficient field, or -1 for a plain term */
  int32_t coef_offset[3]; /* dx, dy, dz of the coefficient read; (0, 0, 0) on a plain term */
  double weight;
} sb_stencil_vterm;

/* Host only.  sb_stencil_check for coefficient terms: the same limits plus coef in -1 .. SB_STENCIL_MAX_COEFS - 1 and
 * |c_a| <= SB_STENCIL_COEF_REACH, and the same reach test applied to every src offset and every coefficient offset. */
int sb_stencil_vcheck(const sb_stencil_vterm *terms, int n, const int64_t radius27[27]);
/* Host only.  The conservative second-order div(kappa grad u) on a grid of spacing[3]: 12 terms.  Coefficient field a
 * holds kappa on the faces normal to axis a, C_a(p) on the face between p - e_a and p.  In double, i_a = 1 / (h_a * h_a);
 * for the axes x, y, z in order: (src +e_a, i_a, coef a at +e_a), (src 0, -i_a, coef a at +e_a), (src 0, -i_a, coef a
 * at 0), (src -e_a, i_a, coef a at 0).  Writes at most cap terms (out may be NULL with cap 0) and returns 12, or
 * SB_ERR_INVALID for a spacing that is not finite and > 0. */
int sb_stencil_div_grad(const double spacing[3], sb_stencil_vterm *out, int cap);
/* sb_stencil_plan_create with coefficient terms and ncoef (0 .. SB_STENCIL_MAX_COEFS) coefficient allocations coef[k],
 * which share dst's zsize.  sb_stencil_plan_create is this call with every coef = -1 and no fields.  Errors beyond
 * sb_stencil_plan_create's (SB_ERR_INVALID with a message, before anything is allocated): ncoef outside 0 .. 4, a term
 * naming a field >= ncoef, a NULL coefficient pointer, a coefficient offset beyond reach 1, a coefficient buffer equal to
 * dst, a coefficient with another pitch or row count or a misaligned pointer, a box whose coefficient reads leave the
 * allocation. */
int sb_stencil_vplan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                            sb_pitched src, sb_pitched aux, const sb_pitched *coef, int ncoef, const int64_t acc_origin[3],
                            int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi);

/* ---------------------------------------------------------------------------------------------
 * Coloured application (DESIGN.md section 2.9): Gauss-Seidel and SOR sweeps in place.  A colouring m is 1, 2 or 8 and a
 * colour c is 0 .. m-1, taken from the GLOBAL compute coordinates (x, y, z) of a cell:
 *   m = 1: every cell has colour 0 (the uncoloured rule)
 *   m = 2: colour (x + y + z) mod 2 (red-black)
 *   m = 8: colour (x mod 2) + 2 (y mod 2) + 4 (z mod 2)
 * A coloured launch evaluates the op rule above (plain or coefficient terms) on the buffers AS THEY WERE BEFORE THE
 * LAUNCH and writes dst[p] = op(p) for the cells p of the boxes of colour c only; every other cell of dst keeps its bits.
 * With m > 1, dst may be src (in place).  The colour condition: every src term with o != 0 reads a cell of another colour
 * than its own, for every cell, that is o_x + o_y + o_z odd for m = 2 and some o_a odd for m = 8.  It is checked
 * whenever m > 1, in place or not: a coloured op that reads its own colour is not a Gauss-Seidel sweep.  Aux terms keep
 * offset 0 and aux may be dst (so src as well); coefficient fields must not be dst, so in place they cannot be src.
 * Coefficient reads need no colour condition: nothing writes them.  On a periodic axis of odd length a cell and its
 * wrapped neighbour can share a colour; that read goes through a ghost cell and sees the old value, as the rule says.
 * Consequence: in place, "before the launch" and "in any order" give the same bits.  Every value a cell uses is its own
 * old value (read before its own write), a cell of another colour (which nothing writes) or a ghost cell (which nothing
 * writes), so a kernel races only on values it never uses.  A sweep is one launch per colour, each after an exchange:
 *   for c in 0 .. m-1:  exchange();  apply the op with colouring (m, c), dst = src = u
 * and it gives the same bits on every partition.
 * ------------------------------------------------------------------------------------------- */
/* Host only.  sb_stencil_vcheck plus, for ncolours > 1, the colour condition.  SB_ERR_INVALID with a message for
 * ncolours not 1, 2 or 8, or a term that reads its own colour (naming the term and its offset). */
int sb_stencil_ccheck(const sb_stencil_vterm *terms, int n, const int64_t radius27[27], int ncolours);
/* Host only.  The SOR update of A u = f (f on aux): u <- u + omega (f - A u) / a_c, for a constant-coefficient op A with
 * exactly one src term at offset 0 (weight a_c != 0) and no aux term.  Terms, in order, weights in double with exactly
 * this association: the centre (src, 0, 1 - omega); each off-centre src term (src, o, w) of A, in A's order, as
 * (src, o, (-omega * w) / a_c); then (aux, 0, omega / a_c).  omega = 1 is Gauss-Seidel (in a coloured sweep) or Jacobi
 * (out of place); 0 < omega < 2 is over- / under-relaxation.  omega outside (0, 2) is accepted but diverges for a
 * symmetric positive definite A.  Writes at most cap terms (out may be NULL with cap 0) and returns n + 1, or
 * SB_ERR_INVALID for an invalid term list, no centre term, two centre terms, a_c = 0, an aux term or omega not finite. */
int sb_stencil_relax(const sb_stencil_term *A, int n, double omega, sb_stencil_term *out, int cap);
/* sb_stencil_vplan_create with a colouring: ncolours m and colour c.  sb_stencil_vplan_create is this call with m = 1,
 * c = 0.  Errors beyond sb_stencil_vplan_create's (SB_ERR_INVALID with a message, before anything is allocated): m not 1,
 * 2 or 8, c outside 0 .. m-1, a term that reads its own colour; dst == src only when m = 1.  sb_stencil_plan_bytes of a
 * coloured plan counts the reads of every cell of the boxes and one element written per cell of the colour. */
int sb_stencil_cplan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                            sb_pitched src, sb_pitched aux, const sb_pitched *coef, int ncoef, int ncolours, int colour,
                            const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi);
/* Diagonal relaxation (DESIGN.md section 2.12): a relaxation sweep of A u = f for an op A whose diagonal varies from
 * cell to cell, such as div(kappa grad u).  A is an op of src terms only (plain or coefficient terms, no aux term, at
 * least one term at offset 0); f is on aux (the `f` argument); omega is the relaxation factor.  For every cell p of
 * colour c under the colouring m, in T with every operation rounded separately (no FMA contraction):
 *   for each term t in list order: k_t = T(w_t), or T(w_t) * C_k(p + c_t) for a coefficient term; m_t = k_t * u(p + o_t);
 *     a = m_0, then a = a + m_t (the op rule above, unchanged)
 *   d = the sum of the factors k_t of the terms with o_t = 0, in list order (the first, then d = d + k_t)
 *   dst[p] = u(p) + T(omega) * ((f(p) - a) / d), with an IEEE round-to-nearest divide
 * With m > 1 dst may be src (in place) and the colour condition applies; with m = 1 and dst != src it is weighted
 * Jacobi.  d = 0 or a non-finite d gives whatever IEEE arithmetic gives; it is not checked.  Errors beyond
 * sb_stencil_cplan_create's (SB_ERR_INVALID with a message, before anything is allocated): an aux term in A, no term
 * at offset 0, omega not finite, f NULL.  sb_stencil_plan_bytes counts as for a coloured plan, f as the aux read. */
int sb_stencil_dplan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                            sb_pitched src, sb_pitched f, const sb_pitched *coef, int ncoef, double omega, int ncolours, int colour,
                            const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi);

/* ---------------------------------------------------------------------------------------------
 * Linear stencil systems: one launch over nin input and nout output allocations.  A term of output j reads input
 * `input` at p + o (|o_a| <= SB_STENCIL_MAX_REACH) and, if coef >= 0, input `coef` at p + c (|c_a| <=
 * SB_STENCIL_COEF_REACH) as its coefficient.  For each output j, over the terms with output == j in list order (terms of
 * different outputs may interleave), in T with every multiply and add rounded separately (no FMA contraction):
 *   coefficient term  m = (T(w) * I_coef(p + c)) * I_in(p + o)
 *   plain term        m = T(w) * I_in(p + o)
 *   acc = m_first;  acc = acc + m for each later term;  O_j[p] = acc
 * A system with one output, src as input 0, aux as input 1 and coefficient field k as input 2 + k gives the bits of
 * sb_stencil_vplan_create.  Aliasing: outputs are pairwise distinct buffers; an output may be an input only if every
 * read of that input (as a source or a coefficient, by any output's terms) is at offset 0; every read of a cell happens
 * before any output of that cell is written.  An input no term reads may be NULL; it is neither checked nor counted.
 * ------------------------------------------------------------------------------------------- */
#define SB_STENCIL_SYS_MAX_INPUTS 8
#define SB_STENCIL_SYS_MAX_OUTPUTS 4
#define SB_STENCIL_SYS_MAX_TERMS 128
typedef struct sb_stencil_sys_term {
  int32_t output;         /* 0 .. nout-1 */
  int32_t input;          /* the source read: 0 .. nin-1 */
  int32_t offset[3];      /* |o_a| <= SB_STENCIL_MAX_REACH */
  int32_t coef;           /* an input read as coefficient, or -1 */
  int32_t coef_offset[3]; /* |c_a| <= SB_STENCIL_COEF_REACH; (0,0,0) when coef = -1 */
  double weight;
} sb_stencil_sys_term;

/* Host only.  The limits (1 .. SB_STENCIL_SYS_MAX_TERMS terms, 1 .. 8 inputs, 1 .. 4 outputs, indices in range, the
 * offset limits above) and the reach test of sb_stencil_check on every source and coefficient offset. */
int sb_stencil_sys_check(const sb_stencil_sys_term *terms, int n, int nin, int nout, const int64_t radius27[27]);
/* Host only.  Difference tables on a grid of spacing[3] (weights in double).  stagger +1: forward, D_a u = (u(p + e_a) -
 * u(p)) / h_a, terms (+e_a, 1/h_a) then (0, -1/h_a); -1: backward, (0, 1/h_a) then (-e_a, -1/h_a); 0: central,
 * (+e_a, 0.5/h_a) then (-e_a, -0.5/h_a).
 *   grad: input 0 -> outputs 0, 1, 2 (D_x, D_y, D_z); 6 terms
 *   div:  inputs 0, 1, 2 -> output 0 (D_x in 0 + D_y in 1 + D_z in 2, in that order); 6 terms
 *   curl: output 0 = D_y in 2 - D_z in 1, output 1 = D_z in 0 - D_x in 2, output 2 = D_x in 1 - D_y in 0, the positive
 *         part first; 12 terms
 * Each writes at most cap terms (out may be NULL with cap 0) and returns the term count, or SB_ERR_INVALID for a
 * stagger outside -1 .. 1 or a spacing that is not finite and > 0.  A forward curl for H and a backward curl for E are
 * the Yee scheme (DESIGN.md section 2.8). */
int sb_stencil_grad(int stagger, const double spacing[3], sb_stencil_sys_term *out, int cap);
int sb_stencil_div(int stagger, const double spacing[3], sb_stencil_sys_term *out, int cap);
int sb_stencil_curl(int stagger, const double spacing[3], sb_stencil_sys_term *out, int cap);
/* A persistent plan of the system over nbox boxes [lo, hi) (global coordinates; acc_origin as for sb_stencil_plan_create)
 * of nout outputs[] and nin inputs[] that share pitch, row count and zsize.  Boxes of at least 8 cells on every axis go
 * to the z-marching tile kernel, one launch each; thinner boxes share one-thread-per-cell launches.  Launch, bytes (per
 * cell one element read of each input a term reads and one written per output) and destroy through sb_stencil_plan_*.
 * Errors (SB_ERR_INVALID with a message, checked before anything is allocated): an unknown dtype, an invalid term list,
 * an output without terms, a NULL output or read input, two equal outputs, an output that is an input read at a
 * non-zero offset, mismatched pitches or row counts, a pointer or pitch that is not a multiple of the element size,
 * lo > hi, a box whose reads leave an allocation, and a system whose tile kernel needs more shared memory than the
 * device allows a block. */
int sb_stencil_sys_plan_create(sb_stencil_plan **out, int device, int dtype, const sb_stencil_sys_term *terms, int n,
                               const sb_pitched *outputs, int nout, const sb_pitched *inputs, int nin,
                               const int64_t acc_origin[3], int64_t zsize, int nbox, const int64_t *lo, const int64_t *hi);

/* ---------------------------------------------------------------------------------------------
 * Multigrid transfers (DESIGN.md section 2.10) between a cell-centred grid and the grid twice as coarse on every axis.
 * Coarse cell I covers the fine cells 2I + d, d in {0,1}^3; all coordinates are global compute coordinates.  In the
 * quantity's type T with every multiply and add rounded separately (no FMA contraction); every weight is exact in T.
 *   Restriction, the 8-cell average, for each coarse cell I of a box:
 *     acc = F(2I + (0,0,0));  acc = acc + F(2I + d) for d = (1,0,0), (0,1,0), (1,1,0), (0,0,1), (1,0,1), (0,1,1), (1,1,1)
 *     C[I] = T(0.125) * acc
 *   It reads only fine cells inside the coarse cells' footprint: no fine ghost cells, no exchange.
 *   Prolongation, trilinear, for each fine cell p of a box: parent P = floor(p / 2) per axis, side s_a = +1 if p_a is
 *   odd, else -1, and
 *     acc = T(27/64) * E[P]
 *     acc = acc + T(9/64) * E[P + s_x e_x];  acc = acc + T(9/64) * E[P + s_y e_y];  acc = acc + T(9/64) * E[P + s_z e_z]
 *     acc = acc + T(3/64) * E[P + s_x e_x + s_y e_y];  then (x, z), then (y, z)
 *     acc = acc + T(1/64) * E[P + s]
 *     dst[p] = aux[p] + acc, or dst[p] = acc without aux
 *   aux may be dst (each cell's aux value is read before that cell is written, by the same thread): u <- u + P e in
 *   place.  dst must not be src.  It reads coarse cells within +-1 of the parent box on every axis, corners included,
 *   so the coarse quantity needs one exchanged ghost layer in all 26 directions.
 * Walls need nothing special: the coarse ghost cells come from the coarse domain's own BC.  ODD(c) and EVEN mirror about
 * the wall face, which is the same plane on both grids, so trilinear interpolation reproduces the linear extrapolation
 * to the wall.  VALUE(c) pins the ghost cell's centre, h/2 beyond the face, and h differs between the grids, so a cycle
 * with VALUE walls on every level is not consistent.
 * ------------------------------------------------------------------------------------------- */
typedef enum sb_transfer_kind { SB_TRANSFER_RESTRICT = 0, SB_TRANSFER_PROLONG = 1 } sb_transfer_kind;
/* Host only.  Whether a fine and a coarse partition pair for transfers that stay on each subdomain's GPU: the same dim,
 * and for every subdomain index (x fastest, fine_dim[0] * fine_dim[1] * fine_dim[2] of them, 3 int64 each) fine origin
 * = 2 * coarse origin and fine size = 2 * coarse size.  coarse_radius27 (the coarse ghost widths) may be NULL, for
 * restriction only; otherwise every one of the 26 directions needs a radius >= 1, as prolongation reads one ghost layer.
 * SB_ERR_INVALID with a message naming the subdomain index and axis, or the missing ghost direction. */
int sb_transfer_check(const int64_t fine_dim[3], const int64_t coarse_dim[3], const int64_t *fine_origin, const int64_t *fine_size,
                      const int64_t *coarse_origin, const int64_t *coarse_size, const int64_t coarse_radius27[27]);
/* A persistent plan of one transfer over the box [lo, hi) of dst, in dst's global coordinates: coarse cells for
 * SB_TRANSFER_RESTRICT (dst coarse, src fine), fine cells for SB_TRANSFER_PROLONG (dst fine, src coarse).  Each
 * allocation has its own pitch, row count, zsize and acc_origin (the global coordinate of its element (0,0,0), as for
 * sb_jacobi3d); aux (prolongation only; ptr NULL: none) shares dst's.  dtype SB_DTYPE_F32 or SB_DTYPE_F64.  Errors
 * (SB_ERR_INVALID with a message, before anything is allocated): an unknown dtype or kind, a NULL dst or src, dst == src,
 * aux given to a restriction, aux with another pitch or row count than dst, a pointer or pitch that is not a multiple of
 * the element size, lo > hi, a box outside dst's allocation, and reads that leave src's allocation (restriction: fine
 * [2 lo, 2 hi); prolongation: coarse [floor(lo / 2) - 1, floor((hi - 1) / 2) + 2) on every axis).  The kernels take
 * allocation coordinates as 32-bit int, so a box or read window that ends past 2^31 - 1 on some axis, a box of 2^32 cells
 * or more, and a prolongation whose 2 * src_acc_origin - dst_acc_origin does not fit 32 bits are SB_ERR_INVALID too, with
 * a message naming the axis; the fused restrictions below check their fine windows the same way.
 * sb_transfer_plan_launch allocates nothing and never synchronises the host.  sb_transfer_plan_bytes: the algorithmic
 * bytes of a launch, every element the rule reads counted once and one element written per cell of the box. */
typedef struct sb_transfer_plan sb_transfer_plan;
int sb_transfer_plan_create(sb_transfer_plan **out, int device, int dtype, int kind, sb_pitched dst, const int64_t dst_acc_origin[3],
                            int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3], int64_t src_zsize, sb_pitched aux,
                            const int64_t lo[3], const int64_t hi[3]);
int sb_transfer_plan_launch(sb_transfer_plan *plan, void *stream);
int64_t sb_transfer_plan_bytes(const sb_transfer_plan *plan);
int sb_transfer_plan_destroy(sb_transfer_plan *plan);
/* Fused residual-restriction (DESIGN.md section 2.11): a plain op (the rule of sb_stencil_plan_create, terms on src and
 * aux) of reach <= 1 on every axis, evaluated on the fine grid and restricted without storing the fine values.  For
 * each coarse cell I of the boxes:
 *   v(p) = op(p) for the eight fine cells p = 2I + d, by the linear stencil rule above, in T, no FMA contraction
 *   C[I] = the restriction above of those eight values, in its order, times T(0.125)
 * The result is the bits of sb_stencil_plan over the fine footprint into a scratch allocation followed by
 * SB_TRANSFER_RESTRICT.  For multigrid the op is the residual: (aux, 0, 1), then (src, o, -w) for each term of A.
 * dst is coarse; src and aux (ptr NULL: none; needed when a term reads aux) are fine and share src's pitch and row
 * count; each acc_origin is the global coordinate of its allocation's element (0,0,0).  nbox boxes [lo, hi) of coarse
 * global coordinates (nbox * 3 int64 each).  Boxes of at least 4 coarse cells on every axis go to a z-marching tile
 * kernel, one launch each; thinner boxes share one-thread-per-coarse-cell launches of up to 16 boxes.  Launch, bytes
 * (per coarse cell of the boxes: 8 x (one src element, plus one aux element if a term reads aux), plus one coarse
 * element written) and destroy go through sb_transfer_plan_*.  Errors (SB_ERR_INVALID with a message, before anything
 * is allocated): an unknown dtype, an invalid term list, an offset beyond 1 cell, an aux term without aux, a NULL dst
 * or src, dst equal to src or aux, aux with another pitch or row count than src, a pointer or pitch that is not a
 * multiple of the element size, lo > hi, a box outside dst's allocation, and fine reads [2 lo - 1, 2 hi + 1) that leave
 * src's allocation on some axis. */
int sb_transfer_oplan_create(sb_transfer_plan **out, int device, int dtype, const sb_stencil_term *terms, int n, sb_pitched dst,
                             const int64_t dst_acc_origin[3], int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3],
                             int64_t src_zsize, sb_pitched aux, int nbox, const int64_t *lo, const int64_t *hi);
/* sb_transfer_oplan_create for an op with coefficient terms (DESIGN.md section 2.12): the same rule, the factor of a
 * coefficient term being T(w) * C_k(p + c) as in sb_stencil_vplan_create, so the result is the bits of
 * sb_stencil_vplan_create over the fine footprint into a scratch allocation followed by SB_TRANSFER_RESTRICT.  coef:
 * ncoef (<= 4) fine fields that share src's pitch, row count, zsize and acc_origin; coefficient offsets reach at most 1.
 * Boxes go to the kernels of sb_transfer_oplan_create, which read the fields through the read-only cache at each term's
 * coefficient offset.  Bytes as sb_transfer_oplan_create's plus 8 elements per
 * coarse cell of each field a term reads.  Errors: sb_transfer_oplan_create's, plus a field index out of range, a NULL
 * field a term names, a field that is dst, and a field with another pitch or row count than src. */
int sb_transfer_voplan_create(sb_transfer_plan **out, int device, int dtype, const sb_stencil_vterm *terms, int n, sb_pitched dst,
                              const int64_t dst_acc_origin[3], int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3],
                              int64_t src_zsize, sb_pitched aux, const sb_pitched *coef, int ncoef, int nbox, const int64_t *lo,
                              const int64_t *hi);
/* Face-coefficient restriction (DESIGN.md section 2.12): a field of values on the faces normal to axis `axis` (C_a(p) on
 * the face between p - e_a and p, the convention of sb_stencil_div_grad) to the coarse grid.  With b < c the two other
 * axes, for each coarse cell I of the box [lo, hi) of dst (coarse global coordinates), in T:
 *   C[I] = T(0.25) * (((F(2I) + F(2I + e_b)) + F(2I + e_c)) + F(2I + e_b + e_c))
 * the four fine faces that make up coarse face I.  It reads only inside the footprint (no fine ghost cells).  Buffers,
 * launch, bytes (4 fine elements read and one written per coarse cell) and destroy as for SB_TRANSFER_RESTRICT, whose
 * errors it shares, plus an axis outside 0 .. 2. */
int sb_transfer_fplan_create(sb_transfer_plan **out, int device, int dtype, int axis, sb_pitched dst, const int64_t dst_acc_origin[3],
                             int64_t dst_zsize, sb_pitched src, const int64_t src_acc_origin[3], int64_t src_zsize,
                             const int64_t lo[3], const int64_t hi[3]);

/* ---------------------------------------------------------------------------------------------
 * 7-point jacobi step (the reference's user kernel, bin/jacobi3d.cu:40-85) over a region.
 * dtype_size 4 = float, 8 = double.  acc_origin = global coordinate of allocation element (0,0,0)
 * (Accessor origin, include/stencil/local_domain.cuh:153-173).  [lo,hi) = region to update,
 * [clo,chi) = the whole distributed compute region (hot/cold sphere placement).
 * dst[p] = 1 in the hot sphere, 0 in the cold sphere, else ((((((0+px)+mx)+py)+my)+pz)+mz)/6 with
 * IEEE round-to-nearest division (bit-identical to the CPU oracle).
 * ------------------------------------------------------------------------------------------- */
int sb_jacobi3d(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3],
                const int64_t hi[3], const int64_t clo[3], const int64_t chi[3], void *stream);
/* The same update over n <= 8 regions in ONE launch: the exterior slabs of a subdomain
 * (bin/jacobi3d.cu:324-342 launches stencil_kernel once per slab).  lo/hi are n*3 int64. */
int sb_jacobi3d_regions(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], int n,
                        const int64_t *lo, const int64_t *hi, const int64_t clo[3], const int64_t chi[3], void *stream);
/* ---------------------------------------------------------------------------------------------
 * Astaroth MHD substep: replaces `integrate_substep` + `solve<step>` of the reference's astaroth extract
 * (astaroth/kernels.cu:62-87, astaroth/user_kernels.h:437-469, astaroth/integration.cuh:14-52).
 * in / out: the VertexBufferArray (astaroth/kernels.h:22-27): 8 device arrays each, order lnrho, uux, uuy, uuz,
 * ax, ay, az, entropy (astaroth/user_defines.h:112-120), all of raw size raw[3] = (mx, my, mz) elements, x fastest,
 * including the radius-3 ghost cells.  [lo, hi): box to update in the reference's memory-offset coordinates
 * (what the driver passes as Rect3 cr, astaroth/astaroth.cu:563-566); every cell needs 3 allocated cells around it.
 * step 0..2 = Williamson RK3 substep; step 0 ignores the previous contents of `out`.
 * params: the uniforms solve<> reads through DCONST (acDeviceLoadMeshInfo / acDeviceLoadScalarUniform,
 * astaroth/kernels.cu:89-163).  variant: 0 auto, 1 cell kernel, 2 tile kernel (one thread per cell), 3 team kernel (two specialised
 * threads per cell on the same shared-memory ring; FP64: ring fed by TMA when the buffers allow it), 4 / 5 the TMA-fed
 * two- / three-team kernel or an error.
 * dtype_size 8 = double (the reference's AcReal), 4 = float.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  double inv_dsx, inv_dsy, inv_dsz;
  double dt;
  double cs2_sound, gamma, cp_sound, lnrho0, lnT0;
  double mu0, nu_visc, zeta, eta;
} sb_astaroth_params;
int sb_astaroth_substep(int step, const void *const in[8], void *const out[8], int dtype_size, const int64_t raw[3],
                        const int64_t lo[3], const int64_t hi[3], const sb_astaroth_params *params, int variant, void *stream);
/* The jacobi step over the WHOLE compute region of a subdomain with the halo exchange of the NEXT iteration fused
 * into it: every cell on a face of [lo, hi) is also stored into the ghost cell of the face neighbour that reads it
 * next iteration.  Replaces, per iteration, the interior stencil_kernel launch + DistributedDomain::exchange()
 * (src/stencil.cu:1002-1186: pack -> copy -> unpack of 6 face messages) + the <= 6 exterior launches of
 * bin/jacobi3d.cu:296-368 by one kernel; results are bit-identical.  Face radius 1 only (bin/jacobi3d.cu:237-246).
 * nbr[d], d = -x,+x,-y,+y,-z,+z: the neighbour's OUTPUT allocation of this iteration (its `next` buffer; may be this
 * subdomain's own dst for a periodic self-neighbour, or a peer GPU's memory mapped by peer access / CUDA IPC);
 * nbr_zsize[d]: planes of that allocation.  ptr == NULL: nothing is pushed in that direction.  The neighbour must
 * have the same extent as this subdomain on the two axes orthogonal to d (always true for a grid partition).
 * The caller orders iterations: this launch may start once every neighbour has finished the previous iteration. */
typedef struct {
  sb_pitched nbr[6];
  int64_t nbr_zsize[6];
  /* Dense x faces (x neighbour owned by another rank): if x_dense[s] != 0 (s = 0: -x side, 1: +x side), nbr[s].ptr is
   * not a field allocation but a dense array in the NEIGHBOUR's memory, (rows x planes) elements indexed [y][z] (z
   * fastest, like the march) in THIS subdomain's allocation coordinates; nbr[s].ysize = rows, nbr_zsize[s] = planes.
   * The kernel stages the column in shared memory and writes 256-byte lines instead of one 8-byte store per row and
   * plane.  x_recv[s], if not NULL, is such an array (this subdomain's rows x planes) received FROM the neighbour on
   * side s: the out-of-subdomain x neighbour of the first / last column is read from it instead of from the ghost
   * column of src.  Needs a 16-byte aligned first compute cell and whole warp strips along x. */
  int64_t x_dense[2];
  const void *x_recv[2];
} sb_halo_push;
int sb_jacobi3d_fused(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3],
                      const int64_t hi[3], const int64_t clo[3], const int64_t chi[3], const sb_halo_push *push, void *stream);
/* The same launch with the ordering BETWEEN RANKS inside the kernel, replacing the reference's per-iteration host
 * synchronisation (DistributedDomain::exchange() returns after MPI_Waitall / stream syncs, src/stencil.cu:1120-1186;
 * bin/jacobi3d.cu:337-365) and this library's own sb_wait / sb_signal launches.
 * Every boundary tile of the kernel (256 threads: one 32-lane strip x 8 rows x one z chunk of 32 planes) parks its face
 * cells in shared memory while it marches and stores them into the neighbour when it is done; there is no fence and no
 * flag per tile.  Instead the FIRST CTA of the launch writes signal_value (release, system scope) into signal_rows[f][0]
 * for every face f with a row -- a uint32 word in the NEIGHBOUR's memory (peer / IPC mapped): its mailbox for the face it
 * shares with this subdomain.  The kernel boundary has completed every store of the previous launch on this stream, so
 * the word says "my previous iteration is complete, pushes and reads".  Before marching, a CTA on face f polls
 * wait_rows[f][0] (this GPU's own mailbox for face f, written by the neighbour across f; ld.acquire.sys) until
 * (int32)(word - wait_value) >= 0.  Protocol: the launch of iteration e carries wait_value = signal_value = e -- a
 * neighbour that has STARTED iteration e has (a) filled the ghost cells iteration e reads here and (b) stopped reading
 * the ghost cells iteration e overwrites there.  Tiles that touch no face never wait.  (One release per boundary tile
 * was slower on 8 ranks -- the releasing warp lingers for an NVLink round trip and keeps its CTA slot -- than the skew
 * between the ranks' kernel starts that one release per kernel costs.)
 * Faces: -x,+x,-y,+y,-z,+z.  NULL rows: no wait / no signal on that face (neighbour in the same process: order the
 * launches with stream events).  sync == NULL: no handshake at all.  The rows keep SB_FUSED_MAX_GROUPS words (the
 * per-tile protocol's size); only word 0 is used. */
#define SB_FUSED_MAX_GROUPS 4096
typedef struct {
  const uint32_t *wait_rows[6];
  uint32_t *signal_rows[6];
  uint32_t wait_value, signal_value;
} sb_step_sync;
int sb_jacobi3d_fused_sync(sb_pitched dst, sb_pitched src, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3],
                           const int64_t hi[3], const int64_t clo[3], const int64_t chi[3], const sb_halo_push *push,
                           const sb_step_sync *sync, void *stream);
/* init_kernel, bin/jacobi3d.cu:18-29: fill region with a constant */
int sb_fill(sb_pitched dst, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3], const int64_t hi[3],
            double value, void *stream);
/* sum over [lo,hi) of (a-b)^2 accumulated in double into *out_dev (device double, zeroed by the
 * call): the FP64 residual BASELINE.json asks for (not in the reference). */
int sb_sqdiff(sb_pitched a, sb_pitched b, int dtype_size, const int64_t acc_origin[3], const int64_t lo[3],
              const int64_t hi[3], double *out_dev, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Device memory + peer plumbing used by the host layers (C++ and Python).
 * ------------------------------------------------------------------------------------------- */
int sb_device_count(int *count);
int sb_malloc(void **ptr, size_t bytes, int device);
int sb_free(void *ptr, int device);
int sb_memset(void *ptr, int value, size_t bytes, int device, void *stream);
/* cudaMemcpyAsync(cudaMemcpyDefault) on `stream` of `device`: host<->device and device<->device (UVA).
 * Host buffers should be pinned for the copy to be asynchronous. */
int sb_memcpy(void *dst, const void *src, size_t bytes, int device, void *stream);
int sb_stream_sync(int device, void *stream);
int sb_device_sync(int device);
/* cudaDeviceEnablePeerAccess both ways if possible (gpu_topo::enable_peer, src/gpu_topology.cpp:97-129);
 * *ok = 1 when src can address dst's memory. */
int sb_enable_peer(int src_device, int dst_device, int *ok);
/* CUDA IPC handle export / import (cudaIpcGetMemHandle / OpenMemHandle, tx_cuda.cuh:225-243). handle = 64 bytes. */
int sb_ipc_export(void *ptr, void *handle64);
int sb_ipc_import(const void *handle64, int device, void **ptr);
int sb_ipc_close(void *ptr, int device);

#ifdef __cplusplus
}
#endif
#endif /* STENCIL_B200_H */
