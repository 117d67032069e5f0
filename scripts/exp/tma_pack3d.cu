// TMA 3-D pack experiment (VERDICT r1 item 8): the halo pack of wide-row messages as north_star words it -- "TMA 3D tiled
// loads from the strided subdomain into shared-memory staging then 128-bit vectorised coalesced stores to a contiguous send
// buffer" -- with boxes of >= 16 KiB per instruction (the round-1 tiles were bx x 1 x 1, <= 2 KiB), two producer warps and a
// 3-stage ring of 32 KiB stages, against the library's LSU path (sb_pack) on the same messages:
//   y / z faces of a 512^3 FP32 / FP64 subdomain with radius 2 and 3, and one field-face of the astaroth exchange
//   (256^3, radius 3, FP64).
// Build (nvcc needs no GPU; run it on an H100):
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -Iinclude scripts/exp/tma_pack3d.cu -o scripts/exp/tma_pack3d \
//        -Lstencil_b200 -lstencil_b200 -Xlinker -rpath -Xlinker '$ORIGIN/../../stencil_b200'
// Prints one line per message: payload, LSU us, TMA us, GB/s (read + write) each, and whether the packed bytes agree.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "stencil_b200.h"

#define CK(x)                                                                                                          \
  do {                                                                                                                 \
    cudaError_t e_ = (x);                                                                                              \
    if (e_ != cudaSuccess) {                                                                                           \
      fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));                                       \
      exit(1);                                                                                                         \
    }                                                                                                                  \
  } while (0)

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *, const cuuint32_t *,
                             const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

constexpr int kStages = 3;
constexpr int kStageBytes = 32 * 1024;
constexpr int kThreads = 256; // warps 0, 1: producers (one elected lane each); all 8 warps drain

__device__ __forceinline__ unsigned s32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *b, unsigned n) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s32(b)), "r"(n) : "memory"); }
__device__ __forceinline__ void mbar_expect(unsigned long long *b, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned long long *b, unsigned parity) {
  asm volatile("{\n.reg .pred p;\nW_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra D_%=;\nbra W_%=;\nD_%=:\n}\n" ::"r"(s32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma3(void *smem, const CUtensorMap *map, unsigned long long *bar, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(s32(smem)), "l"(map),
               "r"(s32(bar)), "r"(x), "r"(y), "r"(z)
               : "memory");
}

// The message is the box [pos, pos + ext) of a 3-D tensor; it is cut into tiles of (bx, by, bz) elements (one TMA box each).
// dst is dense, x fastest: element (x, y, z) of the message at ((z * ext.y + y) * ext.x + x) * es.
struct Msg {
  int pos[3], ext[3], box[3], tiles[3];
  int es;
  int pre; // a box must START on a 16-byte address (measured in round 1): tiles begin `pre` elements before pos.x
  int vec; // bytes per store of the drain: 16 when pre * es is a multiple of 16, else 8
};

__global__ void __launch_bounds__(kThreads) tma_pack_kernel(const __grid_constant__ CUtensorMap map, const __grid_constant__ Msg m, char *__restrict__ dst, int ntiles) {
  extern __shared__ __align__(1024) unsigned char smem[];
  __shared__ unsigned long long full[kStages], empty[kStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) mbar_init(&full[i], 1), mbar_init(&empty[i], kThreads);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const unsigned box_bytes = unsigned(m.box[0]) * m.box[1] * m.box[2] * m.es;
  // this CTA's tiles: blockIdx.x, + gridDim.x, ...
  const int mine = (ntiles - int(blockIdx.x) + int(gridDim.x) - 1) / int(gridDim.x);
  auto coords = [&](int t, int &tx, int &ty, int &tz) {
    tx = t % m.tiles[0];
    t /= m.tiles[0];
    ty = t % m.tiles[1];
    tz = t / m.tiles[1];
  };
  auto issue = [&](int k) { // by the elected producer lane of tile k
    const int s = k % kStages;
    int tx, ty, tz;
    coords(int(blockIdx.x) + k * int(gridDim.x), tx, ty, tz);
    mbar_expect(&full[s], box_bytes);
    tma3(smem + s * kStageBytes, &map, &full[s], m.pos[0] - m.pre + tx * m.box[0], m.pos[1] + ty * m.box[1], m.pos[2] + tz * m.box[2]);
  };
  // producers: lane 0 of warp k % 2 issues tile k; the first kStages tiles need no wait
  if (warp < 2 && lane == 0)
    for (int k = warp; k < mine && k < kStages; k += 2) issue(k);
  // consumers: everybody (the producer lanes join after issuing; their loop above only blocks on stages k - 3)
  for (int k = 0; k < mine; ++k) {
    const int s = k % kStages, use = k / kStages;
    mbar_wait(&full[s], use & 1);
    int tx, ty, tz;
    coords(int(blockIdx.x) + k * int(gridDim.x), tx, ty, tz);
    const int y0 = ty * m.box[1], z0 = tz * m.box[2];
    // message x range covered by this tile: tile tx holds allocation x in [pos.x - pre + tx * box.x, + box.x)
    const int xa = max(0, tx * m.box[0] - m.pre), xb = min(m.ext[0], (tx + 1) * m.box[0] - m.pre); // message-relative
    const int soff = (xa + m.pre - tx * m.box[0]) * m.es;                                         // byte offset inside a tile row
    const int ny = min(m.box[1], m.ext[1] - y0), nz = min(m.box[2], m.ext[2] - z0);
    const int rowv = ((xb - xa) * m.es) / m.vec; // vectors per row of the tile
    const int rows = ny * nz;
    const unsigned char *img = smem + s * kStageBytes;
    const int pitch = m.box[0] * m.es;
    for (int i = tid; i < rows * rowv; i += kThreads) {
      const int r = i / rowv, c = i - r * rowv;
      const int zz = r / ny, yy = r - zz * ny;
      const unsigned char *sp = img + (zz * m.box[1] + yy) * pitch + soff + c * m.vec;
      char *d = dst + ((long long)((z0 + zz) * m.ext[1] + (y0 + yy)) * m.ext[0] + xa) * m.es + c * m.vec;
      if (m.vec == 16) *reinterpret_cast<uint4 *>(d) = *reinterpret_cast<const uint4 *>(sp);
      else *reinterpret_cast<uint2 *>(d) = *reinterpret_cast<const uint2 *>(sp);
    }
    mbar_arrive(&empty[s]);
    // refill this stage with tile k + kStages once everybody has drained it
    const int kn = k + kStages;
    if (kn < mine && lane == 0 && warp == kn % 2) {
      mbar_wait(&empty[s], use & 1);
      issue(kn);
    }
  }
}

static EncodeFn encoder() {
  void *fp = nullptr;
  cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q));
  return (EncodeFn)fp;
}

struct Case {
  const char *name;
  int n, r, es;
  int dir; // 1 = +y face, 2 = +z face
};

int main() {
  EncodeFn enc = encoder();
  const Case cases[] = {{"512^3 f32 r=2 y-face", 512, 2, 4, 1}, {"512^3 f32 r=2 z-face", 512, 2, 4, 2}, {"512^3 f32 r=3 y-face", 512, 3, 4, 1},
                        {"512^3 f32 r=3 z-face", 512, 3, 4, 2}, {"512^3 f64 r=2 y-face", 512, 2, 8, 1}, {"512^3 f64 r=2 z-face", 512, 2, 8, 2},
                        {"256^3 f64 r=3 y-face (astaroth field)", 256, 3, 8, 1}, {"256^3 f64 r=3 z-face (astaroth field)", 256, 3, 8, 2}};
  int sms = 132;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  CK(cudaFuncSetAttribute(tma_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStages * kStageBytes));
  for (const Case &c : cases) {
    const int raw = c.n + 2 * c.r;
    const size_t bytes = size_t(raw) * raw * raw * c.es;
    char *src = nullptr, *d_lsu = nullptr, *d_tma = nullptr;
    CK(cudaMalloc(&src, bytes));
    std::vector<uint32_t> h(bytes / 4);
    for (size_t i = 0; i < h.size(); ++i) h[i] = uint32_t(i * 2654435761u);
    CK(cudaMemcpy(src, h.data(), bytes, cudaMemcpyHostToDevice));
    Msg m{};
    m.es = c.es;
    // the outermost compute cells on the +y / +z side (what a pack sends), x extent = the compute cells
    m.pos[0] = c.r, m.pos[1] = c.dir == 1 ? c.n : c.r, m.pos[2] = c.dir == 2 ? c.n : c.r;
    m.ext[0] = c.n, m.ext[1] = c.dir == 1 ? c.r : c.n, m.ext[2] = c.dir == 2 ? c.r : c.n;
    // box: 256 elements of a row (<= 2 KiB), as many rows / planes as fit in 32 KiB
    m.box[0] = 256;
    if (c.dir == 1) { // r rows per plane, planes apart: box (256, r, nzb)
      m.box[1] = c.r;
      m.box[2] = kStageBytes / (256 * c.es * c.r);
      if (m.box[2] > 256) m.box[2] = 256;
    } else { // whole planes of rows: box (256, nyb, 1)
      m.box[1] = kStageBytes / (256 * c.es);
      if (m.box[1] > 256) m.box[1] = 256;
      m.box[2] = 1;
    }
    m.pre = ((m.pos[0] * c.es) % 16) / c.es;
    m.vec = m.pre == 0 ? 16 : 8;
    for (int a = 0; a < 3; ++a) m.tiles[a] = (m.ext[a] + (a == 0 ? m.pre : 0) + m.box[a] - 1) / m.box[a];
    const int ntiles = m.tiles[0] * m.tiles[1] * m.tiles[2];
    const size_t payload = size_t(m.ext[0]) * m.ext[1] * m.ext[2] * c.es;
    CK(cudaMalloc(&d_lsu, payload));
    CK(cudaMalloc(&d_tma, payload));
    CK(cudaMemset(d_tma, 0, payload));
    CUtensorMap map;
    const cuuint64_t dims[3] = {cuuint64_t(raw), cuuint64_t(raw), cuuint64_t(raw)};
    const cuuint64_t strides[2] = {cuuint64_t(raw) * c.es, cuuint64_t(raw) * raw * c.es};
    const cuuint32_t box[3] = {cuuint32_t(m.box[0]), cuuint32_t(m.box[1]), cuuint32_t(m.box[2])}, estr[3] = {1, 1, 1};
    const CUresult r = enc(&map, c.es == 8 ? CU_TENSOR_MAP_DATA_TYPE_UINT64 : CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, src, dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      printf("%-40s tensor map rejected (%d): rows of %d bytes\n", c.name, int(r), raw * c.es);
      continue;
    }
    const int64_t pos[3] = {m.pos[0], m.pos[1], m.pos[2]}, ext[3] = {m.ext[0], m.ext[1], m.ext[2]};
    const sb_pitched sp{src, int64_t(raw) * c.es, raw};
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const int grid = ntiles < 2 * sms ? ntiles : 2 * sms;
    auto time = [&](auto fn) {
      for (int i = 0; i < 5; ++i) fn();
      CK(cudaDeviceSynchronize());
      float best = 1e9f;
      for (int rep = 0; rep < 5; ++rep) {
        CK(cudaEventRecord(e0));
        for (int i = 0; i < 20; ++i) fn();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms;
        CK(cudaEventElapsedTime(&ms, e0, e1));
        best = ms / 20 < best ? ms / 20 : best;
      }
      return best * 1e3f;
    };
    const float us_lsu = time([&] {
      if (sb_pack(d_lsu, sp, pos, ext, c.es, nullptr) != SB_OK) {
        fprintf(stderr, "sb_pack: %s\n", sb_last_error());
        exit(1);
      }
    });
    const float us_tma = time([&] { tma_pack_kernel<<<grid, kThreads, kStages * kStageBytes>>>(map, m, d_tma, ntiles); });
    CK(cudaGetLastError());
    std::vector<char> a(payload), b(payload);
    CK(cudaMemcpy(a.data(), d_lsu, payload, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(b.data(), d_tma, payload, cudaMemcpyDeviceToHost));
    const bool same = 0 == memcmp(a.data(), b.data(), payload);
    printf("%-40s payload %6.2f MB  box %3dx%3dx%3d = %5.1f KiB, %4d tiles on %3d CTAs | LSU (sb_pack) %6.2f us %6.0f GB/s | TMA 3-D %6.2f us %6.0f GB/s | %s\n",
           c.name, payload / 1e6, m.box[0], m.box[1], m.box[2], m.box[0] * m.box[1] * m.box[2] * c.es / 1024.0, ntiles, grid, us_lsu, 2 * payload / us_lsu / 1e3,
           us_tma, 2 * payload / us_tma / 1e3, same ? "bytes agree" : "MISMATCH");
    cudaFree(src);
    cudaFree(d_lsu);
    cudaFree(d_tma);
  }
  return 0;
}
