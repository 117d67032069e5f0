// Golden-vector generator for the astaroth solve<step> kernels: runs the UNMODIFIED reference kernels
// (<reference>/astaroth/kernels.cu -> integrate_substep, acDeviceLoad*) on a small periodic-free box and dumps
// the `out` fields after each of the three substeps.  Test / baseline infrastructure only (built by
// oracle/ref/build_ref.sh into oracle/_ref/, never linked by the product).
//
//   ref_astaroth_solve <n> <dt> <in.bin> <out.bin>
//
// in.bin  : 16 arrays of (n+6)^3 doubles: in[0..8) then out[0..8), x fastest (the layout LocalDomain gives the driver,
//           astaroth/astaroth.cu:462-473)
// out.bin : 3 x 8 arrays of (n+6)^3 doubles: all `out` fields after substep 0, 1, 2 (no swap in between, as in the
//           reference driver's loop, astaroth/astaroth.cu:551-640)
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "astaroth_utils.h"
#include "kernels.h"

AcResult acHostUpdateBuiltinParams(AcMeshInfo *config); // defined (non-static) in astaroth/astaroth_utils.cu:52

#define CK(x)                                                                                                          \
  do {                                                                                                                 \
    cudaError_t e_ = (x);                                                                                              \
    if (e_ != cudaSuccess) {                                                                                           \
      fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));                                       \
      exit(1);                                                                                                         \
    }                                                                                                                  \
  } while (0)

int main(int argc, char **argv) {
  if (argc < 5) {
    fprintf(stderr, "usage: %s n dt in.bin out.bin\n", argv[0]);
    return 2;
  }
  const int n = atoi(argv[1]);
  const double dt = atof(argv[2]);
  const size_t m = size_t(n) + STENCIL_ORDER;
  const size_t cells = m * m * m;

  AcMeshInfo info{};
  acLoadConfig(AC_DEFAULT_CONFIG, &info);
  info.int_params[AC_nx] = info.int_params[AC_ny] = info.int_params[AC_nz] = n;
  acHostUpdateBuiltinParams(&info);
  info.int3_params[AC_multigpu_offset] = {0, 0, 0};
  CK(cudaSetDevice(0));
  acDeviceLoadDefaultUniforms(0);
  acDeviceLoadMeshInfo(0, info);

  const bool timing_only = argv[3][0] == '-' && argv[3][1] == 0; // "-": synthetic fill, time the kernels, no dump
  std::vector<double> host(16 * cells);
  if (timing_only) {
    unsigned long long x = 88172645463325252ull;
    for (auto &v : host) {
      x ^= x << 13, x ^= x >> 7, x ^= x << 17;
      v = double(x >> 11) / double(1ull << 53) - 0.5;
    }
  } else {
    FILE *f = fopen(argv[3], "rb");
    if (!f || fread(host.data(), sizeof(double), host.size(), f) != host.size()) {
      fprintf(stderr, "cannot read %s\n", argv[3]);
      return 1;
    }
    fclose(f);
  }
  VertexBufferArray vba{};
  for (int i = 0; i < NUM_VTXBUF_HANDLES; ++i) {
    CK(cudaMalloc(&vba.in[i], cells * sizeof(double)));
    CK(cudaMalloc(&vba.out[i], cells * sizeof(double)));
    CK(cudaMemcpy(vba.in[i], &host[size_t(i) * cells], cells * sizeof(double), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(vba.out[i], &host[size_t(8 + i) * cells], cells * sizeof(double), cudaMemcpyHostToDevice));
  }
  cudaStream_t s;
  CK(cudaStreamCreate(&s));
  acDeviceLoadScalarUniform(0, s, AC_dt, dt);
  Rect3 cr(Dim3(3, 3, 3), Dim3(3 + n, 3 + n, 3 + n));
  if (timing_only) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    for (int sub = 0; sub < 3; ++sub) integrate_substep(sub, s, cr, vba);
    CK(cudaStreamSynchronize(s));
    const int reps = 5;
    for (int sub = 0; sub < 3; ++sub) {
      CK(cudaEventRecord(e0, s));
      for (int r = 0; r < reps; ++r) integrate_substep(sub, s, cr, vba);
      CK(cudaEventRecord(e1, s));
      CK(cudaEventSynchronize(e1));
      float ms = 0;
      CK(cudaEventElapsedTime(&ms, e0, e1));
      printf("ref_astaroth_solve n=%d substep %d: %.4f ms per launch (full region, block 32x1x4)\n", n, sub, ms / reps);
    }
    return 0;
  }
  FILE *g = fopen(argv[4], "wb");
  std::vector<double> res(cells);
  for (int sub = 0; sub < 3; ++sub) {
    integrate_substep(sub, s, cr, vba);
    CK(cudaStreamSynchronize(s));
    for (int i = 0; i < NUM_VTXBUF_HANDLES; ++i) {
      CK(cudaMemcpy(res.data(), vba.out[i], cells * sizeof(double), cudaMemcpyDeviceToHost));
      fwrite(res.data(), sizeof(double), cells, g);
    }
  }
  fclose(g);
  // timing of the reference kernel on the conf's own size is printed by ref_astaroth; here only a marker
  printf("ref_astaroth_solve n=%d dt=%g ok\n", n, dt);
  return 0;
}
