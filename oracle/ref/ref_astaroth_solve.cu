// Golden-vector generator for the astaroth solve<step> kernels: runs the UNMODIFIED reference kernels
// (<reference>/astaroth/kernels.cu -> integrate_substep, acDeviceLoad*) on a small periodic-free box and dumps
// the `out` fields after each of the three substeps.  Test / baseline infrastructure only (built by
// oracle/ref/build_ref.sh into oracle/_ref/, never linked by the product).
//
//   ref_astaroth_solve <n> <dt> <in.bin> <out.bin> [nx ny nz dsx dsy dsz cs2_sound gamma cp_sound lnrho0 lnT0 mu0 nu_visc zeta eta]
//
// in.bin  : 16 arrays of (nx+6)(ny+6)(nz+6) doubles: in[0..8) then out[0..8), x fastest (the layout LocalDomain gives the
//           driver, astaroth/astaroth.cu:462-473); nx = ny = nz = n unless the overrides are given
// out.bin : 3 x 8 such arrays: all `out` fields after substep 0, 1, 2 (no swap in between, as in the reference driver's
//           loop, astaroth/astaroth.cu:551-640)
// The 15 optional overrides replace the grid size, the spacings and the nine physical constants of astaroth.conf before
// the mesh info is loaded into the device constants.  AC_inv_ds* is set here as 1 / AC_ds*: acHostUpdateBuiltinParams
// derives it only `#ifdef AC_dsx`, and AC_dsx is an enumerator, not a macro, so solve<> would otherwise keep reading the
// default 1 / 0.04908738521 (user_kernels.h:33) whatever the spacing.
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
  int nn[3] = {n, n, n};
  const bool over = argc >= 5 + 15;
  if (argc > 5 && !over) {
    fprintf(stderr, "overrides: nx ny nz dsx dsy dsz cs2_sound gamma cp_sound lnrho0 lnT0 mu0 nu_visc zeta eta (all 15)\n");
    return 2;
  }
  if (over)
    for (int k = 0; k < 3; ++k) nn[k] = atoi(argv[5 + k]);
  const size_t cells = size_t(nn[0] + STENCIL_ORDER) * size_t(nn[1] + STENCIL_ORDER) * size_t(nn[2] + STENCIL_ORDER);

  AcMeshInfo info{};
  acLoadConfig(AC_DEFAULT_CONFIG, &info);
  info.int_params[AC_nx] = nn[0], info.int_params[AC_ny] = nn[1], info.int_params[AC_nz] = nn[2];
  if (over) {
    const AcRealParam real[12] = {AC_dsx, AC_dsy, AC_dsz, AC_cs2_sound, AC_gamma, AC_cp_sound,
                                  AC_lnrho0, AC_lnT0, AC_mu0, AC_nu_visc, AC_zeta, AC_eta};
    for (int k = 0; k < 12; ++k) info.real_params[real[k]] = AcReal(atof(argv[8 + k]));
  }
  acHostUpdateBuiltinParams(&info);
  if (over) {
    info.real_params[AC_inv_dsx] = AcReal(1.) / info.real_params[AC_dsx];
    info.real_params[AC_inv_dsy] = AcReal(1.) / info.real_params[AC_dsy];
    info.real_params[AC_inv_dsz] = AcReal(1.) / info.real_params[AC_dsz];
  }
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
  Rect3 cr(Dim3(3, 3, 3), Dim3(3 + nn[0], 3 + nn[1], 3 + nn[2]));
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
  printf("ref_astaroth_solve n=%d,%d,%d dt=%g ok\n", nn[0], nn[1], nn[2], dt);
  return 0;
}
