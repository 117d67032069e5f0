// Astaroth MHD substep (`solve<step>`: 8 fields, 6th-order central differences, Williamson RK3) -- H100 rewrite of
// the reference's generated kernel (astaroth/user_kernels.h:36-183, 376-469; astaroth/integration.cuh:14-52;
// astaroth/kernels.cu:62-87).  SURVEY.md section 8 row a18.
#pragma once

#include <cstdint>
#include <cuda_runtime.h>

namespace sb {

// The uniforms solve<> reads through DCONST (astaroth/user_kernels.h:389-427).
struct AcParams {
  double inv_dsx, inv_dsy, inv_dsz;
  double dt;
  double cs2_sound, gamma, cp_sound, lnrho0, lnT0;
  double mu0, nu_visc, zeta, eta;
};

constexpr int kAcFields = 8; // lnrho, uux, uuy, uuz, ax, ay, az, entropy (astaroth/user_defines.h:112-120)

// VertexBufferArray (astaroth/kernels.h:22-27) without the unused profiles
struct AcFields {
  const void *in[kAcFields];
  void *out[kAcFields];
};

enum AcVariant {
  AC_AUTO = 0,   // tile kernel for thick regions, cell kernel for thin ones
  AC_CELL = 1,   // one thread per cell, neighbours through L1/L2
  AC_TILE = 2,   // z-march over a shared-memory ring of halo'd planes (cp.async pipeline), one thread per cell
  AC_TEAM = 3,   // the same ring, two specialised threads per cell (velocity/thermodynamics team + induction team);
                 // FP64: the ring is fed by TMA (one bulk tensor copy per field and plane) when the buffers allow it
  AC_TEAM_TMA = 4,  // the TMA-fed two-team kernel or an error (tests)
  AC_TEAM3_TMA = 5, // the TMA-fed three-team kernel (thermodynamics / velocity / induction) or an error
};

// solve<step> on the box [lo, hi) in memory-offset coordinates (the reference's IDX(i,j,k) = i + j*mx + k*mx*my);
// every cell of the box needs 3 allocated cells around it.  Returns the number of launches (0: empty box), <0: error.
int launch_astaroth_substep(int step, const AcFields &f, int dtype_size, long long mx, long long my, long long mz, const int lo[3],
                            const int hi[3], const AcParams &p, int variant, cudaStream_t stream);

} // namespace sb
