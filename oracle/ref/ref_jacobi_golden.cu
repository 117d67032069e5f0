// Golden-vector generator for the jacobi numerics: drives the UNMODIFIED kernels of the reference driver
// (<reference>/bin/jacobi3d.cu:18-85 -- init_kernel, dist, stencil_kernel -- pulled in by #include with its main()
// renamed) through the reference library's own DistributedDomain on one GPU, and dumps the compute region after
// selected iterations.  The reference has no test and no golden output for these numerics (SURVEY.md section 8c);
// this is the pin.  Test / baseline infrastructure only (built by oracle/ref/build_ref.sh into oracle/_ref/, in two
// flavours: ref_jacobi_golden with the reference's --use_fast_math (bin/CMakeLists.txt:56) and ref_jacobi_golden_ieee
// without); never linked by the product.
//
//   ref_jacobi_golden <nx> <ny> <nz> <out.bin> <iter> [<iter> ...]      (iterations ascending)
//
// out.bin: for every listed iteration count, nx*ny*nz floats (x fastest): the field after that many iterations of
//          exchange -> stencil_kernel over the whole compute region -> swap (the --no-overlap order of
//          bin/jacobi3d.cu:344-353; the overlapped order computes the same values).
#define main reference_jacobi3d_main
#include "jacobi3d.cu" // resolved through -I<reference>/bin
#undef main

#include <cstdio>
#include <cstdlib>
#include <cstring>

int main(int argc, char **argv) {
  if (argc < 6) {
    fprintf(stderr, "usage: %s nx ny nz out.bin iter [iter ...]\n", argv[0]);
    return 2;
  }
  MPI_Init(&argc, &argv);
  const size_t nx = atoll(argv[1]), ny = atoll(argv[2]), nz = atoll(argv[3]);
  FILE *f = fopen(argv[4], "wb");
  if (!f) {
    fprintf(stderr, "cannot write %s\n", argv[4]);
    return 1;
  }
  {
    Radius radius = Radius::constant(0);
    radius.set_face(1);
    DistributedDomain dd(nx, ny, nz);
    dd.set_radius(radius);
    dd.set_gpus({0});
    auto dh = dd.add_data<float>("d");
    dd.realize();
    const Rect3 whole = dd.get_compute_region();
    LocalDomain &d = dd.domains()[0];
    const Rect3 reg = d.get_compute_region();
    const dim3 block = Dim3::make_block_dim(reg.extent(), 256);
    const dim3 grid = (reg.extent() + Dim3(block) - 1) / Dim3(block);
    d.set_device();
    init_kernel<<<grid, block>>>(d.get_curr_accessor<float>(dh), reg, whole);
    CUDA_RUNTIME(cudaDeviceSynchronize());
    int done = 0;
    for (int a = 5; a < argc; ++a) {
      const int target = atoi(argv[a]);
      for (; done < target; ++done) {
        dd.exchange();
        d.set_device();
        stencil_kernel<<<grid, block>>>(d.get_next_accessor<float>(dh), d.get_curr_accessor<float>(dh), reg, whole);
        CUDA_RUNTIME(cudaDeviceSynchronize());
        dd.swap();
      }
      const std::vector<unsigned char> bytes = d.interior_to_host(0);
      if (bytes.size() != nx * ny * nz * sizeof(float) || fwrite(bytes.data(), 1, bytes.size(), f) != bytes.size()) {
        fprintf(stderr, "short write\n");
        return 1;
      }
    }
  }
  fclose(f);
  MPI_Finalize();
  return 0;
}
