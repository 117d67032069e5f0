#!/bin/bash
# Builds the UNMODIFIED reference (cwpearson/stencil) from the sources where they lie, in the checkout named by
# $STENCIL_REFERENCE, into oracle/_ref/ (git-ignored; __graft_entry__.build() runs this when STENCIL_REFERENCE is set):
#   libref_stencil.a      the reference library (all 16 sources), sm_90a, Release, CUDA graphs on
#   ref_jacobi3d          bin/jacobi3d.cu           (reference stencil_kernel + transports)
#   ref_bench_exchange    bin/bench_exchange.cu
#   ref_bench_pack        bin/bench_pack.cu
#   ref_test_cuda         the reference's own Catch2 GPU suite (test/test_cuda_*.cu + test_exchange.cu)
#   ref_test_cpu          the reference's own Catch2 host suite
# No MPI installation is assumed: the reference is linked against our single-process shim
# (include/mpi_shim/mpi.h, src/mpi_shim.cpp).  Nothing is copied out of the reference checkout.
# TEST / BASELINE INFRASTRUCTURE ONLY -- the product never links these files.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REPO="$(cd "$HERE/../.." && pwd)"
REF="${STENCIL_REFERENCE:?set STENCIL_REFERENCE to a cwpearson/stencil checkout}"
OUT="$REPO/oracle/_ref"
OBJ="$OUT/obj"
mkdir -p "$OUT" "$OBJ"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
STAMP="$OUT/.built"
if [ -f "$STAMP" ] && [ "$STAMP" -nt "$HERE/build_ref.sh" ] && [ "$STAMP" -nt "$HERE/ref_exchange_uniform.cu" ] && [ "$STAMP" -nt "$HERE/ref_astaroth_solve.cu" ] && [ "$STAMP" -nt "$HERE/ref_jacobi_golden.cu" ] && [ "$STAMP" -nt "$REPO/src/mpi_shim.cpp" ] && [ -z "${FORCE:-}" ]; then
  echo "oracle/_ref up to date"; exit 0
fi
DEFS="-DSTENCIL_USE_MPI=1 -DSTENCIL_USE_CUDA=1 -DSTENCIL_USE_CUDA_AWARE_MPI=1 -DSTENCIL_USE_CUDA_GRAPH=1 -DSTENCIL_SETUP_STATS=1 -DSTENCIL_OUTPUT_LEVEL=2 -DNDEBUG -DCATCH_CONFIG_NO_POSIX_SIGNALS"
INC="-I$REF/include -I$REF/thirdparty -I$REF/bin -I$REPO/include/mpi_shim -I/usr/local/cuda/include/nvtx3"
FLAGS="-std=c++14 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -rdc=true --expt-extended-lambda -Xcompiler -w -w -x cu $DEFS $INC"
LINK="-gencode arch=compute_90a,code=sm_90a -rdc=true -L/usr/local/cuda/lib64/stubs -lnvidia-ml -ldl -lcudart"

compile() { # src obj
  if [ ! -f "$2" ] || [ "$1" -nt "$2" ]; then $NVCC $FLAGS -c "$1" -o "$2"; fi
}
pids=()
LIBOBJS=()
for f in copy.cu gpu_topology.cpp local_domain.cu machine.cpp numeric.cpp pack_kernel.cu packer.cu placement_intranoderandom.cpp \
         rcstream.cpp stencil.cu timer.cpp topology.cpp translator.cu tx_colocated.cu tx_cuda_aware_mpi.cu tx_ipc.cpp; do
  o="$OBJ/lib_${f%.*}.o"; LIBOBJS+=("$o"); compile "$REF/src/$f" "$o" & pids+=($!)
done
compile "$REPO/src/mpi_shim.cpp" "$OBJ/mpi_shim.o" & pids+=($!)
for f in jacobi3d.cu bench_exchange.cu bench_pack.cu statistics.cpp; do
  compile "$REF/bin/$f" "$OBJ/bin_${f%.*}.o" & pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
rm -f "$OUT/libref_stencil.a"; ar rcs "$OUT/libref_stencil.a" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
for b in jacobi3d bench_exchange bench_pack; do
  $NVCC $LINK -o "$OUT/ref_$b" "$OBJ/bin_$b.o" "$OBJ/bin_statistics.o" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
done
# our own baseline driver over the reference library (uniform radii only, see the file header)
compile "$HERE/ref_exchange_uniform.cu" "$OBJ/ref_exchange_uniform.o"
$NVCC $LINK -o "$OUT/ref_exchange_uniform" "$OBJ/ref_exchange_uniform.o" "$OBJ/bin_statistics.o" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
# golden-vector generator for the jacobi numerics: the reference driver's own kernels (bin/jacobi3d.cu, main renamed),
# once with the reference's --use_fast_math (bin/CMakeLists.txt:56) and once with IEEE division
for flavour in "" "_ieee"; do
  o="$OBJ/ref_jacobi_golden$flavour.o"
  if [ ! -f "$o" ] || [ "$HERE/ref_jacobi_golden.cu" -nt "$o" ]; then
    $NVCC $FLAGS $([ -z "$flavour" ] && echo --use_fast_math) -c "$HERE/ref_jacobi_golden.cu" -o "$o"
  fi
  $NVCC $LINK -o "$OUT/ref_jacobi_golden$flavour" "$o" "$OBJ/bin_statistics.o" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
done
# the reference's astaroth driver against the reference library (+ its config file, data only)
AFLAGS="${FLAGS/-I$REF\/bin/} --use_fast_math -I$REF/astaroth -DAC_DEFAULT_CONFIG=\"oracle/_ref/astaroth.conf\""
pids=()
for f in astaroth.cu kernels.cu astaroth_utils.cu statistics.cpp; do
  compile_a() { if [ ! -f "$2" ] || [ "$1" -nt "$2" ]; then $NVCC $AFLAGS -c "$1" -o "$2"; fi; }
  compile_a "$REF/astaroth/$f" "$OBJ/astro_${f%.*}.o" & pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
$NVCC $LINK -o "$OUT/ref_astaroth" "$OBJ/astro_astaroth.o" "$OBJ/astro_kernels.o" "$OBJ/astro_astaroth_utils.o" "$OBJ/astro_statistics.o" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
cp "$REF/astaroth/astaroth.conf" "$OUT/astaroth.conf"
# golden-vector generator for solve<step>: the reference's kernels.cu driven on a small box (oracle/ref/ref_astaroth_solve.cu)
if [ ! -f "$OBJ/ref_astaroth_solve.o" ] || [ "$HERE/ref_astaroth_solve.cu" -nt "$OBJ/ref_astaroth_solve.o" ]; then
  $NVCC $AFLAGS -c "$HERE/ref_astaroth_solve.cu" -o "$OBJ/ref_astaroth_solve.o"
fi
$NVCC $LINK -o "$OUT/ref_astaroth_solve" "$OBJ/ref_astaroth_solve.o" "$OBJ/astro_kernels.o" "$OBJ/astro_astaroth_utils.o" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"

# the reference's own test suites
pids=(); TC=(); TH=()
for f in test_cuda_main.cu test_cuda_align.cu test_cuda_local_domain.cu test_cuda_pack.cu test_cuda_packer.cu test_cuda_rcstream.cu \
         test_cuda_translate.cu test_cuda_translate_kernel.cu test_cuda_gpu_topo.cu test_exchange.cu; do
  o="$OBJ/t_${f%.*}.o"; TC+=("$o"); compile "$REF/test/$f" "$o" & pids+=($!)
done
for f in test_cpu_main.cpp test_cpu_partition.cpp test_cpu_numeric.cpp test_cpu_radius.cpp test_cpu_accessor.cpp test_cpu_tx.cpp \
         test_cpu_mat2d.cpp test_cpu_qap.cpp; do
  o="$OBJ/t_${f%.*}.o"; TH+=("$o"); compile "$REF/test/$f" "$o" & pids+=($!)
done
for p in "${pids[@]}"; do wait "$p"; done
$NVCC $LINK -o "$OUT/ref_test_cuda" "${TC[@]}" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
$NVCC $LINK -o "$OUT/ref_test_cpu" "${TH[@]}" "${LIBOBJS[@]}" "$OBJ/mpi_shim.o"
touch "$STAMP"
ls -la "$OUT"
