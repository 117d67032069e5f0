#!/bin/bash
# Regenerates tests/golden/ref_geometry.json from the reference's OWN host code.
# Needs STENCIL_REFERENCE (a reference checkout; no GPU); the JSON is committed, this script is its provenance.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REPO="$(cd "$HERE/../.." && pwd)"
REF="${STENCIL_REFERENCE:?set STENCIL_REFERENCE to a cwpearson/stencil checkout}"
OUT="$REPO/oracle/_ref"
mkdir -p "$OUT" "$REPO/tests/golden"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS="-std=c++14 -O1 -gencode arch=compute_90a,code=sm_90a -rdc=true --expt-extended-lambda \
  -I$REF/include -I$REPO/include/mpi_shim -I/usr/local/cuda/include/nvtx3 \
  -DSTENCIL_USE_MPI=1 -DSTENCIL_USE_CUDA=1 -DSTENCIL_OUTPUT_LEVEL=1 -Xcompiler -w -w"
$NVCC $FLAGS -o "$OUT/ref_dump_geometry" "$HERE/ref_dump_geometry.cu" \
  "$REF/src/numeric.cpp" "$REF/src/local_domain.cu" "$REF/src/pack_kernel.cu" "$REF/src/timer.cpp" \
  "$REPO/src/mpi_shim.cpp" -lcudart
"$OUT/ref_dump_geometry" > "$REPO/tests/golden/ref_geometry.json"
python -c "import json,sys; d=json.load(open('$REPO/tests/golden/ref_geometry.json')); print({k: len(v) for k,v in d.items()})"
