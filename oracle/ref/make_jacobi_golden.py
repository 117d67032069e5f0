#!/usr/bin/env python
"""Golden vectors for the jacobi numerics, produced by the REFERENCE's own kernels (bin/jacobi3d.cu:18-85).

Run on a GPU (the reference kernels need a device):
    STENCIL_REFERENCE=<checkout> bash oracle/ref/build_ref.sh   # oracle/_ref/ref_jacobi_golden{,_ieee} (no GPU needed)
    python oracle/ref/make_jacobi_golden.py OUT_DIR             # writes OUT_DIR/jacobi_ref.npz
then copy OUT_DIR/jacobi_ref.npz to tests/golden/.  FP32 (the reference's only dtype), periodic single subdomain,
fields after 1, 10 and 40 iterations of the reference loop, from two builds of the same source:
  fast_*  with --use_fast_math as the reference's CMake builds bin/ (approximate divide -> compare at 1e-6 relative),
  ieee_*  without it (IEEE divide -> the oracle and the CUDA kernels must match bit for bit)."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SHAPES = [(64, 64, 64), (96, 80, 72)]
ITERS = [1, 10, 40]


def main():
    out_dir = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else ".")
    os.makedirs(out_dir, exist_ok=True)
    data = {"shapes": np.array(SHAPES), "iters": np.array(ITERS)}
    for si, (nx, ny, nz) in enumerate(SHAPES):
        for flavour, exe in (("fast", "ref_jacobi_golden"), ("ieee", "ref_jacobi_golden_ieee")):
            tmp = os.path.join(out_dir, "jacobi_golden.bin")
            subprocess.check_call([os.path.join(ROOT, "oracle/_ref", exe), str(nx), str(ny), str(nz), tmp] + [str(i) for i in ITERS], cwd=out_dir)
            a = np.fromfile(tmp, dtype=np.float32).reshape(len(ITERS), nz, ny, nx)
            os.remove(tmp)
            data[f"{flavour}_{si}"] = a
            print(flavour, (nx, ny, nz), "min/max", float(a.min()), float(a.max()), "non-0.5 cells after last iter", int(np.count_nonzero(a[-1] != 0.5)))
    data["source"] = np.array(
        "reference bin/jacobi3d.cu init_kernel + stencil_kernel through the reference DistributedDomain on one GPU; "
        "fast = --use_fast_math (bin/CMakeLists.txt:56), ieee = same source without it"
    )
    np.savez_compressed(os.path.join(out_dir, "jacobi_ref.npz"), **data)
    print("wrote", os.path.join(out_dir, "jacobi_ref.npz"), os.path.getsize(os.path.join(out_dir, "jacobi_ref.npz")), "bytes")


if __name__ == "__main__":
    sys.exit(main())
