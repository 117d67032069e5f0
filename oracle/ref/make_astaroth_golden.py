#!/usr/bin/env python
"""Golden vectors for the astaroth solve<step> substeps, produced by the REFERENCE's own kernels.

Run on a GPU (the reference kernels need a device):
    STENCIL_REFERENCE=<checkout> bash oracle/ref/build_ref.sh   # oracle/_ref/ref_astaroth_solve (no GPU needed)
    python oracle/ref/make_astaroth_golden.py OUT_DIR           # writes OUT_DIR/astaroth_solve_ref.npz
then copy OUT_DIR/astaroth_solve_ref.npz to tests/golden/.  Inputs: 16 arrays (in[8], out[8]) of (n+6)^3 doubles,
seeded uniform(-1, 1) plus a smooth component; outputs: the compute region of all 8 `out` fields after substeps 0, 1, 2
(no swap in between, like astaroth/astaroth.cu:551-640).  dt = 1e-3 (the driver's 1e-8 would hide the rate of change
under the rounding of the state)."""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def make_inputs(n: int, seed: int) -> np.ndarray:
    m = n + 6
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1.0, 1.0, size=(16, m, m, m))
    x = np.arange(m) * 0.04908738521
    Z, Y, X = np.meshgrid(x, x, x, indexing="ij")
    for f in range(16):
        a[f] = 0.25 * a[f] + np.sin((1 + f % 3) * X + 0.3 * f) * np.cos((1 + f % 2) * Y) * np.sin(2 * Z + f)
    return np.ascontiguousarray(a)


def main():
    n, dt, seed = 8, 1e-3, 20240921
    out_dir = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else ".")
    os.makedirs(out_dir, exist_ok=True)
    a = make_inputs(n, seed)
    fin, fout = os.path.join(out_dir, "ac_in.bin"), os.path.join(out_dir, "ac_out.bin")
    a.tofile(fin)
    subprocess.check_call([os.path.join(ROOT, "oracle/_ref/ref_astaroth_solve"), str(n), repr(dt), fin, fout], cwd=ROOT)
    m = n + 6
    res = np.fromfile(fout, dtype=np.float64).reshape(3, 8, m, m, m)
    np.savez_compressed(
        os.path.join(out_dir, "astaroth_solve_ref.npz"),
        n=n, dt=dt, seed=seed, inputs=a, outputs=res[:, :, 3:-3, 3:-3, 3:-3].copy(),
        source="reference astaroth/kernels.cu solve<0,1,2> on one GPU (--use_fast_math as in astaroth/CMakeLists.txt:55)",
    )  # fmt: skip
    os.remove(fin)
    os.remove(fout)
    print("wrote", os.path.join(out_dir, "astaroth_solve_ref.npz"), res.shape, float(np.abs(res).max()))


if __name__ == "__main__":
    sys.exit(main())
