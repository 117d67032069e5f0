#!/usr/bin/env python
"""Golden vectors for the astaroth solve<step> substeps, produced by the REFERENCE's own kernels.

Run on a GPU (the reference kernels need a device):
    STENCIL_REFERENCE=<checkout> bash oracle/ref/build_ref.sh   # oracle/_ref/ref_astaroth_solve (no GPU needed)
    python oracle/ref/make_astaroth_golden.py OUT_DIR           # writes OUT_DIR/astaroth_solve_ref.npz and
                                                                #        OUT_DIR/astaroth_solve_ref_params.npz
then copy them to tests/golden/.  Inputs: 16 arrays (in[8], out[8]) of (n+6)^3 doubles, seeded uniform(-1, 1) plus a
smooth component; outputs: the compute region of all 8 `out` fields after substeps 0, 1, 2 (no swap in between, like
astaroth/astaroth.cu:551-640).  dt = 1e-3 (the driver's 1e-8 would hide the rate of change under the rounding of the
state).  The first file uses the astaroth.conf parameters on an 8^3 grid; the second a non-cubic grid, anisotropic
spacing and the distinct constants of stencil_b200.astaroth.distinct_params (vector potential at a tenth of the
amplitude, as tests/astaroth_util.distinct_fields), passed to the generator as overrides."""
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


def make_inputs_xyz(n, ds, seed: int, magnetic: float) -> np.ndarray:
    m = [v + 6 for v in n]
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1.0, 1.0, size=(16, m[2], m[1], m[0]))
    Z, Y, X = np.meshgrid(np.arange(m[2]) * ds[2], np.arange(m[1]) * ds[1], np.arange(m[0]) * ds[0], indexing="ij")
    for f in range(16):
        a[f] = 0.25 * a[f] + np.sin((1 + f % 3) * X + 0.3 * f) * np.cos((1 + f % 2) * Y) * np.sin(2 * Z + f)
        if f % 8 in (4, 5, 6):
            a[f] *= magnetic
    return np.ascontiguousarray(a)


def distinct(out_dir: str) -> None:
    """astaroth_solve_ref_params.npz: 12 x 9 x 7 cells (an even row length, so the TMA-fed kernels apply too), the
    distinct parameter set"""
    sys.path.insert(0, ROOT)
    from oracle import c_oracle as co

    n, dt, seed = (12, 9, 7), 1e-3, 20261015
    ds = co.DISTINCT_DS
    P = co.distinct_params(dt)
    a = make_inputs_xyz(n, ds, seed, 0.1)
    fin, fout = os.path.join(out_dir, "ac_in.bin"), os.path.join(out_dir, "ac_out.bin")
    a.tofile(fin)
    over = [str(v) for v in n] + [repr(v) for v in ds] + [repr(float(v)) for v in co.DISTINCT.values()]
    subprocess.check_call([os.path.join(ROOT, "oracle/_ref/ref_astaroth_solve"), "0", repr(dt), fin, fout] + over, cwd=ROOT)
    m = [v + 6 for v in n]
    res = np.fromfile(fout, dtype=np.float64).reshape(3, 8, m[2], m[1], m[0])
    params = np.array([getattr(P, k) for k, _ in co.AcParams._fields_])
    np.savez_compressed(
        os.path.join(out_dir, "astaroth_solve_ref_params.npz"),
        n=np.array(n), dt=dt, seed=seed, ds=np.array(ds), params=params, inputs=a, outputs=res[:, :, 3:-3, 3:-3, 3:-3].copy(),
        source="reference astaroth/kernels.cu solve<0,1,2> on one GPU (--use_fast_math as in astaroth/CMakeLists.txt:55), "
        "grid, spacing and constants overridden after acLoadConfig; params in sb_astaroth_params order",
    )  # fmt: skip
    os.remove(fin)
    os.remove(fout)
    print("wrote", os.path.join(out_dir, "astaroth_solve_ref_params.npz"), res.shape, float(np.abs(res).max()))


def main():
    n, dt, seed = 8, 1e-3, 20240921
    out_dir = os.path.abspath(sys.argv[1] if len(sys.argv) > 1 else ".")
    os.makedirs(out_dir, exist_ok=True)
    distinct(out_dir)
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
