"""Shared pieces of the astaroth parity tests (CPU and GPU sides).

Parity budget.  A result in precision T (float32 or float64) is compared with the extended-precision (long double)
oracle run on the same T-rounded inputs.  Field by field, it may deviate from that reference by

    K * (the deviation of the T oracle from it, same inputs, parameters, box and substeps)  +  FLOOR_ULPS ulps of max|out|

so the bound follows the rounding error the computation really has, at any parameters, spacing and dt, instead of a
fixed fraction of the field's magnitude.  K covers what the CUDA kernels round differently from the oracle, which is
compiled with -ffp-contract=off: nvcc contracts a*b + c into FMAs, the team kernels fold the sums in another order,
exp(lnT) is exp(lnT0) * exp(arg), and the device exp / expf round differently from glibc's.
"""
import functools
import os

import numpy as np

from oracle import c_oracle as co

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "astaroth_solve_ref.npz")
GOLDEN_PARAMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "astaroth_solve_ref_params.npz")
DS = 0.04908738521

# The largest kernel-error / oracle-error ratio measured on one H100 80GB HBM3 over every variant, precision and
# parameter set of tests/test_gpu_astaroth*.py is 1.77 (DESIGN.md section 2.3 lists the figures).  A mistake in a term
# moves the result by 70x (conf set, FP32) to 1e3x and more (distinct set) of the oracle's rounding.
K = 4.0
FLOOR_ULPS = 4.0


def make_fields(shape_xyz, seed: int, dtype=np.float64, smooth: float = 1.0, noise: float = 0.25, magnetic: float = 1.0):
    """16 arrays (in[8], out[8]) of raw size shape_xyz (x, y, z): seeded noise + a smooth component, all O(1); the
    vector potential (ax, ay, az) scaled by `magnetic`."""
    mx, my, mz = shape_xyz
    rng = np.random.default_rng(seed)
    a = rng.uniform(-1.0, 1.0, size=(16, mz, my, mx))
    Z, Y, X = np.meshgrid(np.arange(mz) * DS, np.arange(my) * DS, np.arange(mx) * DS, indexing="ij")
    for f in range(16):
        a[f] = noise * a[f] + smooth * np.sin((1 + f % 3) * X + 0.3 * f) * np.cos((1 + f % 2) * Y) * np.sin(2 * Z + f)
        if f % 8 in (4, 5, 6):
            a[f] *= magnetic
    return [np.ascontiguousarray(a[f].astype(dtype)) for f in range(16)]


def ulp_floor(dtype, want) -> float:
    return FLOOR_ULPS * float(np.finfo(dtype).eps) * float(np.abs(want).max())


def budgets(same, ext, dtype):
    """Per-field budgets of a `dtype` result: `same` is the `dtype` oracle's result, `ext` the long double one."""
    return [K * float(np.abs(s.astype(np.longdouble) - e).max()) + ulp_floor(dtype, e) for s, e in zip(same, ext)]


def errors(got, want):
    """Largest absolute deviation per field, computed in long double."""
    return [float(np.abs(np.asarray(g).astype(np.longdouble) - np.asarray(w).astype(np.longdouble)).max()) for g, w in zip(got, want)]


def assert_within(got, want, budget, what, names=None):
    for f, (e, b) in enumerate(zip(errors(got, want), budget)):
        assert e <= b, (what, names[f] if names else f, e, b, e / b)


def reference_substeps(fin, fout, lo, hi, params, nsteps: int = 3):
    """The oracle's `nsteps` substeps (0, 1, 2, ... into the same `out`, as the driver runs them) on the given inputs,
    in long double and in the inputs' own precision.  Returns per substep (ext[8], budget[8])."""
    dtype = fin[0].dtype
    xin = [a.astype(np.longdouble) for a in fin]
    xcur = [a.astype(np.longdouble) for a in fout]
    cur = [a.copy() for a in fout]
    res = []
    for step in range(nsteps):
        co.astaroth_substep(step, xin, xcur, lo, hi, params)
        co.astaroth_substep(step, fin, cur, lo, hi, params)
        res.append(([a.copy() for a in xcur], budgets(cur, xcur, dtype)))
    return res


# With unit amplitude everywhere the Lorentz force j x B / rho is ~1e4 (two derivatives of the noise in j, one in B)
# and its rounding hides every other momentum term: 1 % of nu or zeta moves the result by only ~10x the FP32 rounding.
# At a tenth of the amplitude for A, every term is well above the rounding of the others (test_distinct_params_discriminate).
DISTINCT_MAGNETIC = 0.1


def distinct_fields(shape_xyz, seed: int, dtype=np.float64):
    """make_fields for the distinct parameter set"""
    return make_fields(shape_xyz, seed=seed, dtype=dtype, magnetic=DISTINCT_MAGNETIC)


PARAM_SETS = {"conf": (co.astaroth_conf_params, make_fields), "distinct": (co.distinct_params, distinct_fields)}


@functools.lru_cache(maxsize=32)
def cached_reference(raw, lo, hi, seed, dtype_name, params_name, dt=1e-3):
    """fields, reference_substeps for the fields and oracle parameters of a named set ('conf' or 'distinct'); cached so
    that every kernel variant of a test is checked against one reference.  The arrays are shared: do not modify them."""
    make_params, make = PARAM_SETS[params_name]
    fields = make(raw, seed, np.dtype(dtype_name))
    return fields, reference_substeps(fields[:8], fields[8:], lo, hi, make_params(dt))
