"""The astaroth solve<step> kernels with parameters that cannot stand in for one another, on non-cubic boxes and at
shifted allocations.

The conf parameter set has inv_dsx == inv_dsy == inv_dsz, nu_visc == eta and cs2_sound == cp_sound == 1: a kernel that
swaps two of those or drops a 1 / cp computes the same numbers there.  Here the distinct set (stencil_b200.astaroth.
distinct_params, anisotropic spacing) is used, and every result is compared with the long double oracle under the
rounding budget of astaroth_util, which is tight enough that such a mistake fails at FP32 as well as FP64
(tests/test_oracle_astaroth.py::test_distinct_params_discriminate)."""
import os

import numpy as np
import pytest

import stencil_b200 as sb
from astaroth_util import GOLDEN_PARAMS, cached_reference, distinct_fields
from gpu_util import DevArray
from oracle import c_oracle as co
from stencil_b200 import astaroth as ac
from test_gpu_astaroth import BOXES, check_golden, check_iterations, run_substeps

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not co.HAS_F80, reason="no extended-precision long double on this platform")]

VARIANTS = [ac.AUTO, ac.CELL, ac.TILE, ac.TEAM, ac.TEAM_TMA, ac.TEAM3_TMA]
# mx != my != mz: an odd row length (the TMA-fed kernels do not apply), an even one, and a box that starts off the
# ghost layer in x and y
NONCUBIC = [
    ((41, 29, 35), (3, 3, 3), (38, 26, 32)),
    ((44, 27, 33), (3, 3, 3), (41, 24, 30)),
    ((30, 52, 19), (4, 5, 3), (27, 49, 16)),
]
CASES = [("distinct", b) for b in [BOXES[0], BOXES[3], BOXES[5], BOXES[6]] + NONCUBIC] + [("conf", b) for b in NONCUBIC]
PARAMS = {"conf": ac.conf_params, "distinct": ac.distinct_params}


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("pset,box", CASES, ids=[f"{p}-{b[0]}-{b[1]}-{b[2]}" for p, b in CASES])
def test_substeps_match_extended_reference(dtype, variant, pset, box):
    raw, lo, hi = box
    fields, ref = cached_reference(raw, lo, hi, 7, np.dtype(dtype).name, pset)
    run_substeps(fields, ref, lo, hi, PARAMS[pset](1e-3), variant)


# LocalDomain places an allocation so that its first compute cell is 16-byte aligned: FP64 radius 3 allocations start
# 8 bytes into their block (the TMA-fed kernels then build their tensor map from the 16-byte boundary below and shift
# the box by one element), FP32 ones 4 or 12 bytes in.
LEADS = [(np.float64, 8, v) for v in (ac.AUTO, ac.TEAM, ac.TEAM_TMA, ac.TEAM3_TMA, ac.TILE)]
LEADS += [(np.float32, lead, v) for lead in (4, 12) for v in (ac.AUTO, ac.TILE, ac.TEAM)]


@pytest.mark.parametrize("dtype,lead,variant", LEADS, ids=[f"{np.dtype(d).name}-{l}-{v}" for d, l, v in LEADS])
def test_allocation_lead(dtype, lead, variant):
    raw, lo, hi = NONCUBIC[1]
    fields, ref = cached_reference(raw, lo, hi, 7, np.dtype(dtype).name, "distinct")
    run_substeps(fields, ref, lo, hi, ac.distinct_params(1e-3), variant, lead=lead)


@pytest.mark.parametrize("lead", [0, 8])
def test_tma_not_applicable(lead):
    """Odd row length (rows are not whole 16-byte units) or FP32: the TMA-fed variants asked for by name are an error,
    and AUTO / TEAM fall back to the cp.async-fed kernel with the same results."""
    raw, lo, hi = NONCUBIC[0]
    for dtype in (np.float64, np.float32):
        fields, ref = cached_reference(raw, lo, hi, 7, np.dtype(dtype).name, "distinct")
        es = np.dtype(dtype).itemsize
        din = [DevArray(a, lead=lead) for a in fields[:8]]
        dout = [DevArray(a, lead=lead) for a in fields[8:]]
        try:
            for variant in (ac.TEAM_TMA, ac.TEAM3_TMA):
                with pytest.raises(sb.StencilError, match="code -4"):
                    ac.substep(0, [d.ptr for d in din], [d.ptr for d in dout], es, raw, lo, hi, ac.distinct_params(1e-3), variant)
            assert all(np.array_equal(d.get(), a) for d, a in zip(dout, fields[8:]))  # nothing was launched
        finally:
            for d in din + dout:
                d.free()
    for dtype in (np.float64, np.float32):
        fields, ref = cached_reference(raw, lo, hi, 7, np.dtype(dtype).name, "distinct")
        for variant in (ac.AUTO, ac.TEAM):
            run_substeps(fields, ref, lo, hi, ac.distinct_params(1e-3), variant, lead=lead)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("ndom", [1, 2])
def test_iteration_through_distributed_domain_distinct_params(dtype, ndom):
    """Astaroth.step() with the distinct set: two iterations on 24x20x28 over `ndom` subdomains."""
    import torch

    size = (24, 20, 28)
    ng = torch.cuda.device_count()
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([i % ng for i in range(ndom)])
    dd.set_radius(3)
    handles = [dd.add_data(dtype, name) for name in ac.FIELDS]
    dd.realize()
    try:
        sim = ac.Astaroth(dd, handles, ac.distinct_params(1e-3))
        check_iterations(dd, sim, distinct_fields(size, 3, dtype), co.distinct_params(1e-3), ndom)
    finally:
        dd.close()


@pytest.mark.skipif(not os.path.exists(GOLDEN_PARAMS), reason="golden vectors not generated yet (oracle/ref/make_astaroth_golden.py)")
@pytest.mark.parametrize("variant", [ac.CELL, ac.TILE, ac.TEAM, ac.TEAM_TMA, ac.TEAM3_TMA])
def test_matches_reference_kernel_golden_distinct_params(variant):
    """The reference's own solve<0,1,2> on a 12 x 9 x 7 grid with anisotropic spacing and the distinct constants."""
    z = np.load(GOLDEN_PARAMS)
    raw = tuple(int(v) + 6 for v in z["n"])
    p = [float(v) for v in z["params"]]
    check_golden(z["inputs"], z["outputs"], raw, co.AcParams(*p), ac.AstarothParams(*p), variant)
