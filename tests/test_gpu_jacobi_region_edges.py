"""sb_jacobi3d over regions that end inside a 32-lane strip, against the numpy oracle, bit for bit.  With a lead-aligned
allocation (first compute cell 16-byte aligned) and a ghost width of 1, the vector after the last compute cell hangs
over the end of the row: the ghost cell must still be the last cell's +x neighbour.  (Whole-subdomain updates of 32-cell
wide FP64 subdomains, e.g. 64^3 on two ranks, hit this case.)"""
import ctypes as C

import numpy as np
import pytest

from oracle import np_oracle as no
from stencil_b200._lib import Pitched, check, i3, lib

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("nx,ox,lead", [(64, 0, 8), (32, 0, 8), (32, 32, 8), (32, 32, 0), (48, 16, 8), (16, 0, 8), (96, 3, 8),
                                        (40, 0, 0), (20, 5, 0), (33, 7, 8), (30, 0, 12), (62, 0, 4)])
def test_jacobi_region_ending_inside_a_strip(dtype, nx, ox, lead):
    es = np.dtype(dtype).itemsize
    if lead % es:
        pytest.skip("the lead must be a whole number of elements")
    rng = np.random.default_rng(nx * 100 + ox)
    raw = (nx + 2, 14, 12)
    src = rng.uniform(-1, 1, raw[::-1]).astype(dtype)
    dst0 = rng.uniform(-1, 1, raw[::-1]).astype(dtype)
    ps, pd = C.c_void_p(), C.c_void_p()
    check(lib().sb_malloc(C.byref(ps), src.nbytes + 64, 0))
    check(lib().sb_malloc(C.byref(pd), src.nbytes + 64, 0))
    try:
        s, d = ps.value + lead, pd.value + lead
        check(lib().sb_memcpy(C.c_void_p(s), src.ctypes.data, src.nbytes, 0, None))
        check(lib().sb_memcpy(C.c_void_p(d), dst0.ctypes.data, src.nbytes, 0, None))
        acc, lo, hi = (ox - 1, -1, -1), (ox, 0, 0), (ox + nx, raw[1] - 2, raw[2] - 2)
        clo, chi = (0, 0, 0), (128, raw[1] - 2, raw[2] - 2)
        pit = raw[0] * es
        check(lib().sb_jacobi3d(Pitched(d, pit, raw[1]), Pitched(s, pit, raw[1]), es, i3(acc), i3(lo), i3(hi), i3(clo), i3(chi), None))
        check(lib().sb_device_sync(0))
        got = np.empty_like(dst0)
        check(lib().sb_memcpy(got.ctypes.data, C.c_void_p(d), src.nbytes, 0, None))
        check(lib().sb_stream_sync(0, None))
        want = dst0.copy()
        no.jacobi_region(want, src, acc, lo, hi, clo, chi)
        bad = np.nonzero(got != want)
        assert bad[0].size == 0, f"{bad[0].size} cells differ, x columns {sorted(set(bad[2].tolist()))[:8]}"
    finally:
        lib().sb_free(ps, 0)
        lib().sb_free(pd, 0)
