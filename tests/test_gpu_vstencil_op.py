"""GPU parity of the variable-coefficient stencil operators through the C ABI (sb_stencil_vplan_create): raw bits of the
whole dst allocation against the numpy rule of tests/vstencil_oracle.py, float and double, over div(kappa grad u) with and
without the heat-step centre term, c^2 times Laplacians of order 2 and 4, and a term mix over all four fields and all 27
coefficient directions; on the shapes of test_gpu_stencil_op.py and at every allocation lead.  Every src and coefficient
cell the op does not read is NaN, so is every aux cell outside the box, and every dst cell outside the box must stay NaN."""
import numpy as np
import pytest

import stencil_b200 as sb
import stencil_op_oracle as so
import vstencil_oracle as vo
from gpu_util import DevArray
from stencil_b200._lib import Pitched, check, lib
from test_gpu_stencil_op import SHAPES

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
ACC = (-3, 5, 7)
DIRS = [(x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]


def mix(seed=0):
    rng = np.random.default_rng(seed)
    terms = [(0, DIRS[(7 * i) % 27], float(rng.uniform(-1, 1)), i % 4, c) for i, c in enumerate(DIRS)]
    return terms[:13] + [(1, (0, 0, 0), -0.75, 2, (1, 0, -1)), (0, (2, 0, -1), 0.3)] + terms[13:] + [(1, (0, 0, 0), 0.5)]


OPS = {
    "div_grad": vo.div_grad((0.049, 0.061, 0.037)),
    "heat": [(s, o, 1e-4 * w, k, c) for s, o, w, k, c in vo.div_grad((0.049, 0.061, 0.037))] + [(0, (0, 0, 0), 1.0)],
    "c2lap2": [(0, o, w, 0, (0, 0, 0)) for _, o, w in so.laplacian(2, (1.0, 1.0, 1.0))],
    "c2lap4": [(0, o, w, 0, (0, 0, 0)) for _, o, w in so.laplacian(4, (0.049, 0.061, 0.037))],
    "mix": mix(),
}


def masks(terms, shape, lo, ext):
    """Cells of src and of each coefficient field the op reads."""
    src = np.zeros(shape, bool)
    cf = [np.zeros(shape, bool) for _ in range(4)]
    for t in terms:
        s, o, w, k, c = vo.split(t)
        if s == 0:
            so._view(src, lo, ext, o)[...] = True
        if k >= 0:
            so._view(cf[k], lo, ext, c)[...] = True
    return src, cf


def run_case(terms, dtype, ext, lead=0, extra=0, alias=False, seed=0):
    """alias: coefficient field 1 is the src allocation."""
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    op = sb.StencilOp(terms, dtype)
    rm, rp = vo.reach(terms)
    lo = tuple(rm[a] + extra for a in range(3))
    raw = tuple(ext[a] + rm[a] + rp[a] + 2 * extra for a in range(3))
    shape = raw[::-1]
    ms, mc = masks(terms, shape, lo, ext)
    if alias:
        ms = ms | mc[1]
    src = rng.uniform(-1, 1, shape).astype(dtype)
    src[~ms] = np.nan
    coefs = []
    for k in range(op.ncoef):
        a = rng.uniform(0.5, 2.0, shape).astype(dtype)
        a[~mc[k]] = np.nan
        coefs.append(a)
    if alias:
        coefs[1] = src
    inbox = np.zeros(shape, bool)
    so._view(inbox, lo, ext, (0, 0, 0))[...] = True
    aux = rng.uniform(-1, 1, shape).astype(dtype)
    aux[~inbox] = np.nan
    dst = np.full(shape, np.nan, dtype)
    want = dst.copy()
    vo.apply_box(terms, src, aux, coefs, want, lo, ext)
    d_src, d_aux, d_dst = DevArray(src, lead=lead), DevArray(aux, lead=lead), DevArray(dst, lead=lead)
    d_coefs = [d_src if (alias and k == 1) else DevArray(c, lead=lead) for k, c in enumerate(coefs)]
    glo = tuple(lo[a] + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    plan = sb.StencilPlan(0, op, d_dst.pitched(), d_src.pitched(), d_aux.pitched() if op.has_aux else Pitched(None, 0, 0), ACC, raw[2],
                          [(glo, ghi)], [c.pitched() for c in d_coefs])
    try:
        nf = len({vo.split(t)[3] for t in terms} - {-1})
        assert plan.bytes == int(np.prod(ext)) * dtype.itemsize * ((3 if op.has_aux else 2) + nf)
        plan.launch()
        check(lib().sb_device_sync(0))
        got = d_dst.get()
    finally:
        plan.destroy()
    u = UINT[dtype]
    bad = got.view(u) != want.view(u)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist())
    assert np.array_equal(d_src.get().view(u), src.view(u))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("si", range(len(SHAPES)))
def test_vop_bits(op, dtype, si):
    run_case(OPS[op], dtype, SHAPES[si], lead=4 * (si % 4) if dtype == np.float32 else 8 * (si % 2), extra=si % 2, seed=si)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lead", [0, 4, 8, 12])
@pytest.mark.parametrize("op", ["heat", "c2lap4", "mix"])
def test_vop_leads(op, dtype, lead):
    if np.dtype(dtype).itemsize == 8 and lead % 8:
        pytest.skip("an FP64 allocation starts on an 8-byte boundary")
    for extra in (0, 2):
        run_case(OPS[op], dtype, (45, 19, 17), lead=lead, extra=extra, seed=lead + extra)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(37, 29, 23), (1, 17, 9), (66, 9, 10)])
def test_coefficient_aliases_src(dtype, shape):
    run_case(OPS["mix"], dtype, shape, alias=True, seed=3)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", ["7pt", "lap8", "aux"])
def test_plain_terms_through_vplan(op, dtype):
    """Plain terms through sb_stencil_vplan_create (no fields) and through sb_stencil_plan_create: the same bits."""
    from test_gpu_stencil_op import OPS as PLAIN

    dtype = np.dtype(dtype)
    terms = PLAIN[op]
    rng = np.random.default_rng(4)
    ext = (40, 30, 20)
    rm, rp = so.reach(terms)
    shape = tuple(ext[a] + rm[a] + rp[a] for a in range(3))[::-1]
    src, aux = rng.uniform(-1, 1, shape).astype(dtype), rng.uniform(-1, 1, shape).astype(dtype)
    d_src, d_aux = DevArray(src), DevArray(aux)
    op_ = sb.StencilOp(terms, dtype)
    glo = tuple(rm[a] + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    outs = []
    for coefs in (None, []):
        d_dst = DevArray(np.full(shape, np.nan, dtype))
        plan = sb.StencilPlan(0, op_, d_dst.pitched(), d_src.pitched(), d_aux.pitched(), ACC, shape[0], [(glo, ghi)], coefs)
        plan.launch()
        check(lib().sb_device_sync(0))
        outs.append(d_dst.get())
        plan.destroy()
    u = UINT[dtype]
    assert np.array_equal(outs[0].view(u), outs[1].view(u))
    want = np.full(shape, np.nan, dtype)
    so.apply_box(terms, src, aux, want, rm, ext)
    assert np.array_equal(outs[0].view(u), want.view(u))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_unit_coefficients_match_plain_plan(dtype):
    """c^2 lap4 with c^2 = 1 on the GPU gives the plain lap4 plan's bits (the tile kernel and the cell slabs)."""
    dtype = np.dtype(dtype)
    terms = OPS["c2lap4"]
    ext = (40, 30, 20)
    shape = tuple(e + 4 for e in ext)[::-1]
    rng = np.random.default_rng(6)
    src = rng.uniform(-1, 1, shape).astype(dtype)
    d_src, d_one = DevArray(src), DevArray(np.ones(shape, dtype))
    r = sb.Radius.constant(2)
    glo = tuple(2 + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    import ctypes as C

    ilo, ihi = (C.c_int64 * 3)(), (C.c_int64 * 3)()
    check(lib().sb_interior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), ilo, ihi))
    elo, ehi = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    ne = check(lib().sb_exterior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), elo, ehi))
    cut = [(tuple(ilo), tuple(ihi))] + [(tuple(elo[3 * k : 3 * k + 3]), tuple(ehi[3 * k : 3 * k + 3])) for k in range(ne)]
    outs = []
    for op_, coefs in ((sb.StencilOp(terms, dtype), [d_one.pitched()]), (sb.StencilOp([t[:3] for t in terms], dtype), None)):
        d_dst = DevArray(np.full(shape, np.nan, dtype))
        plan = sb.StencilPlan(0, op_, d_dst.pitched(), d_src.pitched(), Pitched(None, 0, 0), ACC, shape[0], cut, coefs)
        plan.launch()
        check(lib().sb_device_sync(0))
        outs.append(d_dst.get())
        plan.destroy()
    u = UINT[dtype]
    assert np.array_equal(outs[0].view(u), outs[1].view(u))


def test_512_fp64_div_grad():
    """One 512^3 FP64 div(kappa grad u) heat step, bit-identical to the oracle."""
    terms = OPS["heat"]
    n = 512
    shape = (n + 2,) * 3
    rng = np.random.default_rng(512)
    src = rng.uniform(-1, 1, shape)
    coefs = [rng.uniform(0.5, 2.0, shape) for _ in range(3)]
    d_src, d_dst = DevArray(src), DevArray(np.zeros(shape))
    d_c = [DevArray(c) for c in coefs]
    plan = sb.StencilPlan(0, sb.StencilOp(terms, np.float64), d_dst.pitched(), d_src.pitched(), Pitched(None, 0, 0), (0, 0, 0), shape[0],
                          [((1, 1, 1), (1 + n, 1 + n, 1 + n))], [c.pitched() for c in d_c])
    plan.launch()
    got = d_dst.get()
    plan.destroy()
    for a in [d_src, d_dst] + d_c:
        a.free()
    want = np.zeros(shape)
    vo.apply_box(terms, src, None, coefs, want, (1, 1, 1), (n, n, n))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
