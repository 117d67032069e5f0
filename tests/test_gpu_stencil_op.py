"""GPU parity of the linear stencil operators through the C ABI (sb_stencil_plan_*): raw bits of the whole dst allocation
against the numpy rule of tests/stencil_op_oracle.py, float and double, over ops of every reach, odd shapes for the tile
kernel and thin slabs for the cell kernel, allocations at every 4-byte lead.  Every src cell no term reads and every aux
cell outside the box is NaN (a value read from one would show in the result); every dst cell outside the box is NaN too
and must stay so."""
import ctypes as C

import numpy as np
import pytest

import stencil_b200 as sb
import stencil_op_oracle as so
from gpu_util import DevArray
from stencil_b200._lib import Pitched, check, lib

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
ACC = (-3, 5, 7)  # global coordinate of allocation element (0, 0, 0)


def box27():
    rng = np.random.default_rng(3)
    return [(0, (x, y, z), float(rng.uniform(-1, 1))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]


OPS = {
    "7pt": so.laplacian(2, (1.0, 1.0, 1.0)),
    "lap4": so.laplacian(4, (0.049, 0.061, 0.037)),
    "lap6": so.laplacian(6, (0.049, 0.061, 0.037)),
    "lap8": so.laplacian(8, (0.049, 0.061, 0.037)),
    "box27": box27(),
    "upwind": [(0, (0, 0, 0), 1.25), (0, (-1, 0, 0), -0.75), (0, (-2, 0, 0), 0.125), (0, (0, -1, 0), -0.3), (0, (0, 0, -3), 0.01)],
    "aux": [(1, (0, 0, 0), -1.0)] + [(s, o, 0.21 * w) for s, o, w in so.laplacian(2, (1.0, 1.0, 1.0))] + [(0, (0, 0, 0), 2.0)],
}
SHAPES = [(37, 29, 23), (20, 13, 11), (64, 8, 8), (1, 17, 9), (33, 1, 12), (40, 9, 1), (5, 6, 7)]


def read_mask(terms, shape, lo, ext):
    m = np.zeros(shape, bool)
    for s, o, _ in terms:
        if s == 0:
            so._view(m, lo, ext, o)[...] = True
    return m


def run_case(terms, dtype, ext, lead=0, extra=0, dst_is_aux=False, seed=0):
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    rm, rp = so.reach(terms)
    lo = tuple(rm[a] + extra for a in range(3))
    raw = tuple(ext[a] + rm[a] + rp[a] + 2 * extra for a in range(3))
    shape = raw[::-1]
    src = rng.uniform(-1, 1, shape).astype(dtype)
    src[~read_mask(terms, shape, lo, ext)] = np.nan
    inbox = np.zeros(shape, bool)
    so._view(inbox, lo, ext, (0, 0, 0))[...] = True
    aux = rng.uniform(-1, 1, shape).astype(dtype)
    aux[~inbox] = np.nan
    dst = np.full(shape, np.nan, dtype)
    want = (aux if dst_is_aux else dst).copy()
    so.apply_box(terms, src, aux, want, lo, ext)
    op = sb.StencilOp(terms, dtype)
    d_src, d_aux = DevArray(src, lead=lead), DevArray(aux, lead=lead)
    d_dst = d_aux if dst_is_aux else DevArray(dst, lead=lead)
    glo = tuple(lo[a] + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    plan = sb.StencilPlan(0, op, d_dst.pitched(), d_src.pitched(), d_aux.pitched() if op.has_aux else Pitched(None, 0, 0), ACC, raw[2],
                          [(glo, ghi)])
    try:
        assert plan.bytes == int(np.prod(ext)) * dtype.itemsize * (3 if op.has_aux else 2)
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
def test_op_bits(op, dtype, si):
    run_case(OPS[op], dtype, SHAPES[si], lead=4 * (si % 4) if dtype == np.float32 else 8 * (si % 2), extra=si % 2, seed=si)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lead", [0, 4, 8, 12])
@pytest.mark.parametrize("op", ["7pt", "lap8", "box27", "upwind"])
def test_op_leads(op, dtype, lead):
    """Every 4-byte lead of the allocation (FP64 elements sit on 8-byte boundaries: leads 0 and 8), against the exact
    reach (the allocation ends where the op stops reading) and with a NaN margin."""
    if np.dtype(dtype).itemsize == 8 and lead % 8:
        pytest.skip("an FP64 allocation starts on an 8-byte boundary")
    for extra in (0, 2):
        run_case(OPS[op], dtype, (45, 19, 17), lead=lead, extra=extra, seed=lead + extra)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("xsize", [36, 37, 38, 64, 66])
def test_fp32_alternating_row_phase(dtype, xsize):
    """Rows of 38 floats (152 bytes) alternate their 16-byte phase from row to row; other widths shift it every row."""
    run_case(OPS["7pt"], dtype, (xsize, 21, 19), lead=np.dtype(dtype).itemsize, seed=xsize)
    run_case(OPS["aux"], dtype, (xsize, 21, 19), lead=0, seed=xsize)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(37, 29, 23), (1, 9, 9), (24, 16, 16)])
def test_dst_is_aux(dtype, shape):
    """u_new = 2u - u_prev + c lap(u) written over u_prev."""
    run_case(OPS["aux"], dtype, shape, dst_is_aux=True, seed=5)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_interior_and_exterior_boxes(dtype):
    """A region cut as interior + exterior slabs (sb_interior / sb_exterior) in one plan and as one box: the same bits;
    one tile launch plus one launch for all slabs."""
    dtype = np.dtype(dtype)
    terms = OPS["lap4"]
    ext = (40, 30, 20)
    r = sb.Radius.constant(2)
    rng = np.random.default_rng(1)
    shape = tuple(e + 4 for e in ext)[::-1]
    src = rng.uniform(-1, 1, shape).astype(dtype)
    d_src = DevArray(src)
    outs = []
    glo = tuple(2 + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    ilo, ihi = (C.c_int64 * 3)(), (C.c_int64 * 3)()
    check(lib().sb_interior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), ilo, ihi))
    elo, ehi = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    ne = check(lib().sb_exterior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), elo, ehi))
    cut = [(tuple(ilo), tuple(ihi))] + [(tuple(elo[3 * k : 3 * k + 3]), tuple(ehi[3 * k : 3 * k + 3])) for k in range(ne)]
    for boxes, launches in (([(glo, ghi)], 1), (cut, 2)):
        d_dst = DevArray(np.full(shape, np.nan, dtype))
        plan = sb.StencilPlan(0, sb.StencilOp(terms, dtype), d_dst.pitched(), d_src.pitched(), Pitched(None, 0, 0), ACC, shape[0], boxes)
        n0 = lib().sb_launch_count()
        plan.launch()
        assert lib().sb_launch_count() - n0 == launches
        outs.append(d_dst.get())
        plan.destroy()
    want = np.full(shape, np.nan, dtype)
    so.apply_box(terms, src, None, want, (2, 2, 2), ext)
    u = UINT[dtype]
    assert np.array_equal(outs[0].view(u), want.view(u))
    assert np.array_equal(outs[1].view(u), want.view(u))


def test_512_fp64_order8():
    """One 512^3 FP64 order-8 Laplacian, bit-identical to the oracle."""
    terms = OPS["lap8"]
    n, r = 512, 4
    shape = (n + 2 * r,) * 3
    rng = np.random.default_rng(512)
    src = rng.uniform(-1, 1, shape)
    d_src = DevArray(src)
    d_dst = DevArray(np.zeros(shape))
    plan = sb.StencilPlan(0, sb.StencilOp(terms, np.float64), d_dst.pitched(), d_src.pitched(), Pitched(None, 0, 0), (0, 0, 0), shape[0],
                          [((r, r, r), (r + n, r + n, r + n))])
    plan.launch()
    got = d_dst.get()
    plan.destroy()
    d_src.free()
    d_dst.free()
    want = np.zeros(shape)
    so.apply_box(terms, src, None, want, (r, r, r), (n, n, n))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
