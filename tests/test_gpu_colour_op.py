"""GPU parity of coloured application through the C ABI (sb_stencil_cplan_create): raw bits of the whole allocation
against tests/colour_oracle.py, float and double, every colour, in place (dst == src, f on aux) and out of place (dst a
separate allocation that must keep its bits outside the colour), on the shapes of test_gpu_stencil_op.py and at every
allocation lead.  The ops: SOR relaxations (sb_stencil_relax) of the order-2 Laplacian under 2 colours and of a 27-point
box under 8, and a damped update u + theta (div(kappa grad u) - f) with kappa in three coefficient fields.  Every src
cell the op does not read is NaN, so is every aux and coefficient cell outside what the op reads, and every dst cell
outside the box; every cell not of the colour must keep its bits.  A 512^3 FP64 red and black pass in place ends it: a
kernel that used a value written in the same launch fails there."""
import numpy as np
import pytest

import colour_oracle as co
import stencil_b200 as sb
import stencil_op_oracle as so
import vstencil_oracle as vo
from gpu_util import DevArray
from stencil_b200._lib import Pitched, check, lib
from test_gpu_stencil_op import SHAPES

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
ACC = (-3, 5, 7)


def box27_A():
    rng = np.random.default_rng(3)
    return [(0, (x, y, z), float(rng.uniform(-1, 0))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)] + [
        (0, (0, 0, 0), 30.0)]


def damped(theta=0.02):
    """u + theta (div(kappa grad u) - f): by hand, since the relaxation table takes constant coefficients."""
    return [(0, (0, 0, 0), 1.0)] + [(s, o, theta * w, k, c) for s, o, w, k, c in vo.div_grad((0.9, 1.0, 1.1))] + [(1, (0, 0, 0), -theta)]


OPS = {
    "sor7": (co.relax(co.helmholtz(1.0, 0.06), 1.6), 2),
    "gs7": (co.relax(co.helmholtz(0.7, 2.0), 1.0), 2),
    "sor27": (co.relax(box27_A(), 1.3), 8),
    "damped": (damped(), 2),
}


def run_case(op, dtype, ext, colour, lead=0, extra=0, in_place=True, seed=0):
    dtype = np.dtype(dtype)
    terms, m = OPS[op]
    rng = np.random.default_rng(seed)
    rm, rp = vo.reach(terms)
    lo = tuple(rm[a] + extra for a in range(3))
    raw = tuple(ext[a] + rm[a] + rp[a] + 2 * extra for a in range(3))
    shape = raw[::-1]
    src_mask = np.zeros(shape, bool)
    coef_masks = [np.zeros(shape, bool) for _ in range(4)]
    for t in terms:
        s, o, w, k, c = vo.split(t)
        if s == 0:
            so._view(src_mask, lo, ext, o)[...] = True
        if k >= 0:
            so._view(coef_masks[k], lo, ext, c)[...] = True
    inbox = np.zeros(shape, bool)
    so._view(inbox, lo, ext, (0, 0, 0))[...] = True
    u = rng.uniform(-1, 1, shape).astype(dtype)
    u[~src_mask] = np.nan
    f = rng.uniform(-1, 1, shape).astype(dtype)
    f[~inbox] = np.nan
    nk = max([vo.split(t)[3] + 1 for t in terms])
    ks = []
    for k in range(nk):
        a = rng.uniform(0.5, 2.0, shape).astype(dtype)
        a[~coef_masks[k]] = np.nan
        ks.append(a)
    dst0 = u.copy() if in_place else rng.uniform(-1, 1, shape).astype(dtype)
    if not in_place:
        dst0[~inbox] = np.nan
    want = dst0.copy()
    co.apply_box(terms, u, f, ks, want, lo, ext, ACC, m, colour)
    d_u, d_f = DevArray(u, lead=lead), DevArray(f, lead=lead)
    d_dst = d_u if in_place else DevArray(dst0, lead=lead)
    d_k = [DevArray(k, lead=lead) for k in ks]
    glo = tuple(lo[a] + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    plan = sb.StencilPlan(0, sb.StencilOp(terms, dtype), d_dst.pitched(), d_u.pitched(), d_f.pitched(), ACC, raw[2], [(glo, ghi)],
                          [k.pitched() for k in d_k] if nk else None, (m, colour))
    try:
        written = int(co.box_mask(shape, lo, ext, ACC, m, colour).sum())
        assert plan.bytes == (int(np.prod(ext)) * (2 + nk) + written) * dtype.itemsize
        plan.launch()
        check(lib().sb_device_sync(0))
        got = d_dst.get()
    finally:
        plan.destroy()
    t = UINT[dtype]
    bad = got.view(t) != want.view(t)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist())
    if not in_place:
        assert np.array_equal(d_u.get().view(t), u.view(t))
    assert np.array_equal(d_f.get().view(t), f.view(t))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", list(OPS))
@pytest.mark.parametrize("si", range(len(SHAPES)))
def test_colour_bits(op, dtype, si):
    for c in range(OPS[op][1]):
        run_case(op, dtype, SHAPES[si], c, lead=4 * (si % 4) if dtype == np.float32 else 8 * (si % 2), extra=si % 2, seed=si + 10 * c)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lead", [0, 4, 8, 12])
@pytest.mark.parametrize("op", ["sor7", "sor27", "damped"])
def test_colour_leads(op, dtype, lead):
    """Every 4-byte lead of the allocation (FP64: leads 0 and 8), against the exact reach and with a NaN margin; rows of
    38 floats alternate their 16-byte phase from row to row."""
    if np.dtype(dtype).itemsize == 8 and lead % 8:
        pytest.skip("an FP64 allocation starts on an 8-byte boundary")
    for extra in (0, 2):
        for c in range(OPS[op][1]):
            run_case(op, dtype, (45, 19, 17), c, lead=lead, extra=extra, seed=lead + extra + c)
    run_case(op, dtype, (36, 21, 19), 1, lead=lead, seed=lead)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", [(37, 29, 23), (1, 17, 9), (66, 9, 10)])
def test_masked_out_of_place(dtype, shape):
    """m = 2 with dst != src: only the colour's cells of dst change; src and aux keep their bits."""
    for c in range(2):
        run_case("sor7", dtype, shape, c, in_place=False, seed=7 + c)
    run_case("damped", dtype, shape, 1, in_place=False, seed=9)


def test_512_fp64_red_black_in_place():
    """One 512^3 FP64 red pass, then black, in place with f on aux: bit-identical to the oracle after each."""
    terms, m = OPS["sor7"]
    n = 512
    shape = (n + 2,) * 3
    rng = np.random.default_rng(512)
    u = rng.uniform(-1, 1, shape)
    f = rng.uniform(-1, 1, shape)
    d_u, d_f = DevArray(u), DevArray(f)
    op = sb.StencilOp(terms, np.float64)
    box = [((1, 1, 1), (1 + n, 1 + n, 1 + n))]
    for c in range(2):
        plan = sb.StencilPlan(0, op, d_u.pitched(), d_u.pitched(), d_f.pitched(), (0, 0, 0), shape[0], box, None, (2, c))
        plan.launch()
        got = d_u.get()
        plan.destroy()
        co.apply_box(terms, u, f, [], u, (1, 1, 1), (n, n, n), (0, 0, 0), 2, c)
        assert np.array_equal(got.view(np.uint64), u.view(np.uint64)), c
    d_u.free()
    d_f.free()


def test_interior_and_exterior_boxes_in_place():
    """A region cut as interior + exterior slabs in one coloured plan and as one box: the same bits (the tile kernel and
    the cell kernel agree on every cell's colour)."""
    terms, m = OPS["sor27"]
    ext = (40, 30, 20)
    shape = tuple(e + 2 for e in ext)[::-1]
    rng = np.random.default_rng(6)
    u, f = rng.uniform(-1, 1, shape), rng.uniform(-1, 1, shape)
    import ctypes as C

    r = sb.Radius.constant(1)
    glo = tuple(1 + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    ilo, ihi = (C.c_int64 * 3)(), (C.c_int64 * 3)()
    check(lib().sb_interior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), ilo, ihi))
    elo, ehi = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    ne = check(lib().sb_exterior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), elo, ehi))
    cut = [(tuple(ilo), tuple(ihi))] + [(tuple(elo[3 * k : 3 * k + 3]), tuple(ehi[3 * k : 3 * k + 3])) for k in range(ne)]
    for c in (0, 5):
        outs = []
        for boxes in (cut, [(glo, ghi)]):
            d_u, d_f = DevArray(u), DevArray(f)
            plan = sb.StencilPlan(0, sb.StencilOp(terms, np.float64), d_u.pitched(), d_u.pitched(), d_f.pitched(), ACC, shape[0], boxes, None, (m, c))
            plan.launch()
            outs.append(d_u.get())
            plan.destroy()
        want = u.copy()
        co.apply_box(terms, u, f, [], want, (1, 1, 1), ext, ACC, m, c)
        assert np.array_equal(outs[0].view(np.uint64), want.view(np.uint64))
        assert np.array_equal(outs[1].view(np.uint64), want.view(np.uint64))
