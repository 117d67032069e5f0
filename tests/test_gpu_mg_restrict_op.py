"""GPU parity of the fused residual-restriction through the C ABI (sb_transfer_oplan_create): bit for bit against the
op rule followed by the restriction (tests/mg_oracle.py), float and double, 7- and 27-point residual ops with and
without aux, coarse boxes of many shapes (odd origins and extents, thin boxes for the cell kernel), allocation leads of
0 .. 12 bytes on each buffer, NaN in every fine cell the rule does not read and every coarse cell outside the boxes,
interior + exterior slabs against one box, sb_transfer_plan_bytes, an empty box, and one 512^3 -> 256^3 FP64 launch."""
import ctypes as C

import numpy as np
import pytest

import colour_oracle as co
import mg_oracle as mo
import transfer_oracle as to
from gpu_util import DevArray
from stencil_b200._lib import I3, Pitched, StencilTerm, check, lib

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
DT = {np.dtype(np.float32): 1, np.dtype(np.float64): 2}


def same(a, b):
    return np.array_equal(a.view(UINT[a.dtype]), b.view(UINT[b.dtype]))


def seven():
    return to.residual_terms(co.helmholtz(1.0 / 32, 0.5))


def twenty_seven():
    A = [(0, (0, 0, 0), 88.0 / 26)] + [(0, (x, y, z), -(1.0 + 0.1 * (abs(x) + 2 * abs(y) + 3 * abs(z))) / 26)
                                      for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]
    return to.residual_terms(A)


def no_aux(terms):
    return [t for t in terms if t[0] == 0]


def c_terms(terms):
    arr = (StencilTerm * len(terms))()
    for k, (s, o, w) in enumerate(terms):
        arr[k] = StencilTerm(s, (C.c_int32 * 3)(*o), w)
    return arr


def plan(dtype, terms, D, do, S, so, A, boxes):
    lo = (C.c_int64 * (3 * max(1, len(boxes))))(*[v for b in boxes for v in b[0]])
    hi = (C.c_int64 * (3 * max(1, len(boxes))))(*[v for b in boxes for v in b[1]])
    h = C.c_void_p()
    check(lib().sb_transfer_oplan_create(C.byref(h), 0, DT[np.dtype(dtype)], c_terms(terms), len(terms), D.pitched(), I3(*do), D.shape[0],
                                         S.pitched(), I3(*so), S.shape[0], A.pitched() if A is not None else Pitched(None, 0, 0),
                                         len(boxes), lo, hi))
    return h


def run(h):
    check(lib().sb_transfer_plan_launch(h, None))
    check(lib().sb_device_sync(0))


def mask(shape, origin, lo, hi):
    m = np.ones(shape, bool)
    for a in range(3):
        c = np.arange(shape[2 - a]) + origin[a]
        sh = [1, 1, 1]
        sh[2 - a] = shape[2 - a]
        m &= ((c >= lo[a]) & (c < hi[a])).reshape(sh)
    return m


def case(dtype, terms, boxes, lead_d=0, lead_s=0, lead_a=0, pad=(2, 1, 3)):
    """The boxes' union must be one box [lo, hi) (the slabs of a split, or one box)."""
    dtype = np.dtype(dtype)
    lo = [min(b[0][a] for b in boxes) for a in range(3)]
    hi = [max(b[1][a] for b in boxes) for a in range(3)]
    rng = np.random.default_rng(sum(lo) + 7 * sum(hi) + len(terms))
    so = tuple(2 * lo[a] - 1 - pad[a] for a in range(3))
    sshape = tuple(2 * (hi[a] - lo[a]) + 2 + 2 * pad[a] for a in (2, 1, 0))
    reach = max(max(abs(c) for c in t[1]) for t in terms)
    rlo = [2 * lo[a] - reach for a in range(3)]
    rhi = [2 * hi[a] + reach for a in range(3)]
    src = rng.uniform(-1, 1, sshape).astype(dtype)
    src[~mask(sshape, so, rlo, rhi)] = np.nan
    has_aux = any(t[0] == 1 for t in terms)
    aux = rng.uniform(-1, 1, sshape).astype(dtype)
    aux[~mask(sshape, so, [2 * v for v in lo], [2 * v for v in hi])] = np.nan
    do = tuple(lo[a] - 1 for a in range(3))
    dshape = tuple(hi[a] - lo[a] + 3 for a in (2, 1, 0))
    dst0 = np.full(dshape, np.nan, dtype)
    S, D = DevArray(src, lead=lead_s), DevArray(dst0, lead=lead_d)
    A = DevArray(aux, lead=lead_a) if has_aux else None
    h = plan(dtype, terms, D, do, S, so, A, boxes)
    try:
        cells = int(np.prod([hi[a] - lo[a] for a in range(3)]))
        assert lib().sb_transfer_plan_bytes(h) == cells * dtype.itemsize * (8 * (2 if has_aux else 1) + 1)
        run(h)
        want = dst0.copy()
        mo.restrict_op_box(want, do, terms, src, aux if has_aux else None, so, lo, hi)
        assert same(D.get(), want)
        assert same(S.get(), src)
    finally:
        lib().sb_transfer_plan_destroy(h)


def slabs(lo, hi):
    """[lo, hi) as its interior cut by 1 and the six exterior slabs (the host's interior / exterior split)."""
    il, ih = [v + 1 for v in lo], [v - 1 for v in hi]
    out = [(tuple(il), tuple(ih))]
    for a in range(3):
        for side in (0, 1):
            l, h = list(lo), list(hi)
            for b in range(a):
                l[b], h[b] = il[b], ih[b]
            if side == 0:
                h[a] = lo[a] + 1
            else:
                l[a] = hi[a] - 1
            out.append((tuple(l), tuple(h)))
    return out


BOXES = [((0, 0, 0), (1, 1, 1)), ((0, 0, 0), (4, 4, 4)), ((0, 0, 0), (7, 5, 3)), ((3, -2, 1), (11, 6, 9)), ((0, 0, 0), (32, 8, 8)),
         ((-5, 2, 0), (60, 11, 17)), ((1, 1, 1), (66, 35, 21)), ((2, 3, -1), (3, 40, 9))]
OPS = {"7pt": seven, "7pt-noaux": lambda: no_aux(seven()), "27pt": twenty_seven, "27pt-noaux": lambda: no_aux(twenty_seven())}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("op", sorted(OPS))
def test_boxes(dtype, box, op):
    case(dtype, OPS[op](), [box])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", ["d", "s", "a"])
def test_leads(dtype, which):
    es = np.dtype(dtype).itemsize
    for lead in range(0, 16, es):
        case(dtype, seven(), [((1, 0, 2), (40, 9, 7))], **{f"lead_{which}": lead})


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", ["7pt", "27pt"])
def test_interior_and_exterior_equal_one_box(dtype, op):
    lo, hi = (-3, 2, 1), (37, 15, 12)
    case(dtype, OPS[op](), slabs(lo, hi))
    case(dtype, OPS[op](), [(lo, hi)])


def test_empty_box():
    src = np.zeros((6, 6, 6))
    dst = np.full((4, 4, 4), np.nan)
    S, D = DevArray(src), DevArray(dst)
    h = plan(np.float64, no_aux(seven()), D, (0, 0, 0), S, (-1, -1, -1), None, [((1, 1, 1), (1, 2, 2))])
    try:
        assert lib().sb_transfer_plan_bytes(h) == 0
        run(h)
        assert same(D.get(), dst)
    finally:
        lib().sb_transfer_plan_destroy(h)


def test_512_fp64():
    """One 512^3 -> 256^3 FP64 fused residual-restriction (fine ghost width 1), bit for bit, the oracle in slabs."""
    n, m = 512, 256
    rng = np.random.default_rng(512)
    u = rng.uniform(-1, 1, (n + 2,) * 3)
    f = rng.uniform(-1, 1, (n + 2,) * 3)
    U, Fd = DevArray(u), DevArray(f)
    Cd = DevArray(np.full((m,) * 3, np.nan))
    terms = seven()
    h = plan(np.float64, terms, Cd, (0, 0, 0), U, (-1, -1, -1), Fd, [((0, 0, 0), (m, m, m))])
    try:
        run(h)
        got = Cd.get()
    finally:
        lib().sb_transfer_plan_destroy(h)
    for z0 in range(0, m, 32):
        want = np.empty((32, m, m))
        sl = slice(2 * z0, 2 * z0 + 66)  # fine planes 2 z0 - 1 .. 2 z0 + 64 in padded coordinates
        mo.restrict_op_box(want, (0, 0, z0), terms, u[sl], f[sl], (-1, -1, 2 * z0 - 1), (0, 0, z0), (m, m, z0 + 32))
        assert same(got[z0 : z0 + 32], want), z0
