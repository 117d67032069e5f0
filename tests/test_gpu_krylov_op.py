"""GPU parity of the Krylov vector kernels (sb_krylov_plan_*) through the C ABI, bit for bit against tests/krylov_oracle.py:
DOT with one and two pairs (also with aliased sources), XPBY (with T(s) = +-0 a copy that never reads p) and UPDATE, in
float and double, over boxes of many shapes (odd origins and extents, negative origins, thin and one-cell boxes), with
allocation leads of 0 .. 12 bytes on each buffer (16-byte and element-wide accesses), NaN in every cell outside the box
(never read, never written); exact sums against math.fsum, min / max / count against the order-independent rule,
special values against the exact-sum rule; interior + exterior slabs against one box; the bytes of each plan; and one
512^3 FP64 launch of each mode."""
import ctypes as C
import math

import numpy as np
import pytest

import krylov_oracle as ko
from gpu_util import DevArray
from stencil_b200 import _lib
from stencil_b200._lib import I3, Pitched, ReduceExactPart, ReduceResult, check, lib

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
DT = {np.dtype(np.float32): 1, np.dtype(np.float64): 2}
NAMES = {_lib.KRYLOV_DOT: "abc", _lib.KRYLOV_XPBY: "pz", _lib.KRYLOV_UPDATE: "xprq"}


def same(a, b):
    return np.array_equal(a.view(UINT[a.dtype]), b.view(UINT[b.dtype]))


def box_of(a, origin, lo, hi):
    return a[lo[2] - origin[2]:hi[2] - origin[2], lo[1] - origin[1]:hi[1] - origin[1], lo[0] - origin[0]:hi[0] - origin[0]]


class Parts:
    """A device buffer of n sb_reduce_exact_parts."""

    def __init__(self, n):
        self.n = max(1, n)
        p = C.c_void_p()
        check(lib().sb_malloc(C.byref(p), self.n * C.sizeof(ReduceExactPart), 0))
        self.ptr = p.value

    def get(self):
        host = (ReduceExactPart * self.n)()
        check(lib().sb_device_sync(0))
        check(lib().sb_memcpy(C.addressof(host), C.c_void_p(self.ptr), C.sizeof(host), 0, None))
        check(lib().sb_stream_sync(0, None))
        return list(host)

    def free(self):
        lib().sb_free(C.c_void_p(self.ptr), 0)


def rounded(part):
    out = ReduceResult()
    check(lib().sb_reduce_exact_round(C.byref(part), C.byref(out)))
    return out


def combined(parts):
    arr = (ReduceExactPart * len(parts))(*parts)
    out = ReduceExactPart()
    check(lib().sb_reduce_exact_combine(arr, len(parts), C.byref(out)))
    return out


def plan(mode, dtype, devs, origin, lo, hi):
    arr = (Pitched * len(devs))(*[d.pitched() for d in devs])
    h = C.c_void_p()
    check(lib().sb_krylov_plan_create(C.byref(h), 0, mode, DT[np.dtype(dtype)], arr, len(devs), I3(*origin), I3(*lo), I3(*hi)))
    return h


def launch(mode, dtype, devs, origin, boxes, s, nparts):
    """One plan per box, launched in order; returns the parts of each box."""
    out = []
    for lo, hi in boxes:
        P = Parts(nparts)
        h = plan(mode, dtype, devs, origin, lo, hi)
        try:
            check(lib().sb_krylov_plan_launch(h, C.c_double(s), C.c_void_p(P.ptr), None))
            out.append(P.get()[:nparts])
        finally:
            lib().sb_krylov_plan_destroy(h)
            P.free()
    return out


def check_part(part, v):
    """part against the per-cell terms v of one dot: the exact sum, sumsq an exact zero, min / max / count."""
    assert part.count == v.size
    assert all(w == 0 for w in part.sumsq.word) and part.sumsq.flags == 0
    want = ko.exact_dot(v, np.ones_like(v))
    got = rounded(part).sum
    assert (math.isnan(got) and math.isnan(want)) or (got == want and math.copysign(1, got) == math.copysign(1, want)), (got, want)
    mn, mx = ko.ordered_min_max(v)
    for g, w in ((part.min, mn), (part.max, mx)):
        assert np.float64(g).view(np.uint64) == np.float64(w).view(np.uint64), (g, w)


def run(mode, dtype, box, leads=(0, 0, 0, 0), nbuf=None, s=0.625, alias=False, slabs=None, seed=0, special=False):
    """One launch over box (or over the slabs that tile it) of buffers with NaN outside the box."""
    dtype = np.dtype(dtype)
    lo, hi = box
    nbuf = nbuf or {_lib.KRYLOV_DOT: 3, _lib.KRYLOV_XPBY: 2, _lib.KRYLOV_UPDATE: 4}[mode]
    rng = np.random.default_rng(seed + 5 * sum(lo) + 3 * sum(hi) + nbuf + mode)
    pad = (2, 3, 1)
    origin = tuple(lo[a] - pad[a] for a in range(3))
    shape = tuple(hi[a] - lo[a] + 2 * pad[a] for a in (2, 1, 0))
    host = []
    for k in range(nbuf):
        a = np.full(shape, np.nan, dtype)
        box_of(a, origin, lo, hi)[...] = rng.uniform(-2, 2, box_of(a, origin, lo, hi).shape).astype(dtype)
        host.append(a)
    if special:
        v = box_of(host[0], origin, lo, hi)
        b = v.reshape(-1).copy()
        b[:: max(1, b.size // 5)] = dtype.type(1e30 if dtype == np.float32 else 1e300)
        b[1] = -b[0]
        v[...] = b.reshape(v.shape)
    if mode == _lib.KRYLOV_XPBY and dtype.type(s) == 0:
        box_of(host[0], origin, lo, hi)[...] = np.nan  # p is not read
    # leads of 0 .. 12 bytes in steps of one element (float: 0, 4, 8, 12; double: 0, 8)
    devs = [DevArray(a, lead=leads[k % len(leads)] - leads[k % len(leads)] % dtype.itemsize) for k, a in enumerate(host)]
    if alias:  # <a, a> and <a, c>: source b is a
        devs[1] = devs[0]
        host[1] = host[0]
    nparts = nbuf - 1 if mode == _lib.KRYLOV_DOT else 1 if mode == _lib.KRYLOV_UPDATE else 0
    parts = launch(mode, dtype, devs, origin, slabs or [box], s, nparts)
    got = [d.get() for d in devs]
    I = [box_of(a, origin, lo, hi) for a in host]
    want = [a.copy() for a in host]
    W = [box_of(a, origin, lo, hi) for a in want]
    terms = []
    with np.errstate(over="ignore", invalid="ignore"):
        if mode == _lib.KRYLOV_DOT:
            terms = [I[0].astype(np.float64) * I[k].astype(np.float64) for k in range(1, nbuf)]
        elif mode == _lib.KRYLOV_XPBY:
            W[0][...] = ko.xpby(I[0], I[1], s)
        else:
            W[0][...], W[2][...] = ko.update(I[0], I[1], I[2], I[3], s)
            terms = [W[2].astype(np.float64) ** 2]
    for k in range(nbuf):
        assert same(got[k], want[k]), (NAMES[mode][k], np.argwhere(got[k].view(UINT[dtype]) != want[k].view(UINT[dtype]))[:4])
    for j, v in enumerate(terms):
        check_part(combined([p[j] for p in parts]), v)
    for d in set(map(id, devs)):
        next(x for x in devs if id(x) == d).free()
    return parts


BOXES = [((0, 0, 0), (1, 1, 1)), ((0, 0, 0), (8, 8, 8)), ((0, 0, 0), (7, 5, 3)), ((3, -2, 1), (21, 12, 17)), ((-5, 2, 0), (70, 11, 19)),
         ((1, 1, 1), (130, 20, 9)), ((2, 3, -1), (3, 40, 9)), ((0, 0, 0), (517, 3, 2)), ((4, 4, 4), (4, 9, 9))]
LEADS = [(0, 0, 0, 0), (4, 4, 4, 4), (8, 8, 8, 8), (12, 12, 12, 12), (0, 4, 8, 12), (12, 0, 8, 4), (8, 0, 0, 8)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("mode", [_lib.KRYLOV_DOT, _lib.KRYLOV_XPBY, _lib.KRYLOV_UPDATE])
def test_modes_boxes(dtype, box, mode):
    run(mode, dtype, box)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("leads", LEADS)
@pytest.mark.parametrize("mode", [_lib.KRYLOV_DOT, _lib.KRYLOV_XPBY, _lib.KRYLOV_UPDATE])
def test_modes_leads(dtype, leads, mode):
    run(mode, dtype, ((-3, 1, 2), (70, 13, 12)), leads=leads)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s", [0.0, -0.0, 1e-60, -1.75])
def test_xpby_scalars(dtype, s):
    """T(s) = +-0 (also 1e-60 in float32): p = z, with p NaN inside the box too."""
    run(_lib.KRYLOV_XPBY, dtype, ((1, 0, 2), (37, 6, 5)), s=s)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s", [0.0, -1.0 / 3, 1e30])
def test_update_scalars(dtype, s):
    run(_lib.KRYLOV_UPDATE, dtype, ((1, 0, 2), (37, 6, 5)), s=s)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nbuf,alias", [(2, False), (2, True), (3, False), (3, True)])
def test_dot_pairs_and_alias(dtype, nbuf, alias):
    run(_lib.KRYLOV_DOT, dtype, ((0, -1, 0), (45, 9, 7)), nbuf=nbuf, alias=alias, leads=(4, 4, 12))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_dot_special_values(dtype):
    """Huge terms that cancel, overflow in the sum, inf and NaN: the exact-sum rule."""
    run(_lib.KRYLOV_DOT, dtype, ((0, 0, 0), (40, 7, 6)), special=True)
    dtype = np.dtype(dtype)
    for bad in (np.inf, -np.inf, np.nan):
        a = np.ones((3, 4, 40), dtype)
        a[1, 2, 17] = bad
        A, B = DevArray(a), DevArray(np.full_like(a, 2.0))
        (part,), = launch(_lib.KRYLOV_DOT, dtype, [A, B], (0, 0, 0), [((0, 0, 0), (40, 4, 3))], 0.0, 1)
        check_part(part, a.astype(np.float64) * 2.0)
        A.free()
        B.free()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("mode", [_lib.KRYLOV_DOT, _lib.KRYLOV_XPBY, _lib.KRYLOV_UPDATE])
def test_slabs_against_one_box(dtype, mode):
    """The interior and the six exterior slabs of a box give the outputs of one launch over it, and their parts combine
    to the same bytes."""
    lo, hi = (-2, 1, 0), (30, 21, 14)
    il, ih = (1, 4, 3), (27, 18, 11)
    slabs = [(il, ih), ((ih[0], lo[1], lo[2]), hi), ((lo[0], lo[1], lo[2]), (il[0], hi[1], hi[2])), ((il[0], ih[1], lo[2]), (ih[0], hi[1], hi[2])),
             ((il[0], lo[1], lo[2]), (ih[0], il[1], hi[2])), ((il[0], il[1], ih[2]), (ih[0], ih[1], hi[2])), ((il[0], il[1], lo[2]), (ih[0], ih[1], il[2]))]
    assert sum(np.prod([h[a] - l[a] for a in range(3)]) for l, h in slabs) == np.prod([hi[a] - lo[a] for a in range(3)])
    one = run(mode, dtype, (lo, hi), seed=4)
    many = run(mode, dtype, (lo, hi), slabs=slabs, seed=4)
    for j in range(len(one[0])):
        a, b = combined([p[j] for p in many]), one[0][j]
        assert bytes(a.sum) == bytes(b.sum) and a.count == b.count and bytes(C.c_double(a.min)) == bytes(C.c_double(b.min))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_bytes(dtype):
    es = np.dtype(dtype).itemsize
    a = np.zeros((6, 7, 8), dtype)
    D = [DevArray(a) for _ in range(4)]
    n = 5 * 4 * 3
    for mode, devs, want in ((_lib.KRYLOV_DOT, D[:2], 2), (_lib.KRYLOV_DOT, D[:3], 3), (_lib.KRYLOV_DOT, [D[0], D[0]], 1), (_lib.KRYLOV_DOT, [D[0], D[0], D[1]], 2),
                             (_lib.KRYLOV_XPBY, D[:2], 3), (_lib.KRYLOV_UPDATE, D, 6)):
        h = plan(mode, dtype, devs, (0, 0, 0), (1, 2, 3), (6, 6, 6))
        assert lib().sb_krylov_plan_bytes(h) == want * n * es
        lib().sb_krylov_plan_destroy(h)
    for d in D:
        d.free()


def test_512_fp64_each_mode():
    n = 512
    rng = np.random.default_rng(9)
    host = [rng.uniform(-1, 1, (n, n, n)) for _ in range(4)]
    devs = [DevArray(a, lead=8) for a in host]
    box = [((0, 0, 0), (n, n, n))]
    try:
        p2, = launch(_lib.KRYLOV_DOT, np.float64, devs[:3], (0, 0, 0), box, 0.0, 2)
        for j in range(2):
            assert rounded(p2[j]).sum == math.fsum((host[0] * host[j + 1]).ravel().tolist())
        launch(_lib.KRYLOV_XPBY, np.float64, devs[:2], (0, 0, 0), box, 0.375, 0)
        host[0] = ko.xpby(host[0], host[1], 0.375)
        assert same(devs[0].get(), host[0])
        pu, = launch(_lib.KRYLOV_UPDATE, np.float64, devs, (0, 0, 0), box, -0.8125, 1)
        xn, rn = ko.update(host[0], host[1], host[2], host[3], -0.8125)
        assert same(devs[0].get(), xn) and same(devs[2].get(), rn)
        assert rounded(pu[0]).sum == math.fsum((rn * rn).ravel().tolist())
        assert pu[0].count == n**3
    finally:
        for d in devs:
            d.free()
