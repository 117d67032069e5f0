"""GPU parity of the BiCGStab Krylov modes through the C ABI, bit for bit against tests/bicgstab_oracle.py: BICG_P
(p = r + T(beta) (p - T(omega) v)) and UPDATE with c (<r', r'> and <c, r'>, also with c aliasing p or q), in float and
double, over boxes of many shapes with allocation leads of 0 .. 12 bytes on each buffer and NaN in every cell outside
the box; special values in the dots; interior + exterior slabs against one box; sb_krylov_plan_launch refusing a
BICG_P plan; the bytes of each plan; and one 512^3 FP64 launch of each."""
import ctypes as C
import math

import numpy as np
import pytest

import bicgstab_oracle as bo
import krylov_oracle as ko
from gpu_util import DevArray
from stencil_b200 import _lib
from stencil_b200._lib import check, lib
from test_gpu_krylov_op import BOXES, LEADS, UINT, Parts, box_of, check_part, combined, plan, rounded, same

pytestmark = pytest.mark.gpu

BICG, UPD = _lib.KRYLOV_BICG_P, _lib.KRYLOV_UPDATE
NAMES = {BICG: "prv", UPD: "xprqc"}


def launch2(mode, dtype, devs, origin, boxes, s, t, nparts):
    """One plan per box, launched in order by sb_krylov_plan_launch2; returns the parts of each box."""
    out = []
    for lo, hi in boxes:
        P = Parts(nparts)
        h = plan(mode, dtype, devs, origin, lo, hi)
        try:
            check(lib().sb_krylov_plan_launch2(h, C.c_double(s), C.c_double(t), C.c_void_p(P.ptr), None))
            out.append(P.get()[:nparts])
        finally:
            lib().sb_krylov_plan_destroy(h)
            P.free()
    return out


def run(mode, dtype, box, leads=(0, 0, 0, 0, 0), s=0.625, t=-0.375, c_is=None, slabs=None, seed=0, special=False):
    """One launch over box (or over the slabs that tile it) of buffers with NaN outside the box.  c_is: UPDATE's c is
    buffer 1 (p) or 3 (q)."""
    dtype = np.dtype(dtype)
    lo, hi = box
    nbuf = 3 if mode == BICG else 5
    rng = np.random.default_rng(seed + 5 * sum(lo) + 3 * sum(hi) + nbuf)
    pad = (2, 3, 1)
    origin = tuple(lo[a] - pad[a] for a in range(3))
    shape = tuple(hi[a] - lo[a] + 2 * pad[a] for a in (2, 1, 0))
    host = []
    for k in range(nbuf):
        a = np.full(shape, np.nan, dtype)
        box_of(a, origin, lo, hi)[...] = rng.uniform(-2, 2, box_of(a, origin, lo, hi).shape).astype(dtype)
        host.append(a)
    if special:  # huge terms that cancel and overflow in <c, r'>: c large, q = 0 so r' = r
        v = box_of(host[4], origin, lo, hi).reshape(-1)
        b = v.copy()
        b[:: max(1, b.size // 5)] = dtype.type(1e30 if dtype == np.float32 else 1e300)
        b[1] = -b[0]
        box_of(host[4], origin, lo, hi)[...] = b.reshape(box_of(host[4], origin, lo, hi).shape)
        box_of(host[3], origin, lo, hi)[...] = 0
    devs = [DevArray(a, lead=leads[k % len(leads)] - leads[k % len(leads)] % dtype.itemsize) for k, a in enumerate(host)]
    if c_is is not None:
        devs[4].free()
        devs[4], host[4] = devs[c_is], host[c_is]
    nparts = 2 if mode == UPD else 0
    parts = launch2(mode, dtype, devs, origin, slabs or [box], s, t, nparts)
    got = [d.get() for d in devs]
    I = [box_of(a, origin, lo, hi) for a in host]
    want = [a.copy() for a in host]
    W = [box_of(a, origin, lo, hi) for a in want]
    terms = []
    with np.errstate(over="ignore", invalid="ignore"):
        if mode == BICG:
            W[0][...] = bo.bicg_p(I[0], I[1], I[2], s, t)
        else:
            W[0][...], W[2][...] = ko.update(I[0], I[1], I[2], I[3], s)
            r = W[2].astype(np.float64)
            terms = [r * r, I[4].astype(np.float64) * r]
    for k in range(nbuf):
        if c_is is not None and k == 4:
            continue
        assert same(got[k], want[k]), (NAMES[mode][k], np.argwhere(got[k].view(UINT[dtype]) != want[k].view(UINT[dtype]))[:4])
    for j, v in enumerate(terms):
        check_part(combined([p[j] for p in parts]), v)
    for d in {id(x): x for x in devs}.values():
        d.free()
    return parts


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("mode", [BICG, UPD])
def test_modes_boxes(dtype, box, mode):
    run(mode, dtype, box)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("leads", LEADS + [(0, 4, 8, 12, 4), (12, 8, 4, 0, 8)])
@pytest.mark.parametrize("mode", [BICG, UPD])
def test_modes_leads(dtype, leads, mode):
    run(mode, dtype, ((-3, 1, 2), (70, 13, 12)), leads=tuple(leads) + (leads[0],) * (5 - len(leads)))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s,t", [(0.0, 0.5), (-0.0, 1.0), (1.5, 0.0), (1e-60, 1e30), (-1.0 / 3, 1.0 / 7)])
def test_bicg_p_scalars(dtype, s, t):
    """T(beta) = +-0 still reads p (no copy shortcut); T(omega) = 0 leaves p - 0 v."""
    run(BICG, dtype, ((1, 0, 2), (37, 6, 5)), s=s, t=t)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("c_is", [1, 3])
def test_update_c_aliasing_p_or_q(dtype, c_is):
    run(UPD, dtype, ((0, -1, 0), (45, 9, 7)), c_is=c_is, leads=(4, 4, 12, 8, 0))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_update_c_special_values(dtype):
    """Huge terms that cancel and overflow in <c, r'>, then inf and NaN in c: the exact-sum rule."""
    run(UPD, dtype, ((0, 0, 0), (40, 7, 6)), s=0.5, special=True)
    dtype = np.dtype(dtype)
    for bad in (np.inf, -np.inf, np.nan):
        x, p, r, q = (np.ones((3, 4, 40), dtype) for _ in range(4))
        c = np.full_like(x, 2.0)
        c[1, 2, 17] = bad
        D = [DevArray(a) for a in (x, p, r, q, c)]
        (parts,) = launch2(UPD, dtype, D, (0, 0, 0), [((0, 0, 0), (40, 4, 3))], 0.5, 0.0, 2)
        rn = np.full_like(x, 0.5).astype(np.float64)
        check_part(parts[0], rn * rn)
        check_part(parts[1], c.astype(np.float64) * rn)
        for d in D:
            d.free()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("mode", [BICG, UPD])
def test_slabs_against_one_box(dtype, mode):
    lo, hi = (-2, 1, 0), (30, 21, 14)
    il, ih = (1, 4, 3), (27, 18, 11)
    slabs = [(il, ih), ((ih[0], lo[1], lo[2]), hi), ((lo[0], lo[1], lo[2]), (il[0], hi[1], hi[2])), ((il[0], ih[1], lo[2]), (ih[0], hi[1], hi[2])),
             ((il[0], lo[1], lo[2]), (ih[0], il[1], hi[2])), ((il[0], il[1], ih[2]), (ih[0], ih[1], hi[2])), ((il[0], il[1], lo[2]), (ih[0], ih[1], il[2]))]
    one = run(mode, dtype, (lo, hi), seed=4)
    many = run(mode, dtype, (lo, hi), slabs=slabs, seed=4)
    for j in range(len(one[0])):
        a, b = combined([p[j] for p in many]), one[0][j]
        assert bytes(a.sum) == bytes(b.sum) and a.count == b.count and bytes(C.c_double(a.min)) == bytes(C.c_double(b.min))


def test_launch_refuses_bicg_p():
    a = np.zeros((4, 4, 8))
    D = [DevArray(a) for _ in range(3)]
    h = plan(BICG, np.float64, D, (0, 0, 0), (0, 0, 0), (8, 4, 4))
    try:
        assert lib().sb_krylov_plan_launch(h, C.c_double(1.0), None, None) == -1
        assert "use sb_krylov_plan_launch2" in lib().sb_last_error().decode()
    finally:
        lib().sb_krylov_plan_destroy(h)
        for d in D:
            d.free()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_bytes(dtype):
    es = np.dtype(dtype).itemsize
    a = np.zeros((6, 7, 8), dtype)
    D = [DevArray(a) for _ in range(5)]
    n = 5 * 4 * 3
    for mode, devs, want in ((BICG, D[:3], 4), (BICG, [D[0], D[1], D[1]], 3), (UPD, D, 7), (UPD, D[:4] + [D[1]], 6)):
        h = plan(mode, dtype, devs, (0, 0, 0), (1, 2, 3), (6, 6, 6))
        assert lib().sb_krylov_plan_bytes(h) == want * n * es
        lib().sb_krylov_plan_destroy(h)
    for d in D:
        d.free()


def test_512_fp64_each():
    n = 512
    rng = np.random.default_rng(9)
    host = [rng.uniform(-1, 1, (n, n, n)) for _ in range(5)]
    devs = [DevArray(a, lead=8) for a in host]
    box = [((0, 0, 0), (n, n, n))]
    try:
        launch2(BICG, np.float64, devs[:3], (0, 0, 0), box, 0.375, -1.25, 0)
        host[0] = bo.bicg_p(host[0], host[1], host[2], 0.375, -1.25)
        assert same(devs[0].get(), host[0])
        (pu,) = launch2(UPD, np.float64, devs, (0, 0, 0), box, -0.8125, 0.0, 2)
        xn, rn = ko.update(host[0], host[1], host[2], host[3], -0.8125)
        assert same(devs[0].get(), xn) and same(devs[2].get(), rn)
        assert rounded(pu[0]).sum == math.fsum((rn * rn).ravel().tolist())
        assert rounded(pu[1]).sum == math.fsum((host[4] * rn).ravel().tolist())
        assert pu[0].count == pu[1].count == n**3
    finally:
        for d in devs:
            d.free()
