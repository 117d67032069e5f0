"""Host-side checks of the multigrid transfers (no GPU): the numpy rule of tests/transfer_oracle.py against a per-cell
loop, the exact identities (weights, constants, linear fields), sb_transfer_check on pairing and non-pairing layouts,
every sb_transfer_plan_create error, the new symbols, and the h-independent convergence of the numpy V(2,2) cycle."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import stencil_b200 as sb
import transfer_oracle as to
from stencil_b200 import _lib
from stencil_b200._lib import I3, Pitched, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lo,hi", [((0, 0, 0), (3, 4, 2)), ((-2, 1, 3), (1, 4, 5)), ((5, -3, 0), (6, 2, 4))])
def test_restrict_box_is_the_loop(dtype, lo, hi):
    rng = np.random.default_rng(1)
    so = (2 * lo[0] - 3, 2 * lo[1] - 1, 2 * lo[2] - 2)
    src = rng.uniform(-1, 1, tuple(2 * (hi[a] - lo[a]) + 5 for a in (2, 1, 0))).astype(dtype)
    do = (lo[0] - 1, lo[1] - 2, lo[2])
    a = np.full(tuple(hi[a] - lo[a] + 3 for a in (2, 1, 0)), np.nan, dtype)
    b = a.copy()
    to.restrict_box(a, do, src, so, lo, hi)
    to.restrict_loop(b, do, src, so, lo, hi)
    assert np.array_equal(a, b, equal_nan=True)
    assert np.isnan(a).sum() == a.size - np.prod([hi[k] - lo[k] for k in range(3)])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lo,hi", [((0, 0, 0), (6, 4, 2)), ((-3, 1, 3), (2, 4, 8)), ((5, -3, 1), (6, 2, 4))])
@pytest.mark.parametrize("aux", [None, "dst", "other"])
def test_prolong_box_is_the_loop(dtype, lo, hi, aux):
    rng = np.random.default_rng(2)
    plo = [lo[a] // 2 - 1 for a in range(3)]
    phi = [(hi[a] - 1) // 2 + 2 for a in range(3)]
    so = tuple(plo[a] - 1 for a in range(3))
    src = rng.uniform(-1, 1, tuple(phi[a] - plo[a] + 2 for a in (2, 1, 0))).astype(dtype)
    do = (lo[0] - 2, lo[1] - 1, lo[2] - 3)
    shape = tuple(hi[a] - lo[a] + 4 for a in (2, 1, 0))
    a = rng.uniform(-1, 1, shape).astype(dtype)
    b = a.copy()
    other = rng.uniform(-1, 1, shape).astype(dtype)
    to.prolong_box(a, do, src, so, lo, hi, aux=None if aux is None else a if aux == "dst" else other)
    to.prolong_loop(b, do, src, so, lo, hi, aux=None if aux is None else b if aux == "dst" else other)
    assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------ exact identities
def test_prolongation_weights_sum_to_one():
    assert sum(w for w, _ in to.PROLONG_ORDER) == 64
    for T in (np.float32, np.float64):
        assert sum(T(w / 64.0) for w, _ in to.PROLONG_ORDER) == T(1)
        for w, _ in to.PROLONG_ORDER:
            assert float(T(w / 64.0)) == w / 64.0  # exact in both types


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_constant_restricts_and_prolongs_to_itself(dtype):
    c = dtype(-0.8125)
    fine = np.full((10, 12, 8), c, dtype)
    coarse = np.full((5, 6, 4), np.nan, dtype)
    to.restrict_box(coarse, (0, 0, 0), fine, (0, 0, 0), (0, 0, 0), (4, 6, 5))
    assert np.all(coarse == c)
    back = np.full((10, 12, 8), np.nan, dtype)
    to.prolong_box(back, (0, 0, 0), coarse, (0, 0, 0), (2, 2, 2), (6, 10, 8))
    assert np.all(back[2:8, 2:10, 2:6] == c)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_linear_fields(dtype):
    """phi = g . (p + 1/2) + c0 on fine cell centres; the coarse cell I has its centre at fine coordinate 2 I + 1.  Away
    from the wrap, prolongation of the coarse samples gives the fine samples, and restriction of the fine ones the coarse
    ones, exactly (every value dyadic)."""
    g, c0 = (0.5, -0.25, 1.0), 3.0
    n = 16
    z, y, x = np.indices((n, n, n))
    fine = (g[0] * (x + 0.5) + g[1] * (y + 0.5) + g[2] * (z + 0.5) + c0).astype(dtype)
    Z, Y, X = np.indices((n // 2,) * 3)
    coarse = (g[0] * (2 * X + 1) + g[1] * (2 * Y + 1) + g[2] * (2 * Z + 1) + c0).astype(dtype)
    got = np.full_like(coarse, np.nan)
    to.restrict_box(got, (0, 0, 0), fine, (0, 0, 0), (0, 0, 0), (n // 2,) * 3)
    assert np.array_equal(got, coarse)
    back = np.full_like(fine, np.nan)
    to.prolong_box(back, (0, 0, 0), coarse, (0, 0, 0), (2, 2, 2), (n - 2,) * 3)
    assert np.array_equal(back[2:-2, 2:-2, 2:-2], fine[2:-2, 2:-2, 2:-2])


# ------------------------------------------------------------------------------------------ sb_transfer_check
def layouts(size, dim, scale=1):
    """(origins, sizes) of an even cut of size into dim parts, x fastest, scaled by 1 / scale."""
    idx = [(i, j, k) for k in range(dim[2]) for j in range(dim[1]) for i in range(dim[0])]
    base = [size[a] // dim[a] for a in range(3)]
    return [tuple(i[a] * base[a] // scale for a in range(3)) for i in idx], [tuple(base[a] // scale for a in range(3)) for i in idx]


def check(fdim, cdim, fo, fs, co_, cs, radius=None):
    sb.transfer_check(fdim, cdim, fo, fs, co_, cs, radius)


def test_check_accepts_pairing_layouts():
    for dim in ((1, 1, 1), (2, 1, 1), (3, 1, 1), (2, 2, 1), (2, 2, 2)):
        size = (96, 32, 32) if dim == (3, 1, 1) else (32, 32, 32)
        fo, fs = layouts(size, dim)
        co_, cs = layouts(size, dim, 2)
        check(dim, dim, fo, fs, co_, cs)
        check(dim, dim, fo, fs, co_, cs, sb.Radius.constant(1))


def test_check_rejects():
    fo, fs = layouts((32, 32, 32), (2, 2, 1))
    co_, cs = layouts((32, 32, 32), (2, 2, 1), 2)
    with pytest.raises(sb.StencilError, match="fine partition is 2 x 2 x 1 subdomains, the coarse one 4 x 1 x 1"):
        check((2, 2, 1), (4, 1, 1), fo, fs, co_, cs)
    bad = list(cs)
    bad[3] = (8, 8, 15)  # an odd fine size cannot pair
    with pytest.raises(sb.StencilError, match=r"subdomain \(1, 1, 0\): fine size 32 on axis z is not twice the coarse size 15"):
        check((2, 2, 1), (2, 2, 1), fo, fs, co_, bad)
    shifted = list(co_)
    shifted[1] = (9, 0, 0)
    with pytest.raises(sb.StencilError, match=r"subdomain \(1, 0, 0\): fine origin 16 on axis x is not twice the coarse origin 9"):
        check((2, 2, 1), (2, 2, 1), fo, fs, shifted, cs)
    # an uneven cut of 33 cells leaves an odd subdomain
    with pytest.raises(sb.StencilError, match="fine size 17 on axis x"):
        check((2, 1, 1), (2, 1, 1), [(0, 0, 0), (17, 0, 0)], [(17, 8, 8), (16, 8, 8)], [(0, 0, 0), (8, 0, 0)], [(8, 4, 4), (8, 4, 4)])
    fo1, fs1 = layouts((16, 16, 16), (1, 1, 1))
    co1, cs1 = layouts((16, 16, 16), (1, 1, 1), 2)
    check((1, 1, 1), (1, 1, 1), fo1, fs1, co1, cs1, sb.Radius.face_edge_corner(1, 1, 1))
    with pytest.raises(sb.StencilError, match=r"direction \(-1, -1, -1\) is 0"):
        check((1, 1, 1), (1, 1, 1), fo1, fs1, co1, cs1, sb.Radius.face_edge_corner(1, 1, 0))
    with pytest.raises(sb.StencilError, match=r"direction \(-1, -1, -1\) is 0"):
        check((1, 1, 1), (1, 1, 1), fo1, fs1, co1, cs1, sb.Radius.face_edge_corner(1, 0, 0))
    r = sb.Radius.constant(1)
    r.set_dir((0, 1, 0), 0)
    with pytest.raises(sb.StencilError, match=r"direction \(0, 1, 0\) is 0"):
        check((1, 1, 1), (1, 1, 1), fo1, fs1, co1, cs1, r)
    check((1, 1, 1), (1, 1, 1), fo1, fs1, co1, cs1, None)  # restriction needs no ghost cells


# ------------------------------------------------------------------------------------------ plan-creation errors
def create(dtype=2, kind=0, dst=(0x10000, 64 * 8, 20), do=(0, 0, 0), dz=20, src=(0x200000, 128 * 8, 40), so=(0, 0, 0), sz=40,
           aux=(None, 0, 0), lo=(0, 0, 0), hi=(8, 8, 8)):
    h = C.c_void_p()
    rc = lib().sb_transfer_plan_create(C.byref(h), 0, dtype, kind, Pitched(*dst), I3(*do), dz, Pitched(*src), I3(*so), sz, Pitched(*aux),
                                       I3(*lo), I3(*hi))
    return rc, lib().sb_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=0), "dtype 0 must be"),
    (dict(dtype=3), "dtype 3 must be"),
    (dict(kind=2), "kind 2 must be"),
    (dict(kind=-1), "kind -1 must be"),
    (dict(dst=(0x200000, 128 * 8, 40)), "dst must not be src"),
    (dict(kind=1, src=(0x10000, 64 * 8, 20)), "dst must not be src"),
    (dict(aux=(0x300000, 64 * 8, 20)), "a restriction takes no aux"),
    (dict(kind=1, aux=(0x300000, 64 * 8, 21)), "aux has another pitch or row count than dst"),
    (dict(dst=(0x10004, 64 * 8, 20)), "dst: pointer and pitch must be positive multiples of the 8-byte element"),
    (dict(src=(0x200000, 128 * 8 + 4, 40)), "src: pointer and pitch must be positive multiples"),
    (dict(kind=1, aux=(0x300002, 64 * 8, 20)), "aux: pointer and pitch"),
    (dict(lo=(0, 3, 0), hi=(8, 2, 8)), "lo > hi on axis y"),
    (dict(hi=(65, 8, 8)), "dst is written at cells 0 .. 64 on axis x, outside the allocation's 0 .. 63"),
    (dict(do=(0, 0, 1)), "dst is written at cells -1 .. 6 on axis z"),
    (dict(dst=(0x10000, 32 * 8, 20), dz=20, hi=(8, 8, 20), src=(0x200000, 128 * 8, 40), sz=39), "the restriction reads fine cells 0 .. 39 on axis z"),
    (dict(so=(1, 0, 0)), "the restriction reads fine cells -1 .. 14 on axis x"),
    (dict(kind=1, dst=(0x10000, 16 * 8, 16), dz=16, src=(0x200000, 9 * 8, 10), sz=10, so=(-1, -1, -1), lo=(0, 0, 0), hi=(16, 16, 16)),
     "the prolongation reads coarse cells 0 .. 9 on axis x, outside the allocation's 0 .. 8"),
    (dict(kind=1, dst=(0x10000, 16 * 8, 16), dz=16, src=(0x200000, 10 * 8, 10), sz=10, so=(0, -1, -1), lo=(1, 0, 0), hi=(16, 16, 16)),
     "the prolongation reads coarse cells -1 .. 8 on axis x"),
])
def test_plan_errors(kw, msg):
    rc, err = create(**kw)
    assert rc == -1, (rc, err)
    assert msg in err, err


def test_plan_error_null_buffers():
    rc, err = create(dst=(None, 64 * 8, 20))
    assert rc == -1 and "dst and src must not be NULL" in err


# ------------------------------------------------------------------------------------------ symbols
def test_new_symbols():
    names = ["sb_transfer_check", "sb_transfer_plan_create", "sb_transfer_plan_launch", "sb_transfer_plan_bytes", "sb_transfer_plan_destroy"]
    with open(os.path.join(ROOT, "include", "stencil_b200.h")) as f:
        header = f.read()
    for n in names:
        assert re.search(rf"\b{n}\(", header), n
        assert n in _lib._SIGS
        assert getattr(lib(), n) is not None
    assert "SB_TRANSFER_RESTRICT = 0, SB_TRANSFER_PROLONG = 1" in header
    assert (_lib.TRANSFER_RESTRICT, _lib.TRANSFER_PROLONG) == (0, 1)
    assert lib().sb_transfer_plan_bytes(None) == 0
    assert lib().sb_transfer_plan_destroy(None) == 0
    assert lib().sb_transfer_plan_launch(None, None) == -1


# ------------------------------------------------------------------------------------------ the numpy V(2,2) cycle
def cycle_factors(n, periodic, sigma, cycles=6):
    lv = to.hierarchy((n, n, n), int(np.log2(n)), sigma, np.float64, periodic)  # down to 2^3
    lv[0].interior(lv[0].f)[...] = np.random.default_rng(0).standard_normal((n, n, n))
    r = [to.residual_norm(lv[0])]
    for _ in range(cycles):
        to.vcycle(lv, coarse_sweeps=50)
        r.append(to.residual_norm(lv[0]))
    return [r[k + 1] / r[k] for k in range(cycles)]


@pytest.mark.parametrize("walls", ["odd", "periodic"])
def test_vcycle_converges_independently_of_h(walls):
    """V(2,2), red-black Gauss-Seidel, 8-cell restriction, trilinear prolongation, rediscretised coarse operators:
    ODD(0) Poisson and periodic Helmholtz (sigma = 1).  After the first cycle each factor is <= 0.15, and the factor
    of each cycle differs by < 0.02 between 16^3, 32^3 and 64^3."""
    periodic, sigma = ((False,) * 3, 0.0) if walls == "odd" else ((True,) * 3, 1.0)
    fs = {n: cycle_factors(n, periodic, sigma) for n in (16, 32, 64)}
    for n, f in fs.items():
        assert max(f[1:]) <= 0.15, (n, f)
    for k in range(1, 6):
        vals = [fs[n][k] for n in fs]
        assert max(vals) - min(vals) < 0.02, (k, fs)
