"""Host-side checks of the fused residual-restriction and the multigrid solver (no GPU): the numpy rule of
tests/mg_oracle.py against a per-cell loop, every sb_transfer_oplan_create error, the new symbols, the hierarchy and
boundary-condition rules of stencil_b200.multigrid, and the convergence of the numpy cycle on inhomogeneous ODD(c) walls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import colour_oracle as co
import mg_oracle as mo
import stencil_b200 as sb
import transfer_oracle as to
from stencil_b200 import _lib
from stencil_b200._lib import I3, Pitched, StencilTerm, lib
from stencil_b200.multigrid import coarse_bc, level_count, residual_op

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEVEN = to.residual_terms(co.helmholtz(0.25, 0.5))
CORNERS = SEVEN + [(0, (1, 1, 1), 0.125), (0, (-1, 1, -1), -0.25)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lo,hi", [((0, 0, 0), (3, 4, 2)), ((-2, 1, 3), (1, 4, 5))])
@pytest.mark.parametrize("terms", [SEVEN, CORNERS, [t for t in SEVEN if t[0] == 0]])
def test_rule_is_the_loop(dtype, lo, hi, terms):
    rng = np.random.default_rng(3)
    so = (2 * lo[0] - 3, 2 * lo[1] - 1, 2 * lo[2] - 2)
    shape = tuple(2 * (hi[a] - lo[a]) + 5 for a in (2, 1, 0))
    src, aux = (rng.uniform(-1, 1, shape).astype(dtype) for _ in range(2))
    do = (lo[0] - 1, lo[1] - 2, lo[2])
    a = np.full(tuple(hi[k] - lo[k] + 3 for k in (2, 1, 0)), np.nan, dtype)
    b = a.copy()
    mo.restrict_op_box(a, do, terms, src, aux, so, lo, hi)
    mo.restrict_op_loop(b, do, terms, src, aux, so, lo, hi)
    assert np.array_equal(a, b, equal_nan=True)
    assert np.isnan(a).sum() == a.size - np.prod([hi[k] - lo[k] for k in range(3)])


def create(terms=SEVEN, dtype=2, dst=(0x10000, 64 * 8, 20), do=(0, 0, 0), dz=20, src=(0x200000, 130 * 8, 42), so=(-1, -1, -1), sz=42,
           aux=(0x400000, 130 * 8, 42), lo=((0, 0, 0),), hi=((8, 8, 8),)):
    arr = (StencilTerm * max(1, len(terms)))()
    for k, (s, o, w) in enumerate(terms):
        arr[k] = StencilTerm(s, (C.c_int32 * 3)(*o), w)
    L = (C.c_int64 * (3 * max(1, len(lo))))(*[v for b in lo for v in b])
    H = (C.c_int64 * (3 * max(1, len(hi))))(*[v for b in hi for v in b])
    h = C.c_void_p()
    rc = lib().sb_transfer_oplan_create(C.byref(h), 0, dtype, arr, len(terms), Pitched(*dst), I3(*do), dz, Pitched(*src), I3(*so), sz,
                                        Pitched(*aux), len(lo), L, H)
    return rc, lib().sb_last_error().decode()


@pytest.mark.parametrize("kw,msg", [
    (dict(dtype=0), "dtype 0 must be"),
    (dict(terms=[]), "an op has 1 to 64 terms, not 0"),
    (dict(terms=[(2, (0, 0, 0), 1.0)]), "term 0: source 2 must be"),
    (dict(terms=SEVEN + [(0, (2, 0, 0), 1.0)]), "term 8: offset (2, 0, 0) reaches beyond 1 cell"),
    (dict(aux=(None, 0, 0)), "a term reads aux, but aux is NULL"),
    (dict(dst=(None, 64 * 8, 20)), "dst and src must not be NULL"),
    (dict(src=(None, 130 * 8, 42)), "dst and src must not be NULL"),
    (dict(dst=(0x200000, 130 * 8, 42)), "dst must not be src"),
    (dict(dst=(0x400000, 130 * 8, 42)), "dst must not be aux"),
    (dict(aux=(0x400000, 130 * 8, 41)), "aux has another pitch or row count than src"),
    (dict(aux=(0x400004, 130 * 8, 42)), "aux: pointer and pitch must be positive multiples of the 8-byte element"),
    (dict(dst=(0x10004, 64 * 8, 20)), "dst: pointer and pitch must be positive multiples"),
    (dict(lo=((0, 3, 0),), hi=((8, 2, 8),)), "box 0: lo > hi on axis y"),
    (dict(hi=((65, 8, 8),)), "dst is written at cells 0 .. 64 on axis x, outside the allocation's 0 .. 63"),
    (dict(so=(0, -1, -1)), "the fused restriction reads fine cells -1 .. 16 on axis x"),
    (dict(sz=17, lo=((0, 0, 0),), hi=((8, 8, 8),)), "the fused restriction reads fine cells 0 .. 17 on axis z, outside the allocation's 0 .. 16"),
])
def test_oplan_errors(kw, msg):
    rc, err = create(**kw)
    assert rc == -1, (rc, err)
    assert msg in err, err


def test_oplan_without_aux_ignores_aux():
    """A plan whose op reads no aux takes aux NULL; the error checks come before any device call."""
    rc, err = create(terms=[t for t in SEVEN if t[0] == 0], aux=(None, 0, 0), hi=((8, 8, 0),))
    assert rc == 0, err


def test_new_symbols():
    with open(os.path.join(ROOT, "include", "stencil_b200.h")) as f:
        header = f.read()
    assert re.search(r"\bsb_transfer_oplan_create\(", header)
    assert "sb_transfer_oplan_create" in _lib._SIGS
    assert lib().sb_transfer_oplan_create is not None
    assert sb.Multigrid is not None


def test_level_count():
    assert level_count([(32, 32, 32)]) == 5  # 32 .. 2
    assert level_count([(32, 32, 32)], 4) == 4
    assert level_count([(16, 32, 32)] * 2) == 4  # 16 .. 2 per subdomain
    assert level_count([(32, 32, 32)] * 3) == 5
    assert level_count([(12, 8, 8)] * 4) == 3  # 12 -> 6 -> 3, then odd
    assert level_count([(8, 8, 8)] * 8) == 3
    assert level_count([(17, 16, 16)]) == 1
    assert level_count([(4, 4, 4)]) == 2
    assert level_count([(2, 4, 4)]) == 1  # a half of 1 is too small


def test_coarse_bc():
    assert coarse_bc(sb.BC.ODD(0.75)) == sb.BC.ODD(0.0)
    assert coarse_bc(sb.BC.EVEN()) == sb.BC.EVEN()
    with pytest.raises(sb.StencilError, match="VALUE walls"):
        coarse_bc(sb.BC.VALUE(1.0))
    with pytest.raises(sb.StencilError, match="ODD or EVEN"):
        coarse_bc(sb.BC.NONE())


def test_residual_op():
    A = sb.StencilOp(co.helmholtz(0.5, 1.0), np.float64)
    assert list(residual_op(A).terms) == [(1, (0, 0, 0), 1.0)] + [(0, o, -w) for _, o, w in co.helmholtz(0.5, 1.0)]


def test_cycle_clears_to_positive_zero():
    """The solver's cycle sets the coarse u to +0; transfer_oracle.vcycle's 0 * f gives -0 where f < 0: the same values."""
    lv = mo.hierarchy((8, 8, 8), 2, lambda l: co.helmholtz(2.0 ** l / 8, 0.0), np.float64, (False,) * 3, {f: ("odd", 0.0) for f in range(6)})
    ref = to.hierarchy((8, 8, 8), 2, 0.0, np.float64, (False,) * 3)
    f = np.random.default_rng(5).uniform(-1, 1, (8, 8, 8))
    lv[0].interior(lv[0].f)[...] = f
    ref[0].interior(ref[0].f)[...] = f
    mo.vcycle(lv)
    to.vcycle(ref)
    assert np.array_equal(lv[0].u, ref[0].u)


def cycle_factors(n, cycles=5):
    walls = {0: ("odd", 0.0), 1: ("odd", 0.25), 2: ("odd", -0.5), 3: ("odd", 1.0), 4: ("odd", 0.125), 5: ("odd", -1.0)}
    lv = mo.hierarchy((n, n, n), int(np.log2(n)) - 1, lambda l: co.helmholtz(2.0 ** l / n, 0.0), np.float64, (False,) * 3, walls)
    # a known discrete solution: u* smooth plus noise, f = A u* with u*'s ghost cells from the walls
    x = (np.arange(n) + 0.5) / n
    ustar = np.zeros((n + 2,) * 3)
    ustar[1:-1, 1:-1, 1:-1] = np.sin(np.pi * x)[None, None, :] * np.cos(2 * x)[None, :, None] * (1 + x)[:, None, None]
    mo.fill_ghosts(ustar, (False,) * 3, walls)
    import stencil_op_oracle as so

    so.apply_box(lv[0].A, ustar, None, lv[0].f, (1, 1, 1), (n, n, n))
    r = [lv[0].residual_norm()]
    for _ in range(cycles):
        mo.vcycle(lv)
        r.append(lv[0].residual_norm())
    return [r[k + 1] / r[k] for k in range(cycles)]


def test_cycle_converges_on_inhomogeneous_walls():
    """ODD(c) walls with a different c on each face: after the first cycle each factor is <= 0.15, and the factor of
    each cycle agrees within 0.02 between 16^3, 32^3 and 64^3."""
    fs = {n: cycle_factors(n) for n in (16, 32, 64)}
    for n, f in fs.items():
        assert max(f[1:]) <= 0.15, (n, f)
    for k in range(1, 5):
        vals = [fs[n][k] for n in fs]
        assert max(vals) - min(vals) < 0.02, (k, fs)
