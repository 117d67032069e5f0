"""Host-side checks of the variable-coefficient stencil operators (no GPU): the numpy oracle of tests/vstencil_oracle.py
against a per-cell loop, against the constant-coefficient oracle with every coefficient 1, against the analytic
div(kappa grad u) (second-order convergence) and against the telescoping sum of a conservative op; sb_stencil_div_grad
against a restatement; sb_stencil_vcheck against the rule; every sb_stencil_vplan_create error that needs no device; the
C layout of sb_stencil_vterm; the Python StencilOp with coefficient terms."""
import ctypes as C
import itertools
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import stencil_b200 as sb
import stencil_op_oracle as so
import vstencil_oracle as vo
from stencil_b200._lib import Pitched, StencilVTerm, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIRS = [(x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]


def c_vterms(terms):
    arr = (StencilVTerm * max(1, len(terms)))()
    for k, t in enumerate(terms):
        s, o, w, c, co = vo.split(t)
        arr[k] = StencilVTerm(s, (C.c_int32 * 3)(*o), c, (C.c_int32 * 3)(*co), w)
    return arr


def heat(spacing, dt):
    return [(s, o, dt * w, k, c) for s, o, w, k, c in vo.div_grad(spacing)] + [(0, (0, 0, 0), 1.0)]


def mix(seed=0):
    """All four fields, coefficient offsets in all 27 directions, a coefficient on an aux term, plain terms between."""
    rng = np.random.default_rng(seed)
    terms = [(0, DIRS[(7 * i) % 27], float(rng.uniform(-1, 1)), i % 4, c) for i, c in enumerate(DIRS)]
    return terms[:13] + [(1, (0, 0, 0), -0.75, 2, (1, 0, -1)), (0, (2, 0, -1), 0.3)] + terms[13:] + [(1, (0, 0, 0), 0.5)]


OPS = {"heat": heat((0.3, 0.7, 1.1), 0.01), "div_grad": vo.div_grad((1.0, 0.9, 1.3)),
       "c2lap4": [(0, o, w, 0, (0, 0, 0)) for _, o, w in so.laplacian(4, (0.049, 0.061, 0.037))], "mix": mix()}


# ------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", list(OPS))
def test_oracle_matches_cell_loop(dtype, op):
    rng = np.random.default_rng(7)
    terms = OPS[op]
    rm, rp = vo.reach(terms)
    ext = (5, 4, 3)
    shape = tuple(ext[a] + rm[a] + rp[a] + 1 for a in range(3))[::-1]
    src, aux = rng.uniform(-1, 1, shape).astype(dtype), rng.uniform(-1, 1, shape).astype(dtype)
    coefs = [rng.uniform(0.5, 2, shape).astype(dtype) for _ in range(4)]
    a, b = np.full(shape, np.nan, dtype), np.full(shape, np.nan, dtype)
    vo.apply_box(terms, src, aux, coefs, a, rm, ext)
    vo.apply_cell_loop(terms, src, aux, coefs, b, rm, ext)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", list(OPS))
def test_unit_coefficients_give_the_plain_op(dtype, op):
    """T(w) * 1 is exact, so with every C = 1 the rule is the constant-coefficient rule of the plain terms."""
    rng = np.random.default_rng(8)
    terms = OPS[op]
    rm, rp = vo.reach(terms)
    ext = (6, 5, 4)
    shape = tuple(ext[a] + rm[a] + rp[a] for a in range(3))[::-1]
    src, aux = rng.uniform(-1, 1, shape).astype(dtype), rng.uniform(-1, 1, shape).astype(dtype)
    ones = [np.ones(shape, dtype)] * 4
    a, b = np.zeros(shape, dtype), np.zeros(shape, dtype)
    vo.apply_box(terms, src, aux, ones, a, rm, ext)
    so.apply_box([tuple(t[:3]) for t in terms], src, aux, b, rm, ext)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_div_grad_converges_at_second_order():
    """kappa = 1 + 0.5 sin x cos y, u = sin(x + 2y) cos z on a periodic 2 pi cube (anisotropic cell counts), kappa
    sampled on the faces: the max error against the analytic div(kappa grad u) falls by about 4 per halving of h."""
    errs = []
    for n in (16, 32, 64):
        nx, ny, nz = n, n + n // 2, n // 2 + 4
        h = (2 * np.pi / nx, 2 * np.pi / ny, 2 * np.pi / nz)
        z, y, x = np.meshgrid(np.arange(nz) * h[2], np.arange(ny) * h[1], np.arange(nx) * h[0], indexing="ij")
        kap = lambda x, y, z: 1 + 0.5 * np.sin(x) * np.cos(y)  # noqa: E731
        u = np.sin(x + 2 * y) * np.cos(z)
        coefs = [kap(x - h[0] / 2, y, z), kap(x, y - h[1] / 2, z), kap(x, y, z - h[2] / 2)]
        got = vo.apply_periodic(vo.div_grad(h), u, None, coefs)
        k, kx, ky = kap(x, y, z), 0.5 * np.cos(x) * np.cos(y), -0.5 * np.sin(x) * np.sin(y)
        ux, uy, uz = np.cos(x + 2 * y) * np.cos(z), 2 * np.cos(x + 2 * y) * np.cos(z), -np.sin(x + 2 * y) * np.sin(z)
        lap = -5 * np.sin(x + 2 * y) * np.cos(z) - np.sin(x + 2 * y) * np.cos(z)
        want = kx * ux + ky * uy + k * lap
        _ = uz
        errs.append(float(np.abs(got - want).max()))
    rates = [math.log2(errs[i] / errs[i + 1]) for i in range(2)]
    assert all(1.8 < r < 2.3 for r in rates), (errs, rates)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_div_grad_is_conservative(dtype):
    """In exact arithmetic the div-grad terms telescope to zero over a periodic grid, so the exactly rounded sum of the
    oracle's cells lies within sum over cells of gamma_{n+2} * sum_t |m_t| (n + 1 roundings of the sum, one more for the
    second multiply), with m_t the exact products of the rounded inputs."""
    rng = np.random.default_rng(21)
    spacing = (0.3, 0.7, 1.1)
    terms = vo.div_grad(spacing)
    shape = (6, 7, 9)
    u = rng.uniform(-1, 1, shape).astype(dtype)
    coefs = [rng.uniform(0.1, 3, shape).astype(dtype) for _ in range(3)]
    out = vo.apply_periodic(terms, u, None, coefs)
    uu = float(np.finfo(dtype).eps) / 2
    n = len(terms)
    gamma = (n + 2) * uu / (1 - (n + 2) * uu)
    T = np.dtype(dtype).type
    bound = 0.0
    for t in terms:
        s, o, w, k, c = vo.split(t)
        cv = np.roll(coefs[k], (-c[2], -c[1], -c[0]), axis=(0, 1, 2)).astype(np.float64)
        sv = np.roll(u, (-o[2], -o[1], -o[0]), axis=(0, 1, 2)).astype(np.float64)
        bound += math.fsum(np.abs(float(T(w)) * cv * sv).ravel())
    total = math.fsum(out.astype(np.float64).ravel())
    assert abs(total) <= gamma * bound * 1.0000001, (total, gamma * bound)
    assert bound > 0


# ------------------------------------------------------------------------------------------ sb_stencil_div_grad
@pytest.mark.parametrize("spacing", [(1.0, 1.0, 1.0), (0.049, 0.061, 0.037), (3.0, 0.5, 1e-3)])
def test_div_grad_table(spacing):
    h = (C.c_double * 3)(*spacing)
    assert lib().sb_stencil_div_grad(h, None, 0) == 12
    buf = (StencilVTerm * 12)()
    assert lib().sb_stencil_div_grad(h, buf, 12) == 12
    got = [(t.source, tuple(t.offset), t.weight, t.coef, tuple(t.coef_offset)) for t in buf]
    want = vo.div_grad(spacing)
    assert [(s, o, k, c) for s, o, _, k, c in got] == [(s, o, k, c) for s, o, _, k, c in want]
    assert [w.hex() for _, _, w, _, _ in got] == [w.hex() for _, _, w, _, _ in want]
    part = (StencilVTerm * 5)()
    assert lib().sb_stencil_div_grad(h, part, 5) == 12 and [t.weight for t in part] == [t.weight for t in buf[:5]]
    op = sb.StencilOp.div_grad(spacing, np.float64)
    assert op.terms == tuple(want) and op.has_coef and op.ncoef == 3 and not op.has_aux


@pytest.mark.parametrize("spacing", [(0, 1, 1), (1, -1, 1), (1, 1, float("inf")), (float("nan"), 1, 1)])
def test_div_grad_rejects(spacing):
    assert lib().sb_stencil_div_grad((C.c_double * 3)(*spacing), None, 0) == -1
    assert "spacing" in lib().sb_last_error().decode()
    with pytest.raises(sb.StencilError, match="spacing"):
        sb.StencilOp.div_grad(spacing, np.float32)


def test_div_grad_bad_output():
    assert lib().sb_stencil_div_grad((C.c_double * 3)(1, 1, 1), None, 3) == -1
    assert "bad output buffer" in lib().sb_last_error().decode()


# ------------------------------------------------------------------------------------------ sb_stencil_vcheck
def radii():
    asym = sb.Radius.constant(1)
    asym.set_dir((1, 0, 0), 2)
    asym.set_dir((0, -1, 0), 3)
    asym.set_dir((0, 0, 1), 0)
    left = sb.Radius.constant(0)
    left.set_dir((-1, 0, 0), 4)
    return {"f1": sb.Radius.face_edge_corner(1, 0, 0), "f1e1": sb.Radius.face_edge_corner(1, 1, 0), "fec1": sb.Radius.face_edge_corner(1, 1, 1),
            "f2e1": sb.Radius.face_edge_corner(2, 1, 0), "c4": sb.Radius.constant(4), "asym": asym, "left4": left}


@pytest.mark.parametrize("rname", list(radii()))
def test_vcheck_every_offset(rname):
    """Every src offset in [-5, 5]^3 (with a centre coefficient) and every coefficient offset in [-2, 2]^3 (on a centre
    term, on a src offset of reach 1 and on an aux term), as a one-term op and behind a centre term, accepted exactly
    when the rule says so."""
    r = radii()[rname]
    r27 = list(r.c27())
    cases = [(0, o, 1.0, 1, (0, 0, 0)) for o in itertools.product(range(-5, 6), repeat=3)]
    for c in itertools.product(range(-2, 3), repeat=3):
        cases += [(0, (0, 0, 0), 1.0, 3, c), (1, (0, 0, 0), 1.0, 0, c)] + [(0, o, 1.0, 2, c) for o in DIRS[::5]]
    accepted = 0
    for t in cases:
        for terms in ([t], [(0, (0, 0, 0), -1.0), t]):
            want = vo.check_rule(terms, r27)
            rc = lib().sb_stencil_vcheck(c_vterms(terms), len(terms), r.c27())
            assert rc == (0 if want else -1), (t, rc)
            if not want:
                assert "term" in lib().sb_last_error().decode()
            accepted += want
    assert accepted > 0


@pytest.mark.parametrize("terms,what", [
    ([(0, (0, 0, 0), 1.0, 4, (0, 0, 0))], "coefficient field 4"),
    ([(0, (0, 0, 0), 1.0, -2, (0, 0, 0))], "coefficient field -2"),
    ([(0, (0, 0, 0), 1.0, 0, (2, 0, 0))], "reaches beyond 1 cell"),
    ([(0, (0, 0, 0), 1.0, 0, (0, 0, -2))], "reaches beyond 1 cell"),
    ([(0, (0, 0, 0), 1.0, -1, (0, 1, 0))], "without a coefficient field"),
    ([(1, (1, 0, 0), 1.0, 0, (0, 0, 0))], "aux term"),
    ([(0, (5, 0, 0), 1.0, 0, (0, 0, 0))], "reaches beyond 4"),
    ([], "1 to 64 terms"),
])  # fmt: skip
def test_vcheck_limits(terms, what):
    assert lib().sb_stencil_vcheck(c_vterms(terms), len(terms), sb.Radius.constant(4).c27()) == -1
    assert what in lib().sb_last_error().decode()
    if terms and terms[0][3] != -1:
        with pytest.raises(sb.StencilError, match=what):
            sb.StencilOp(terms, np.float64)


def test_plain_check_unchanged_through_vcheck():
    """sb_stencil_check is sb_stencil_vcheck on the same terms without coefficients."""
    r = radii()["asym"]
    for o in itertools.product(range(-3, 4), repeat=3):
        plain = [(0, (0, 0, 0), 1.0), (0, o, 0.5)]
        v = [(0, (0, 0, 0), 1.0, -1, (0, 0, 0)), (0, o, 0.5, -1, (0, 0, 0))]
        a = lib().sb_stencil_check(so_terms(plain), 2, r.c27())
        b = lib().sb_stencil_vcheck(c_vterms(v), 2, r.c27())
        assert a == b


def so_terms(terms):
    from stencil_b200._lib import StencilTerm

    arr = (StencilTerm * len(terms))()
    for k, (s, o, w) in enumerate(terms):
        arr[k] = StencilTerm(s, (C.c_int32 * 3)(*o), w)
    return arr


# ------------------------------------------------------------------------------------------ sb_stencil_vplan_create errors
ES = 8
DST, SRC, AUX = Pitched(0x100000, 12 * ES, 12), Pitched(0x200000, 12 * ES, 12), Pitched(0x300000, 12 * ES, 12)
K = [Pitched(0x400000 + 0x10000 * k, 12 * ES, 12) for k in range(4)]


def plan_args(**kw):
    """Valid arguments for an F64 div-grad plan over a 10^3 box inside a 12^3 allocation at fake (never dereferenced)
    addresses; kw overrides."""
    a = dict(dtype=2, terms=vo.div_grad((1, 1, 1)), dst=DST, src=SRC, aux=Pitched(None, 0, 0), coefs=K[:3], ncoef=None, acc=(-1, -1, -1),
             zsize=12, boxes=[((0, 0, 0), (10, 10, 10))])
    a.update(kw)
    return a


def create(a):
    h = C.c_void_p()
    nb = len(a["boxes"])
    lo = (C.c_int64 * (3 * max(1, nb)))(*[v for b in a["boxes"] for v in b[0]])
    hi = (C.c_int64 * (3 * max(1, nb)))(*[v for b in a["boxes"] for v in b[1]])
    cs = a["coefs"]
    carr = (Pitched * max(1, len(cs or [])))(*(cs or []))
    nc = len(cs or []) if a["ncoef"] is None else a["ncoef"]
    rc = lib().sb_stencil_vplan_create(C.byref(h), 0, a["dtype"], c_vterms(a["terms"]), len(a["terms"]), a["dst"], a["src"], a["aux"],
                                       carr if cs is not None else None, nc, (C.c_int64 * 3)(*a["acc"]), a["zsize"], nb, lo, hi)
    if rc == 0:
        lib().sb_stencil_plan_destroy(h)
    return rc, lib().sb_last_error().decode()


@pytest.mark.parametrize("kw,what", [
    (dict(ncoef=5, coefs=K + K[:1]), "ncoef 5"),
    (dict(ncoef=-1), "ncoef -1"),
    (dict(coefs=None, ncoef=3), "coefficient array is NULL"),
    (dict(coefs=K[:2]), "names coefficient field 2, but ncoef is 2"),
    (dict(coefs=[]), "names coefficient field 0, but ncoef is 0"),
    (dict(coefs=[K[0], Pitched(None, 12 * ES, 12), K[2]]), "coefficient field 1 is NULL"),
    (dict(terms=[(0, (0, 0, 0), 1.0, 0, (0, 2, 0))]), "reaches beyond 1 cell"),
    (dict(terms=[(0, (0, 0, 0), 1.0, 4, (0, 0, 0))]), "coefficient field 4"),
    (dict(coefs=[K[0], DST, K[2]]), "coefficient field 1 is dst"),
    (dict(coefs=[K[0], K[1], Pitched(0x420000, 13 * ES, 12)]), "coefficient field 2 has another pitch"),
    (dict(coefs=[Pitched(0x400000, 12 * ES, 11), K[1], K[2]]), "coefficient field 0 has another pitch"),
    (dict(coefs=[K[0], Pitched(0x410004, 12 * ES, 12), K[2]]), "coefficient field 1: pointer and pitch"),
    (dict(boxes=[((0, 0, 0), (11, 10, 10))]), "outside the allocation"),
    (dict(terms=[(0, (0, 0, 0), 1.0, 0, (1, 0, 0))], boxes=[((0, 0, 0), (11, 10, 10))]), "coefficient field 0 is read at cells"),
    (dict(terms=[(0, (0, 0, 0), 1.0, 1, (0, -1, 0))], boxes=[((0, -1, 0), (10, 10, 10))]), "coefficient field 1 is read at cells"),
    (dict(terms=[(0, (0, 0, 0), 1.0, 2, (0, 0, 1))], zsize=11), "coefficient field 2 is read at cells"),
    (dict(dtype=0), "dtype"),
    (dict(terms=[(0, (0, 0, 0), 1.0), (1, (0, 0, 0), 1.0, 0, (0, 0, 0))]), "aux is NULL"),
    (dict(dst=SRC), "dst must not be src"),
])  # fmt: skip
def test_vplan_create_errors(kw, what):
    rc, msg = create(plan_args(**kw))
    assert rc == -1 and what in msg, msg


def test_vplan_create_null_handle():
    assert lib().sb_stencil_vplan_create(None, 0, 2, c_vterms(vo.div_grad((1, 1, 1))), 12, DST, SRC, Pitched(None, 0, 0), (Pitched * 3)(*K[:3]),
                                         3, (C.c_int64 * 3)(0, 0, 0), 12, 0, None, None) == -1


# ------------------------------------------------------------------------------------------ C layout
@pytest.mark.skipif(shutil.which("cc") is None and shutil.which("gcc") is None, reason="no C compiler")
def test_vterm_layout_matches_ctypes(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "stencil_b200.h"\n'
        "int main(void) { printf(\"%zu %zu %zu %zu %zu %zu %d %d\\n\", offsetof(sb_stencil_vterm, source), offsetof(sb_stencil_vterm, offset),"
        " offsetof(sb_stencil_vterm, coef), offsetof(sb_stencil_vterm, coef_offset), offsetof(sb_stencil_vterm, weight),"
        " sizeof(sb_stencil_vterm), SB_STENCIL_MAX_COEFS, SB_STENCIL_COEF_REACH); return 0; }\n"
    )
    exe = tmp_path / "probe"
    cc = shutil.which("cc") or shutil.which("gcc")
    subprocess.check_call([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    V = StencilVTerm
    assert got == [V.source.offset, V.offset.offset, V.coef.offset, V.coef_offset.offset, V.weight.offset, C.sizeof(V), 4, 1]
    from stencil_b200 import _lib

    assert (_lib.STENCIL_MAX_COEFS, _lib.STENCIL_COEF_REACH) == (4, 1)


# ------------------------------------------------------------------------------------------ Python StencilOp
def test_op_with_coefficients():
    a = sb.StencilOp(OPS["mix"], np.float64)
    assert a.has_coef and a.has_aux and a.ncoef == 4 and a.reach() == 2
    assert sb.StencilOp(OPS["c2lap4"], np.float32).ncoef == 1
    # a 5-tuple with coef -1 is the plain term
    p = sb.StencilOp([(0, (1, 0, 0), 0.5, -1, (0, 0, 0))], np.float64)
    assert p == sb.StencilOp([(0, (1, 0, 0), 0.5)], np.float64) and not p.has_coef and p.ncoef == 0
    # key() tells apart ops that differ only in a coefficient field or offset
    base = [(0, (1, 0, 0), 0.5, 0, (0, 0, 0))]
    keys = {sb.StencilOp(t, np.float64).key() for t in (base, [(0, (1, 0, 0), 0.5, 1, (0, 0, 0))], [(0, (1, 0, 0), 0.5, 0, (1, 0, 0))],
                                                          [(0, (1, 0, 0), 0.5)])}
    assert len(keys) == 4
    assert sb.StencilOp(base, np.float64) == sb.StencilOp([(0, [1, 0, 0], 0.5, 0, [0, 0, 0])], np.float64)
    # scaled() keeps the coefficient part
    s = sb.StencilOp.div_grad((1, 2, 3), np.float64).scaled(0.25)
    assert [t[3:] for t in s.terms] == [t[3:] for t in vo.div_grad((1, 2, 3))]
    assert [t[2] for t in s.terms] == [0.25 * t[2] for t in vo.div_grad((1, 2, 3))]


def test_op_validation():
    with pytest.raises(sb.StencilError, match="without a coefficient field"):
        sb.StencilOp([(0, (0, 0, 0), 1.0, -1, (1, 0, 0))], np.float64)
    with pytest.raises(sb.StencilError, match="weight"):
        sb.StencilOp([(0, (0, 0, 0), 1.0, 0)], np.float64)
    with pytest.raises(sb.StencilError, match="coefficient offset"):
        sb.StencilOp([(0, (0, 0, 0), 1.0, 2, (0, 0, 1))], np.float64).check(sb.Radius.face_edge_corner(0, 0, 0))
    op = sb.StencilOp([(0, (0, 0, 0), 1.0, 0, (1, 1, 0))], np.float64)
    op.check(sb.Radius.face_edge_corner(1, 1, 0))
    with pytest.raises(sb.StencilError, match="coefficient offset"):
        op.check(sb.Radius.face_edge_corner(1, 0, 0))
