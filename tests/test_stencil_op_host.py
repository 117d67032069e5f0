"""Host-side checks of the linear stencil operators (no GPU): the numpy oracle against a per-cell loop and against an
exactly rounded sum, sb_stencil_laplacian against an independent coefficient table, sb_stencil_check against the rule,
every sb_stencil_plan_create error that needs no device, and the C layout of sb_stencil_term against ctypes."""
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
from stencil_b200._lib import I27, Pitched, StencilTerm, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def c_terms(terms):
    arr = (StencilTerm * max(1, len(terms)))()
    for k, (s, o, w) in enumerate(terms):
        arr[k] = StencilTerm(s, (C.c_int32 * 3)(*o), w)
    return arr


def box27(seed=3):
    rng = np.random.default_rng(seed)
    return [(0, (x, y, z), float(rng.uniform(-1, 1))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]


# ------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", ["lap2", "lap8", "box27", "aux"])
def test_oracle_matches_cell_loop(dtype, op):
    rng = np.random.default_rng(7)
    terms = {"lap2": so.laplacian(2, (0.3, 0.7, 1.1)), "lap8": so.laplacian(8, (0.049, 0.061, 0.037)), "box27": box27(),
             "aux": so.laplacian(2, (1, 1, 1)) + [(1, (0, 0, 0), -0.37), (0, (0, 0, 0), 2.0)]}[op]
    rm, rp = so.reach(terms)
    ext = (5, 4, 3)
    shape = tuple(ext[a] + rm[a] + rp[a] + 1 for a in range(3))[::-1]
    src = rng.uniform(-1, 1, shape).astype(dtype)
    aux = rng.uniform(-1, 1, shape).astype(dtype)
    a, b = np.full(shape, np.nan, dtype), np.full(shape, np.nan, dtype)
    so.apply_box(terms, src, aux, a, rm, ext)
    so.apply_cell_loop(terms, src, aux, b, rm, ext)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_oracle_within_summation_bound(dtype):
    """Each cell is within gamma_{n+1} * sum |T(w) v| of the exactly rounded sum of the products."""
    rng = np.random.default_rng(11)
    terms = so.laplacian(8, (0.049, 0.061, 0.037)) + box27(5)
    ext = (4, 3, 3)
    shape = tuple(e + 8 for e in ext)[::-1]
    src = rng.uniform(-1, 1, shape).astype(dtype)
    out = np.zeros(shape, dtype)
    so.apply_box(terms, src, None, out, (4, 4, 4), ext)
    u = float(np.finfo(dtype).eps) / 2
    n = len(terms)
    gamma = (n + 1) * u / (1 - (n + 1) * u)
    T = np.dtype(dtype).type
    for z, y, x in itertools.product(range(ext[2]), range(ext[1]), range(ext[0])):
        prods = [float(T(w)) * float(src[4 + z + o[2], 4 + y + o[1], 4 + x + o[0]]) for _, o, w in terms]
        exact = math.fsum(prods)
        bound = gamma * math.fsum(abs(p) for p in prods) + 2 * u * abs(exact)
        assert abs(float(out[4 + z, 4 + y, 4 + x]) - exact) <= bound


# ------------------------------------------------------------------------------------------ sb_stencil_laplacian
@pytest.mark.parametrize("order", [2, 4, 6, 8])
@pytest.mark.parametrize("spacing", [(1.0, 1.0, 1.0), (0.049, 0.061, 0.037), (3.0, 0.5, 1e-3)])
def test_laplacian_table(order, spacing):
    h = (C.c_double * 3)(*spacing)
    n = lib().sb_stencil_laplacian(order, h, None, 0)
    assert n == 1 + 3 * order
    buf = (StencilTerm * n)()
    assert lib().sb_stencil_laplacian(order, h, buf, n) == n
    got = [(t.source, tuple(t.offset), t.weight) for t in buf]
    want = so.laplacian(order, spacing)
    assert [(s, o) for s, o, _ in got] == [(s, o) for s, o, _ in want]
    assert [w.hex() for _, _, w in got] == [w.hex() for _, _, w in want]
    op = sb.StencilOp.laplacian(order, spacing, np.float64)
    assert [w.hex() for _, _, w in op.terms] == [w.hex() for _, _, w in want]
    # the weights sum to (about) zero: a Laplacian of a constant vanishes
    assert abs(math.fsum(w for _, _, w in got)) <= 1e-12 * max(abs(w) for _, _, w in got)


@pytest.mark.parametrize("order,spacing", [(3, (1, 1, 1)), (10, (1, 1, 1)), (0, (1, 1, 1)), (2, (0, 1, 1)), (2, (1, -1, 1)), (2, (1, 1, float("inf")))])
def test_laplacian_rejects(order, spacing):
    assert lib().sb_stencil_laplacian(order, (C.c_double * 3)(*spacing), None, 0) == -1
    with pytest.raises(sb.StencilError):
        sb.StencilOp.laplacian(order, spacing, np.float32)


# ------------------------------------------------------------------------------------------ sb_stencil_check
def radii():
    asym = sb.Radius.constant(1)
    asym.set_dir((1, 0, 0), 2)
    asym.set_dir((0, -1, 0), 3)
    asym.set_dir((0, 0, 1), 0)
    left = sb.Radius.constant(0)
    left.set_dir((-1, 0, 0), 4)
    return {
        "f1": sb.Radius.face_edge_corner(1, 0, 0),
        "f1e1": sb.Radius.face_edge_corner(1, 1, 0),
        "fec1": sb.Radius.face_edge_corner(1, 1, 1),
        "f2e1": sb.Radius.face_edge_corner(2, 1, 0),
        "c4": sb.Radius.constant(4),
        "asym": asym,
        "left4": left,
    }


@pytest.mark.parametrize("rname", list(radii()))
def test_check_every_single_offset(rname):
    """Every offset in [-5, 5]^3, as a one-term op and behind a centre term, accepted exactly when the rule says so."""
    r = radii()[rname]
    r27 = list(r.c27())
    accepted = 0
    for o in itertools.product(range(-5, 6), repeat=3):
        for terms in ([(0, o, 1.0)], [(0, (0, 0, 0), -1.0), (0, o, 0.5)]):
            want = so.check_rule(terms, r27)
            rc = lib().sb_stencil_check(c_terms(terms), len(terms), r.c27())
            assert rc == (0 if want else -1), (o, rc)
            if not want:
                assert "term" in lib().sb_last_error().decode()
            accepted += want
    assert accepted > 0


@pytest.mark.parametrize("op,rname,ok", [
    ("lap2", "f1", True), ("lap2", "f1e1", True), ("box27", "f1", False), ("box27", "f1e1", False), ("box27", "fec1", True),
    ("lap4", "f1", False), ("lap4", "f2e1", True), ("lap8", "f2e1", False), ("lap8", "c4", True),
    ("upwind", "left4", True), ("upwind", "asym", False), ("lap2", "asym", False), ("lap2", "left4", False),
])  # fmt: skip
def test_check_ops(op, rname, ok):
    terms = {"lap2": so.laplacian(2, (1, 1, 1)), "lap4": so.laplacian(4, (1, 1, 1)), "lap8": so.laplacian(8, (1, 1, 1)), "box27": box27(),
             "upwind": [(0, (0, 0, 0), 1.5), (0, (-1, 0, 0), -2.0), (0, (-2, 0, 0), 0.5), (0, (-4, 0, 0), 0.25)]}[op]
    r = radii()[rname]
    assert so.check_rule(terms, list(r.c27())) == ok
    rc = lib().sb_stencil_check(c_terms(terms), len(terms), r.c27())
    assert rc == (0 if ok else -1), lib().sb_last_error()
    o = sb.StencilOp(terms, np.float64)
    if ok:
        o.check(r)
    else:
        with pytest.raises(sb.StencilError, match="term"):
            o.check(r)


@pytest.mark.parametrize("terms,what", [
    ([(0, (5, 0, 0), 1.0)], "reaches beyond"),
    ([(0, (0, 0, -5), 1.0)], "reaches beyond"),
    ([], "1 to 64 terms"),
    ([(0, (0, 0, 0), 1.0)] * 65, "1 to 64 terms"),
    ([(0, (0, 0, 0), 1.0), (1, (1, 0, 0), 1.0)], "aux term"),
    ([(2, (0, 0, 0), 1.0)], "source"),
])  # fmt: skip
def test_check_limits(terms, what):
    rc = lib().sb_stencil_check(c_terms(terms), len(terms), sb.Radius.constant(4).c27())
    assert rc == -1
    assert what in lib().sb_last_error().decode()
    with pytest.raises(sb.StencilError, match=what):
        sb.StencilOp(terms, np.float32)


def test_op_basics():
    assert lib().sb_stencil_check(c_terms([(0, (0, 0, 0), 1.0)] * 64), 64, sb.Radius.constant(0).c27()) == 0
    with pytest.raises(sb.StencilError, match="float32 or float64"):
        sb.StencilOp([(0, (0, 0, 0), 1.0)], np.int32)
    a = sb.StencilOp.laplacian(2, (1, 1, 1), np.float32)
    assert a == sb.StencilOp(so.laplacian(2, (1, 1, 1)), np.float32) and a != sb.StencilOp(so.laplacian(2, (1, 1, 1)), np.float64)
    assert a.reach() == 1 and not a.has_aux


# ------------------------------------------------------------------------------------------ sb_stencil_plan_create errors
ES = 8


def plan_args(**kw):
    """Valid arguments for an F64 7-point plan over a 10^3 box inside a 12^3 allocation at fake (never dereferenced)
    addresses; kw overrides."""
    a = dict(dtype=2, terms=so.laplacian(2, (1, 1, 1)), dst=Pitched(0x100000, 12 * ES, 12), src=Pitched(0x200000, 12 * ES, 12),
             aux=Pitched(None, 0, 0), acc=(-1, -1, -1), zsize=12, boxes=[((0, 0, 0), (10, 10, 10))])
    a.update(kw)
    return a


def create(a):
    h = C.c_void_p()
    nb = len(a["boxes"])
    lo = (C.c_int64 * (3 * max(1, nb)))(*[v for b in a["boxes"] for v in b[0]])
    hi = (C.c_int64 * (3 * max(1, nb)))(*[v for b in a["boxes"] for v in b[1]])
    rc = lib().sb_stencil_plan_create(C.byref(h), 0, a["dtype"], c_terms(a["terms"]), len(a["terms"]), a["dst"], a["src"], a["aux"],
                                      (C.c_int64 * 3)(*a["acc"]), a["zsize"], nb, lo, hi)
    if rc == 0:
        lib().sb_stencil_plan_destroy(h)
    return rc, lib().sb_last_error().decode()


@pytest.mark.parametrize("kw,what", [
    (dict(dtype=0), "dtype"),
    (dict(dtype=3), "dtype"),
    (dict(terms=[]), "1 to 64 terms"),
    (dict(terms=[(0, (0, 0, 0), 1.0)] * 65), "1 to 64 terms"),
    (dict(terms=[(0, (0, 5, 0), 1.0)]), "reaches beyond"),
    (dict(terms=[(1, (0, 0, 1), 1.0)]), "aux term"),
    (dict(terms=[(0, (0, 0, 0), 1.0), (1, (0, 0, 0), 1.0)]), "aux is NULL"),
    (dict(dst=Pitched(0x200000, 12 * ES, 12)), "dst must not be src"),
    (dict(dst=Pitched(None, 12 * ES, 12)), "must not be NULL"),
    (dict(dst=Pitched(0x100000, 13 * ES, 12)), "another pitch"),
    (dict(dst=Pitched(0x100000, 12 * ES, 11)), "another pitch"),
    (dict(terms=[(1, (0, 0, 0), 1.0)], aux=Pitched(0x300000, 12 * ES, 13)), "another pitch"),
    (dict(src=Pitched(0x200004, 12 * ES, 12)), "multiples"),
    (dict(src=Pitched(0x200000, 12 * ES + 4, 12), dst=Pitched(0x100000, 12 * ES + 4, 12)), "multiples"),
    (dict(zsize=0), "zsize"),
    (dict(boxes=[((0, 0, 0), (10, -1, 10))]), "lo > hi"),
    (dict(boxes=[((-1, 0, 0), (10, 10, 10))]), "outside the allocation"),
    (dict(boxes=[((0, 0, 0), (11, 10, 10))]), "outside the allocation"),
    (dict(boxes=[((0, -1, 0), (10, 10, 10))]), "outside the allocation"),
    (dict(boxes=[((0, 0, 0), (10, 11, 10))]), "outside the allocation"),
    (dict(boxes=[((0, 0, -1), (10, 10, 10))]), "outside the allocation"),
    (dict(boxes=[((0, 0, 0), (10, 10, 11))]), "outside the allocation"),
    (dict(zsize=11), "outside the allocation"),
    (dict(terms=[(0, (0, 0, 0), 1.0), (0, (0, 0, 2), 1.0)]), "outside the allocation"),
    (dict(terms=[(0, (-2, 0, 0), 1.0)]), "outside the allocation"),
])  # fmt: skip
def test_plan_create_errors(kw, what):
    rc, msg = create(plan_args(**kw))
    assert rc == -1 and what in msg, msg


def test_plan_create_null_handle():
    assert lib().sb_stencil_plan_create(None, 0, 2, c_terms([(0, (0, 0, 0), 1.0)]), 1, Pitched(0x100000, 96, 12), Pitched(0x200000, 96, 12),
                                        Pitched(None, 0, 0), (C.c_int64 * 3)(0, 0, 0), 12, 0, None, None) == -1


# ------------------------------------------------------------------------------------------ C layout
@pytest.mark.skipif(shutil.which("cc") is None and shutil.which("gcc") is None, reason="no C compiler")
def test_term_layout_matches_ctypes(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "stencil_b200.h"\n'
        "int main(void) { printf(\"%zu %zu %zu %zu %d %d\\n\", offsetof(sb_stencil_term, source), offsetof(sb_stencil_term, offset),"
        " offsetof(sb_stencil_term, weight), sizeof(sb_stencil_term), SB_STENCIL_MAX_TERMS, SB_STENCIL_MAX_REACH); return 0; }\n"
    )
    exe = tmp_path / "probe"
    cc = shutil.which("cc") or shutil.which("gcc")
    subprocess.check_call([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert got == [StencilTerm.source.offset, StencilTerm.offset.offset, StencilTerm.weight.offset, C.sizeof(StencilTerm), 64, 4]
    from stencil_b200 import _lib

    assert (_lib.STENCIL_MAX_TERMS, _lib.STENCIL_MAX_REACH) == (64, 4)
