"""Linear stencil systems without a GPU: the numpy rule of tests/system_oracle.py against a per-cell loop and against the
single-output rules, the grad / div / curl tables of the C library term for term, exact discrete identities, the reach
check, every plan-creation error (all raised before the library touches a device), the sb_stencil_sys_term layout and
the new symbols."""
import ctypes as C
import itertools

import numpy as np
import pytest

import stencil_b200 as sb
import stencil_op_oracle as so
import system_oracle as yo
import vstencil_oracle as vo
from stencil_b200._lib import I27, Pitched, StencilSysTerm, check, lib
from test_gpu_stencil_op import OPS as PLAIN_OPS
from test_gpu_system_op import SYSTEMS, as_system
from test_gpu_vstencil_op import OPS as VOPS

H = (0.5, 0.25, 0.5)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(SYSTEMS))
def test_oracle_matches_cell_loop(name, dtype):
    terms, nin, alias = SYSTEMS[name]
    rng = np.random.default_rng(1)
    shape = (9, 10, 11)
    lo, ext = (2, 2, 2), (6, 5, 4)
    a = [rng.uniform(-1, 1, shape).astype(dtype) for _ in range(nin)]
    b = [x.copy() for x in a]
    nout = yo.nout_of(terms)
    outs_a = [a[alias[j]] if j in alias else np.zeros(shape, dtype) for j in range(nout)]
    outs_b = [b[alias[j]] if j in alias else np.zeros(shape, dtype) for j in range(nout)]
    yo.apply_box(terms, a, outs_a, lo, ext)
    yo.apply_cell_loop(terms, b, outs_b, lo, ext)
    for x, y in zip(outs_a, outs_b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", [("plain", k) for k in PLAIN_OPS] + [("coef", k) for k in VOPS])
def test_single_output_ops_as_systems(op, dtype):
    """src = input 0, aux = input 1, coefficient field k = input 2 + k: the bits of the single-output rules."""
    kind, name = op
    terms = PLAIN_OPS[name] if kind == "plain" else VOPS[name]
    rng = np.random.default_rng(2)
    shape = (14, 15, 16)
    lo, ext = (4, 4, 4), (8, 7, 6)
    ins = [rng.uniform(-1, 1, shape).astype(dtype) for _ in range(6)]
    want = np.zeros(shape, dtype)
    if kind == "plain":
        so.apply_box(terms, ins[0], ins[1], want, lo, ext)
    else:
        vo.apply_box(terms, ins[0], ins[1], ins[2:], want, lo, ext)
    got = np.zeros(shape, dtype)
    yo.apply_box(as_system(terms), ins, [got], lo, ext)
    assert np.array_equal(got, want)


def c_table(fn, stagger, h):
    hh = (C.c_double * 3)(*h)
    n = check(fn(stagger, hh, None, 0))
    buf = (StencilSysTerm * n)()
    assert check(fn(stagger, hh, buf, n)) == n
    return [(t.output, t.input, tuple(t.offset), t.weight) + ((t.coef, tuple(t.coef_offset)) if t.coef >= 0 else ()) for t in buf]


@pytest.mark.parametrize("stagger", [-1, 0, 1])
@pytest.mark.parametrize("name", ["grad", "div", "curl"])
def test_tables(name, stagger):
    h = (0.7, 1.3, 0.9)
    got = c_table(getattr(lib(), f"sb_stencil_{name}"), stagger, h)
    assert got == getattr(yo, name)(stagger, h)
    assert len(got) == (12 if name == "curl" else 6)
    assert sb.StencilSystem.__dict__[name].__func__(stagger, h, np.float64).terms == tuple(getattr(yo, name)(stagger, h))
    # the forward difference along x of grad: (+e_x, 1/h) then (0, -1/h)
    if name == "grad" and stagger == 1:
        assert got[:2] == [(0, 0, (1, 0, 0), 1 / 0.7), (0, 0, (0, 0, 0), -1 / 0.7)]


@pytest.mark.parametrize("name", ["grad", "div", "curl"])
def test_table_errors(name):
    fn = getattr(lib(), f"sb_stencil_{name}")
    with pytest.raises(sb.StencilError, match="stagger 2"):
        check(fn(2, (C.c_double * 3)(1, 1, 1), None, 0))
    for bad in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(sb.StencilError, match="finite and > 0"):
            check(fn(1, (C.c_double * 3)(1, bad, 1), None, 0))
    assert check(fn(0, (C.c_double * 3)(1, 1, 1), None, 0)) in (6, 12)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("h", [0.5, 0.25])
@pytest.mark.parametrize("stagger", [-1, 0, 1])
def test_exact_identities(stagger, h, dtype):
    """Integer-valued fields (|u| < 2^16) and h = 0.5 or 0.25: every value is exact, so curl(grad u) and div(curl v) are 0."""
    rng = np.random.default_rng(3)
    sp = (h, h, 2 * h)
    u = rng.integers(-(2**16) + 1, 2**16, (12, 13, 14)).astype(dtype)
    g = yo.apply_periodic(yo.grad(stagger, sp), [u])
    for c in yo.apply_periodic(yo.curl(stagger, sp), g):
        assert not c.any()
    v = [rng.integers(-(2**16) + 1, 2**16, (12, 13, 14)).astype(dtype) for _ in range(3)]
    (d,) = yo.apply_periodic(yo.div(stagger, sp), yo.apply_periodic(yo.curl(stagger, sp), v))
    assert not d.any()


RADII = [sb.Radius.constant(1), sb.Radius.constant(2), sb.Radius.face_edge_corner(1, 0, 0), sb.Radius.face_edge_corner(3, 1, 0)]


@pytest.mark.parametrize("ri", range(len(RADII)))
def test_sys_check_reach(ri):
    r27 = RADII[ri].c27()
    for o in itertools.product(range(-5, 6), repeat=3):
        terms = [(0, 0, o, 1.0)]
        got = lib().sb_stencil_sys_check(sb.StencilSystem.c_terms(_Fake(terms)), 1, 1, 1, r27) == 0
        assert got == yo.check_rule(terms, 1, 1, list(r27)), o
    for c in itertools.product(range(-2, 3), repeat=3):
        terms = [(0, 0, (0, 0, 0), 1.0, 1, c)]
        got = lib().sb_stencil_sys_check(sb.StencilSystem.c_terms(_Fake(terms)), 1, 2, 1, r27) == 0
        assert got == yo.check_rule(terms, 2, 1, list(r27)), c


class _Fake:
    """A term list that c_terms can convert without the checks of StencilSystem's constructor."""

    def __init__(self, terms):
        self.terms = tuple(terms)


def test_sys_check_limits():
    r27 = I27(*([4] * 27))

    def rc(terms, nin=2, nout=2):
        return lib().sb_stencil_sys_check(sb.StencilSystem.c_terms(_Fake(terms)), len(terms), nin, nout, r27)

    assert rc([(0, 0, (0, 0, 0), 1.0), (1, 1, (4, -4, 4), 1.0, 0, (1, -1, 1))]) == 0
    cases = [
        ([(2, 0, (0, 0, 0), 1.0)], "output 2 must be 0 .. 1"),
        ([(0, 2, (0, 0, 0), 1.0)], "input 2 must be 0 .. 1"),
        ([(0, 0, (5, 0, 0), 1.0)], "reaches beyond 4 cells"),
        ([(0, 0, (0, 0, 0), 1.0, 2, (0, 0, 0))], "coefficient input 2 must be -1"),
        ([(0, 0, (0, 0, 0), 1.0, 1, (2, 0, 0))], "reaches beyond 1 cell"),
        ([(0, 0, (0, 0, 0), 1.0, -1, (1, 0, 0))], "without a coefficient field"),
    ]
    for terms, msg in cases:
        with pytest.raises(sb.StencilError, match=msg):
            check(rc(terms))
    with pytest.raises(sb.StencilError, match="1 to 8 inputs, not 9"):
        check(rc([(0, 0, (0, 0, 0), 1.0)], nin=9))
    with pytest.raises(sb.StencilError, match="1 to 4 outputs, not 5"):
        check(rc([(0, 0, (0, 0, 0), 1.0)], nout=5))
    with pytest.raises(sb.StencilError, match="1 to 128 terms, not 129"):
        check(rc([(0, 0, (0, 0, 0), 1.0)] * 129))


SH = (20, 20, 20)  # x, y, z of the fake allocations


def fake(k, pitch=SH[0] * 8, ysize=SH[1]):
    return Pitched(0x100000 * (k + 1), pitch, ysize)


def create(terms, outs, ins, nin=None, boxes=(((2, 2, 2), (10, 10, 10)),), dtype=2, zsize=SH[2]):
    arr = sb.StencilSystem.c_terms(_Fake(terms))
    nb = len(boxes)
    lo = (C.c_int64 * (3 * max(1, nb)))(*[v for b in boxes for v in b[0]])
    hi = (C.c_int64 * (3 * max(1, nb)))(*[v for b in boxes for v in b[1]])
    h = C.c_void_p()
    rc = lib().sb_stencil_sys_plan_create(C.byref(h), 0, dtype, arr, len(terms), (Pitched * max(1, len(outs)))(*outs), len(outs),
                                          (Pitched * max(1, len(ins)))(*ins), len(ins) if nin is None else nin, (C.c_int64 * 3)(0, 0, 0),
                                          zsize, nb, lo, hi)
    if rc == 0:
        lib().sb_stencil_plan_destroy(h)
    return rc


def test_plan_errors():
    one = [(0, 0, (1, 0, 0), 1.0)]
    cases = [
        (dict(terms=one, outs=[fake(9)], ins=[fake(0)], dtype=3), "dtype 3"),
        (dict(terms=[(1, 0, (0, 0, 0), 1.0)], outs=[fake(9), fake(8)], ins=[fake(0)]), "output 0 has no terms"),
        (dict(terms=one, outs=[Pitched(None, 160, 20)], ins=[fake(0)]), "output 0 is NULL"),
        (dict(terms=one, outs=[fake(9)], ins=[Pitched(None, 160, 20)]), "input 0 is read by a term, but it is NULL"),
        (dict(terms=[(0, 0, (0, 0, 0), 1.0), (1, 0, (0, 0, 0), 1.0)], outs=[fake(9), fake(9)], ins=[fake(0)]), "outputs 0 and 1 are the same"),
        (dict(terms=one, outs=[fake(0)], ins=[fake(0)]), "output 0 is input 0, which a term reads at a non-zero offset"),
        # the offset that forbids the alias may be another output's, and a coefficient read
        (dict(terms=[(0, 0, (0, 0, 0), 1.0), (1, 1, (0, 0, 0), 1.0, 0, (0, 1, 0))], outs=[fake(0), fake(8)], ins=[fake(0), fake(1)]),
         "output 0 is input 0"),
        (dict(terms=one, outs=[fake(9)], ins=[fake(0, pitch=168)]), "input 0 has another pitch or row count than output 0"),
        (dict(terms=one, outs=[fake(9)], ins=[fake(0, ysize=21)]), "input 0 has another pitch or row count than output 0"),
        (dict(terms=one, outs=[fake(9, pitch=164), fake(8, pitch=164)][:1], ins=[fake(0, pitch=164)]), "positive multiples of the 8-byte element"),
        (dict(terms=one, outs=[Pitched(0x100004, 160, 20)], ins=[fake(0)]), "positive multiples of the 8-byte element"),
        (dict(terms=one, outs=[fake(9)], ins=[fake(0)], zsize=0), "zsize >= 1"),
        (dict(terms=one, outs=[fake(9)], ins=[fake(0)], boxes=(((5, 2, 2), (4, 10, 10)),)), "lo > hi"),
        (dict(terms=one, outs=[fake(9)], ins=[fake(0)], boxes=(((2, 2, 2), (20, 10, 10)),)), r"box 0: input 0 is read at cells 2 \.\. 20 on axis x"),
        (dict(terms=[(0, 0, (0, 0, 0), 1.0, 1, (0, 0, -1))], outs=[fake(9)], ins=[fake(0), fake(1)], boxes=(((2, 2, 0), (10, 10, 10)),)),
         r"box 0: input 1 is read at cells -1 \.\. 9 on axis z"),
        (dict(terms=one, outs=[fake(9)], ins=[fake(0)], nin=0), "1 to 8 inputs, not 0"),
    ]
    for kw, msg in cases:
        with pytest.raises(sb.StencilError, match=msg):
            check(create(**kw))
    # an input no term reads may be NULL, an output may be an input read only at offset 0: no error before the device
    rc = create([(0, 1, (0, 0, 0), 1.0)], [fake(1)], [Pitched(None, 0, 0), fake(1)])
    assert rc == 0 or "device" in lib().sb_last_error().decode() or "CUDA" in lib().sb_last_error().decode()


def test_term_layout():
    assert C.sizeof(StencilSysTerm) == 48
    offs = {n: getattr(StencilSysTerm, n).offset for n, _ in StencilSysTerm._fields_}
    assert offs == {"output": 0, "input": 4, "offset": 8, "coef": 20, "coef_offset": 24, "weight": 40}


def test_symbols():
    for name in ("sb_stencil_sys_check", "sb_stencil_grad", "sb_stencil_div", "sb_stencil_curl", "sb_stencil_sys_plan_create"):
        assert hasattr(lib(), name)


def test_system_class():
    curl = sb.StencilSystem.curl(1, H, np.float64)
    assert (curl.nin, curl.nout) == (3, 3)
    e = sb.StencilSystem([(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)], np.float64, nin=6) + curl.scaled(0.5)
    assert (e.nin, e.nout, len(e.terms)) == (6, 3, 15)
    assert e.terms[3:] == tuple(yo.scaled(yo.curl(1, H), 0.5))
    s = sb.StencilSystem([(0, 0, (1, 0, 0), 1.0, 1, (0, 0, 1))], np.float32).shifted(2, 1)
    assert s.terms == ((1, 2, (1, 0, 0), 1.0, 3, (0, 0, 1)),) and (s.nin, s.nout) == (4, 2)
    assert s.moved_inputs() == {2, 3} and s.read_inputs() == {2, 3}
    assert sb.StencilSystem([(0, 0, (0, 0, 0), 1.0, -1, (0, 0, 0))], np.float64).terms == ((0, 0, (0, 0, 0), 1.0),)
    with pytest.raises(sb.StencilError, match="coefficient offset"):
        sb.StencilSystem([(0, 0, (0, 0, 0), 1.0, -1, (1, 0, 0))], np.float64)
    with pytest.raises(sb.StencilError, match="output 5 must be"):
        sb.StencilSystem([(5, 0, (0, 0, 0), 1.0)], np.float64, nout=2)
    with pytest.raises(sb.StencilError, match="float16"):
        sb.StencilSystem([(0, 0, (0, 0, 0), 1.0)], np.float16)
    with pytest.raises(sb.StencilError, match="cannot concatenate"):
        curl + sb.StencilSystem.curl(1, H, np.float32)
    assert curl == sb.StencilSystem.curl(1, H, np.float64) and hash(curl) == hash(sb.StencilSystem.curl(1, H, np.float64))
    with pytest.raises(sb.StencilError, match="face radius"):
        sb.StencilSystem([(0, 0, (2, 0, 0), 1.0)], np.float64).check(sb.Radius.constant(1))
