"""Host-side checks of coloured application and the relaxation table (no GPU): the snapshot oracle of
tests/colour_oracle.py against a literal in-place Gauss-Seidel loop, sb_stencil_relax term for term and its errors,
sb_stencil_ccheck against the rule, every new sb_stencil_cplan_create error, the new symbols, and the contraction rates
of red-black Gauss-Seidel and SOR against theory on a periodic Helmholtz problem."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

import colour_oracle as co
import stencil_b200 as sb
import stencil_op_oracle as so
import vstencil_oracle as vo
from stencil_b200._lib import Pitched, StencilTerm, StencilVTerm, lib
from test_vstencil_host import radii


def c_terms(terms):
    arr = (StencilTerm * max(1, len(terms)))()
    for k, (s, o, w) in enumerate(terms):
        arr[k] = StencilTerm(s, (C.c_int32 * 3)(*o), w)
    return arr


def c_vterms(terms):
    arr = (StencilVTerm * max(1, len(terms)))()
    for k, t in enumerate(terms):
        s, o, w, f, c = vo.split(t)
        arr[k] = StencilVTerm(s, (C.c_int32 * 3)(*o), f, (C.c_int32 * 3)(*c), w)
    return arr


def box27(seed=3):
    rng = np.random.default_rng(seed)
    return [(0, (x, y, z), float(rng.uniform(-1, 1))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]


# ------------------------------------------------------------------------------------------ the oracle
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("m,op", [(2, "lap2"), (2, "upwind3"), (8, "box27"), (1, "lap2")])
def test_snapshot_rule_is_gauss_seidel(dtype, m, op):
    """Within a colour, evaluating every cell on the snapshot before the pass gives the bits of the literal loop that
    updates u in place in lexicographic order (m = 1 is the exception: there the loop reads updated cells, so only the
    coloured m > 1 cases are compared; m = 1 checks that the loop then differs, so the comparison has teeth)."""
    A = {"lap2": co.helmholtz(1.0, 0.06), "box27": [t for t in box27() if any(t[1])] + [(0, (0, 0, 0), 30.0)],
         "upwind3": [(0, (0, 0, 0), 2.0), (0, (-1, 0, 0), -0.5), (0, (0, -3, 0), 0.25), (0, (1, 1, 1), 0.125)]}[op]
    terms = co.relax(A, 1.3)
    rng = np.random.default_rng(3)
    rm, rp = so.reach(terms)
    ext = (6, 5, 7)
    lo = tuple(rm[a] for a in range(3))
    shape = tuple(ext[a] + rm[a] + rp[a] for a in range(3))[::-1]
    origin = (-3, 5, 2)
    u0 = rng.uniform(-1, 1, shape).astype(dtype)
    f = rng.uniform(-1, 1, shape).astype(dtype)
    for c in range(m):
        a, b = u0.copy(), u0.copy()
        co.apply_box(terms, a, f, [], a, lo, ext, origin, m, c)
        co.sweep_loop(terms, b, f, lo, ext, origin, m, c)
        if m == 1:
            assert not np.array_equal(a, b)
        else:
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), c
            keep = ~co.box_mask(shape, lo, ext, origin, m, c)
            assert np.array_equal(a[keep].view(np.uint8), u0[keep].view(np.uint8))


def test_colours():
    col = co.colours((2, 2, 3), (1, 0, 0), 8)
    assert col[0, 0].tolist() == [1, 0, 1] and col[1, 1].tolist() == [7, 6, 7]
    assert co.colours((1, 1, 4), (-1, 0, 0), 2)[0, 0].tolist() == [1, 0, 1, 0]


# ------------------------------------------------------------------------------------------ sb_stencil_relax
def relax_c(A, omega):
    n = len(A)
    need = lib().sb_stencil_relax(c_terms(A), n, omega, None, 0)
    if need < 0:
        return None, lib().sb_last_error().decode()
    out = (StencilTerm * need)()
    assert lib().sb_stencil_relax(c_terms(A), n, omega, out, need) == need
    return [(t.source, tuple(t.offset), t.weight) for t in out], ""


@pytest.mark.parametrize("A", [co.helmholtz(0.37, 2.5), so.laplacian(2, (0.3, 0.7, 1.1)), box27(), so.laplacian(8, (1, 1, 1))[::-1]])
@pytest.mark.parametrize("omega", [1.0, 1.75, 0.4, 2.5, -0.3])
def test_relax_table(A, omega):
    got, _ = relax_c(A, omega)
    want = co.relax(A, omega)
    assert len(got) == len(A) + 1
    assert [(s, o) for s, o, _ in got] == [(s, o) for s, o, _ in want]
    assert [np.float64(w).view(np.uint64) for _, _, w in got] == [np.float64(w).view(np.uint64) for _, _, w in want]
    # Python: the same table
    op = sb.StencilOp(A, np.float64).relax(omega)
    assert op.terms == tuple(want)


def test_relax_weights_by_hand():
    A = [(0, (1, 0, 0), -1.0), (0, (0, 0, 0), 4.0), (0, (0, -1, 0), -3.0)]
    got, _ = relax_c(A, 1.5)
    assert got == [(0, (0, 0, 0), -0.5), (0, (1, 0, 0), 0.375), (0, (0, -1, 0), 1.125), (1, (0, 0, 0), 0.375)]


@pytest.mark.parametrize("A,omega,what", [
    ([(0, (1, 0, 0), 1.0)], 1.0, "no term at offset (0, 0, 0)"),
    ([(0, (0, 0, 0), 1.0), (0, (1, 0, 0), 1.0), (0, (0, 0, 0), 2.0)], 1.0, "terms 0 and 2 are both at offset (0, 0, 0)"),
    ([(0, (0, 0, 0), 0.0), (0, (1, 0, 0), 1.0)], 1.0, "centre weight of A is 0"),
    ([(0, (0, 0, 0), 6.0), (1, (0, 0, 0), 1.0)], 1.0, "term 1 reads aux"),
    ([(0, (0, 0, 0), 6.0)], math.nan, "omega = nan must be finite"),
    ([(0, (0, 0, 0), 6.0)], math.inf, "must be finite"),
    ([(0, (0, 0, 0), 6.0), (0, (5, 0, 0), 1.0)], 1.0, "reaches beyond 4"),
    ([], 1.0, "1 to 64 terms"),
    ([(0, (0, 0, 0), 6.0)] + [(0, (1, 0, 0), 1.0)] * 63, 1.0, "at most 64"),
])  # fmt: skip
def test_relax_errors(A, omega, what):
    got, msg = relax_c(A, omega)
    assert got is None and what in msg, msg
    if A and "1 to 64" not in what and "beyond" not in what:
        with pytest.raises(sb.StencilError, match="relax"):
            sb.StencilOp(A, np.float64).relax(omega)


def test_relax_refuses_coefficient_ops():
    with pytest.raises(sb.StencilError, match="constant coefficients"):
        sb.StencilOp.div_grad((1, 1, 1), np.float64).relax(1.0)


def test_relax_bad_output_buffer():
    A = co.helmholtz(1.0, 0.5)
    assert lib().sb_stencil_relax(c_terms(A), len(A), 1.0, None, 3) == -1
    assert "bad output buffer" in lib().sb_last_error().decode()


# ------------------------------------------------------------------------------------------ sb_stencil_ccheck
@pytest.mark.parametrize("rname", ["f1", "fec1", "c4", "asym"])
@pytest.mark.parametrize("m", [1, 2, 8])
def test_ccheck_every_offset(rname, m):
    """Every src offset in [-5, 5]^3 behind a centre term, and every coefficient offset in [-2, 2]^3 on a centre term and
    on an odd src offset: accepted exactly when the reach rule and the colour condition say so."""
    r = radii()[rname]
    r27 = list(r.c27())
    cases = [[(0, (0, 0, 0), -1.0), (0, o, 1.0)] for o in itertools.product(range(-5, 6), repeat=3)]
    for c in itertools.product(range(-2, 3), repeat=3):
        cases += [[(0, (0, 0, 0), 1.0, 3, c)], [(0, (0, 0, 0), 1.0), (0, (1, 0, 0), 1.0, 0, c)], [(1, (0, 0, 0), 1.0, 1, c)]]
    seen = {True: 0, False: 0}
    colour_refused = 0
    for terms in cases:
        want = vo.check_rule(terms, r27) and co.colour_ok(terms, m)
        rc = lib().sb_stencil_ccheck(c_vterms(terms), len(terms), r.c27(), m)
        assert rc == (0 if want else -1), (terms, m, rc)
        seen[want] += 1
        if vo.check_rule(terms, r27) and not want:
            colour_refused += 1
            msg = lib().sb_last_error().decode()
            assert "term 1: offset" in msg and f"own colour under {m} colours" in msg, msg
        if m == 1:
            assert rc == lib().sb_stencil_vcheck(c_vterms(terms), len(terms), r.c27())
    assert seen[True] > 0 and seen[False] > 0
    # within reach 1 every non-zero offset has an odd component, so m = 8 refuses an offset only where a radius reaches 2;
    # face radius 1 reaches only the six face offsets, which m = 2 accepts as well
    assert (colour_refused > 0) == (rname in {1: (), 2: ("fec1", "c4", "asym"), 8: ("c4", "asym")}[m])


@pytest.mark.parametrize("m", [0, 3, 4, -2, 16])
def test_ccheck_bad_colouring(m):
    terms = [(0, (0, 0, 0), 1.0)]
    assert lib().sb_stencil_ccheck(c_vterms(terms), 1, sb.Radius.constant(1).c27(), m) == -1
    assert f"ncolours {m}: a colouring has 1, 2 or 8 colours" in lib().sb_last_error().decode()


def test_python_check_colours():
    lap2, lap4 = sb.StencilOp.laplacian(2, (1, 1, 1), np.float64), sb.StencilOp.laplacian(4, (1, 1, 1), np.float64)
    r = sb.Radius.constant(2)
    lap2.check(r, colours=2)
    lap2.check(r, colours=8)
    lap4.check(r)
    with pytest.raises(sb.StencilError, match=r"term 7: offset \(-2, 0, 0\) reads a cell of its own colour under 2"):
        lap4.check(r, colours=2)
    with pytest.raises(sb.StencilError, match="own colour under 8"):
        sb.StencilOp([(0, (0, 0, 0), 1.0), (0, (2, 0, 2), 1.0)], np.float64).check(r, colours=8)
    with pytest.raises(sb.StencilError, match="own colour under 2"):
        sb.StencilOp(box27(), np.float64).check(r, colours=2)
    sb.StencilOp(box27(), np.float64).check(r, colours=8)


# ------------------------------------------------------------------------------------------ sb_stencil_cplan_create errors
ES = 8
DST, SRC, AUX = Pitched(0x100000, 12 * ES, 12), Pitched(0x200000, 12 * ES, 12), Pitched(0x300000, 12 * ES, 12)
K = Pitched(0x400000, 12 * ES, 12)


def cplan(terms, m, c, dst=DST, src=SRC, aux=AUX, coefs=()):
    h = C.c_void_p()
    lo, hi = (C.c_int64 * 3)(0, 0, 0), (C.c_int64 * 3)(10, 10, 10)
    carr = (Pitched * max(1, len(coefs)))(*coefs)
    rc = lib().sb_stencil_cplan_create(C.byref(h), 0, 2, c_vterms(terms), len(terms), dst, src, aux, carr, len(coefs), m, c,
                                       (C.c_int64 * 3)(-1, -1, -1), 12, 1, lo, hi)
    if rc == 0:
        lib().sb_stencil_plan_destroy(h)
    return rc, lib().sb_last_error().decode()


SOR = co.relax(co.helmholtz(1.0, 0.06), 1.5)


@pytest.mark.parametrize("terms,m,c,kw,what", [
    (SOR, 3, 0, {}, "ncolours 3: a colouring has 1, 2 or 8 colours"),
    (SOR, 0, 0, {}, "ncolours 0"),
    (SOR, 2, 2, {}, "colour 2: 0 .. 1 under 2 colours"),
    (SOR, 8, -1, {}, "colour -1: 0 .. 7 under 8 colours"),
    (SOR, 1, 1, {}, "colour 1: 0 .. 0 under 1 colours"),
    (SOR + [(0, (2, 0, 0), 0.5)], 2, 0, {}, "term 8: offset (2, 0, 0) reads a cell of its own colour under 2 colours"),
    (SOR + [(0, (1, 1, 0), 0.5)], 2, 1, {}, "term 8: offset (1, 1, 0) reads a cell of its own colour under 2 colours"),
    (SOR + [(0, (0, 2, -2), 0.5)], 8, 5, {}, "term 8: offset (0, 2, -2) reads a cell of its own colour under 8 colours"),
    (SOR, 1, 0, dict(dst=SRC), "dst must not be src (dst may be aux)"),
    (SOR + [(0, (1, 0, 0), 0.5, 0, (0, 0, 0))], 2, 0, dict(dst=SRC, coefs=(SRC,)), "coefficient field 0 is dst"),
    ([(0, (0, 0, 0), 1.0, 0, (1, 0, 0))], 2, 0, dict(coefs=(DST,)), "coefficient field 0 is dst"),
])  # fmt: skip
def test_cplan_create_errors(terms, m, c, kw, what):
    rc, msg = cplan(terms, m, c, **kw)
    assert rc == -1 and what in msg, msg


def test_vplan_keeps_its_message():
    """sb_stencil_vplan_create is the coloured planner with m = 1: dst == src keeps its message word for word."""
    h = C.c_void_p()
    lo, hi = (C.c_int64 * 3)(0, 0, 0), (C.c_int64 * 3)(10, 10, 10)
    rc = lib().sb_stencil_vplan_create(C.byref(h), 0, 2, c_vterms(SOR), len(SOR), SRC, SRC, AUX, None, 0, (C.c_int64 * 3)(-1, -1, -1), 12, 1,
                                       lo, hi)
    assert rc == -1 and lib().sb_last_error().decode() == "dst must not be src (dst may be aux)"


def test_in_place_passes_validation():
    """dst == src (and aux == dst) with m > 1 gets past every check; on a machine without a device the planner then stops
    at the device, never at validation."""
    for m, c in ((2, 0), (2, 1), (8, 7)):
        rc, msg = cplan(SOR, m, c, dst=SRC, aux=SRC)
        assert rc == 0 or "CUDA device" in msg, msg


def test_new_symbols():
    for name in ("sb_stencil_ccheck", "sb_stencil_relax", "sb_stencil_cplan_create"):
        assert hasattr(lib(), name)


# ------------------------------------------------------------------------------------------ convergence against theory
def helmholtz_problem(shape=(8, 6, 10), sigma=0.06, seed=9):
    """Periodic FP64 -lap u + sigma u = f, h = 1, even sizes (a 2-cyclic red-black graph), sigma h^2 = 0.06."""
    A = co.helmholtz(1.0, sigma)
    rho_j = 6.0 / (6.0 + sigma)
    f = np.random.default_rng(seed).uniform(-1, 1, shape)
    return A, rho_j, f


def sweep(terms, u, f, m=2):
    for c in range(m):
        u = co.apply_periodic(terms, u, f, [], u, m, c)
    return u


def rates(terms, f, sweeps):
    u = np.zeros_like(f)
    norms = []
    for _ in range(sweeps):
        nu = sweep(terms, u, f)
        norms.append(float(np.linalg.norm(nu - u)))
        u = nu
    return [norms[k + 1] / norms[k] for k in range(len(norms) - 1)]


def test_red_black_gauss_seidel_rate():
    """Red-black Gauss-Seidel contracts by rho_J^2 per sweep (asymptotically), within 1 %."""
    A, rho_j, f = helmholtz_problem()
    r = rates(co.relax(A, 1.0), f, 400)
    assert abs(r[-1] / rho_j**2 - 1) < 0.01, (r[-1], rho_j**2)


def test_sor_optimal_rate():
    """Red-black SOR at omega_opt = 2 / (1 + sqrt(1 - rho_J^2)) contracts by omega_opt - 1 over late sweeps, within 10 %
    (the eigenvalue is defective at omega_opt, which slows the approach)."""
    A, rho_j, f = helmholtz_problem()
    w = 2.0 / (1.0 + math.sqrt(1.0 - rho_j**2))
    r = rates(co.relax(A, w), f, 120)
    late = math.exp(np.mean(np.log(r[80:])))
    assert abs(late / (w - 1) - 1) < 0.10, (late, w - 1)
    # and far faster than Gauss-Seidel
    assert late < 0.8 * rho_j**2
