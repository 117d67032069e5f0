"""Host-side checks of multigrid-preconditioned CG (no GPU): the three per-cell Krylov modes of tests/krylov_oracle.py
against per-cell loops in both dtypes (XPBY with T(s) = +-0 never reading p), the exact dot rule against
fractions.Fraction sums on adversarial data, every error of sb_krylov_plan_create and the new symbols, the BC mapping of
the Krylov vectors, and the convergence of the numpy flexible CG preconditioned by one V(2,2) cycle: smooth kappa on
ODD(0) walls and periodic Helmholtz, a 10^3 jump in kappa on ODD(0) walls (where the V-cycle alone stalls), and the
breakdown of an indefinite op."""
import ctypes as C
import math
import os
import re
from fractions import Fraction

import numpy as np
import pytest

import krylov_oracle as ko
import vmg_oracle as vm
import stencil_b200 as sb
from stencil_b200 import _lib
from stencil_b200._lib import I3, Pitched, lib
from stencil_b200.krylov import homogeneous_bc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------- the per-cell modes
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s", [0.75, -1.0 / 3, 1e-30, 0.0, -0.0, 1e300])
def test_modes_are_the_loops(dtype, s):
    rng = np.random.default_rng(3)
    x, p, r, q, z = (rng.uniform(-2, 2, (3, 4, 5)).astype(dtype) for _ in range(5))
    with np.errstate(over="ignore", invalid="ignore"):
        assert np.array_equal(ko.xpby(p, z, s), ko.xpby_loop(p, z, s), equal_nan=True)
        for a, b in zip(ko.update(x, p, r, q, s), ko.update_loop(x, p, r, q, s)):
            assert np.array_equal(a, b, equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_xpby_zero_does_not_read_p(dtype):
    z = np.arange(12, dtype=dtype).reshape(2, 2, 3) - 5
    p = np.full_like(z, np.nan)
    for s in (0.0, -0.0, 1e-60):  # 1e-60 rounds to +0 in float32 only
        got = ko.xpby(p, z, s)
        if dtype(s) == 0:
            assert np.array_equal(got, z) and not np.isnan(got).any()
        else:
            assert np.isnan(got).all()


def test_update_rounds_each_operation():
    """No FMA contraction: r - T(s) q rounds the product first."""
    x = np.array([1.0], np.float32)
    p = np.array([1.0 + 2.0**-23], np.float32)
    r = np.array([1.0], np.float32)
    q = np.array([1.0 + 2.0**-23], np.float32)
    s = 1.0 - 2.0**-23
    xn, rn = ko.update(x, p, r, q, s)
    prod = np.float32(np.float32(s) * q[0])
    assert rn[0] == np.float32(r[0] - prod) and xn[0] == np.float32(x[0] + prod)


# ------------------------------------------------------------------------------------------- the dot rule
def fraction_dot(a, b):
    return float(sum((Fraction(float(u)) * Fraction(float(v)) if a.dtype == np.float32 else Fraction(float(u) * float(v)) for u, v in zip(a.ravel(), b.ravel())),
                     Fraction(0)))


ADVERSARIAL = {
    "cancellation": (np.array([1e16, 1.0, -1e16, 3.0, 1e-16, -4.0]), np.array([1.0, 1.0, 1.0, 1.0, 1.0, 1.0])),
    "tiny": (np.array([5e-324, 2.5e-308, -1e-300, 7e-320]), np.array([1.0, 0.5, 1e-10, 3.0])),
    "huge": (np.array([1e300, 1e300, -1e300, 1e150]), np.array([1e7, 1e8, 1.1e8, 1e150])),
    "mixed": (np.array([1e308, 1.0, -1e308, 2.0**-1074, 2.0**-1022]), np.array([1.0, 2.0**-60, 1.0, 1.0, 3.0])),
}


@pytest.mark.parametrize("name", sorted(ADVERSARIAL))
def test_dot_rule_is_exact(name):
    a, b = ADVERSARIAL[name]
    assert ko.dot(a, b) == fraction_dot(a, b) == ko.exact_dot(a, b)


def test_dot_rule_float32_products_are_exact():
    rng = np.random.default_rng(5)
    a = (rng.uniform(-1, 1, 64) * 10.0 ** rng.integers(-30, 30, 64)).astype(np.float32)
    b = (rng.uniform(-1, 1, 64) * 10.0 ** rng.integers(-30, 30, 64)).astype(np.float32)
    assert ko.dot(a, b) == float(sum((Fraction(float(u)) * Fraction(float(v)) for u, v in zip(a, b)), Fraction(0)))


@pytest.mark.parametrize("terms,want", [
    ([1.0, float("nan"), 2.0], "nan"),
    ([float("inf"), 1.0], math.inf),
    ([-float("inf"), 1.0], -math.inf),
    ([float("inf"), -float("inf")], "nan"),
    ([1.7e308, 1.7e308], math.inf),
    ([-1.7e308, -1.7e308], -math.inf),
    ([1.7e308, 1.7e308, -1.7e308], 1.7e308),
    ([0.0, -0.0], 0.0),
    ([-0.0, -0.0], 0.0),
])
def test_exact_sum_special_values(terms, want):
    got = ko.exact_sum(terms)
    if want == "nan":
        assert math.isnan(got)
    else:
        assert got == want and math.copysign(1.0, got) == math.copysign(1.0, want)


def test_ordered_min_max():
    assert ko.ordered_min_max([0.0, -0.0]) == (-0.0, 0.0)
    assert math.copysign(1, ko.ordered_min_max([0.0, -0.0])[0]) == -1
    assert ko.ordered_min_max([]) == (math.inf, -math.inf)
    mn, mx = ko.ordered_min_max([1.0, float("nan"), -3.0])
    assert math.isnan(mn) and math.isnan(mx)


# ------------------------------------------------------------------------------------------- the C ABI
ROW, ROWS = 24 * 8, 20
BUFS = [(0x100000 + 0x100000 * k, ROW, ROWS) for k in range(4)]


def kcreate(mode=_lib.KRYLOV_UPDATE, dtype=2, bufs=BUFS, nbuf=None, origin=(-1, -1, -1), lo=(0, 0, 0), hi=(8, 8, 8)):
    arr = (Pitched * 4)(*[Pitched(*b) for b in (list(bufs) + [(None, 0, 0)] * 4)[:4]])
    h = C.c_void_p()
    rc = lib().sb_krylov_plan_create(C.byref(h), 0, mode, dtype, arr, len(bufs) if nbuf is None else nbuf, I3(*origin), I3(*lo), I3(*hi))
    err = lib().sb_last_error().decode()
    if rc == 0:  # on a machine with a GPU a valid plan is built (it never launches on these addresses)
        lib().sb_krylov_plan_destroy(h)
    return rc, err


@pytest.mark.parametrize("kw,msg", [
    (dict(mode=3), "unknown krylov mode 3"),
    (dict(mode=-1), "unknown krylov mode -1"),
    (dict(dtype=0), "dtype 0 must be SB_DTYPE_F32 or SB_DTYPE_F64"),
    (dict(nbuf=3), "SB_KRYLOV_UPDATE takes 4 buffers, not 3"),
    (dict(mode=_lib.KRYLOV_XPBY, nbuf=3), "SB_KRYLOV_XPBY takes 2 buffers, not 3"),
    (dict(mode=_lib.KRYLOV_DOT, nbuf=4), "SB_KRYLOV_DOT takes 2 or 3 buffers, not 4"),
    (dict(mode=_lib.KRYLOV_DOT, nbuf=1), "SB_KRYLOV_DOT takes 2 or 3 buffers, not 1"),
    (dict(bufs=BUFS[:2] + [(None, ROW, ROWS)] + BUFS[3:]), "buffer r is NULL"),
    (dict(bufs=BUFS[:3] + [(0x500000, ROW + 8, ROWS)]), "the buffers have different pitches or row counts"),
    (dict(bufs=BUFS[:3] + [(0x500000, ROW, ROWS + 1)]), "the buffers have different pitches or row counts"),
    (dict(bufs=BUFS[:1] + [(0x200004, ROW, ROWS)] + BUFS[2:]), "buffer p: pointer and pitch must be multiples of the 8-byte element"),
    (dict(bufs=[(b[0], ROW + 4, ROWS) for b in BUFS]), "buffer x: pointer and pitch must be multiples of the 8-byte element"),
    (dict(lo=(0, 3, 0), hi=(8, 2, 8)), "lo > hi on axis 1"),
    (dict(hi=(24, 8, 8)), "box outside the allocation"),
    (dict(hi=(8, 20, 8)), "box outside the allocation"),
    (dict(lo=(-2, 0, 0)), "buffer x: region outside the allocation on axis 0"),
    (dict(bufs=BUFS[:2] + [BUFS[0]] + BUFS[3:]), "x, p, r and q must be four distinct buffers (r is x)"),
    (dict(bufs=BUFS[:3] + [BUFS[1]]), "x, p, r and q must be four distinct buffers (q is p)"),
    (dict(mode=_lib.KRYLOV_XPBY, bufs=[BUFS[0], BUFS[0]]), "SB_KRYLOV_XPBY: p must not be z"),
    (dict(bufs=[BUFS[0], (0x100008, ROW, ROWS)] + BUFS[2:]), "SB_KRYLOV_UPDATE: buffers x and p overlap over the box"),
    (dict(bufs=BUFS[:3] + [(0x300000 + 7 * ROW * ROWS, ROW, ROWS)]), "SB_KRYLOV_UPDATE: buffers r and q overlap over the box"),
    (dict(mode=_lib.KRYLOV_XPBY, bufs=[BUFS[0], (0x100000 + ROW * ROWS, ROW, ROWS)]), "SB_KRYLOV_XPBY: buffers p and z overlap over the box"),
    (dict(bufs=[(0x10000000000 * (k + 1), (2**27 + 8) * 8, ROWS) for k in range(4)], hi=(2**27 + 1, 8, 8)), "rows of more than 2^27 cells"),
    (dict(bufs=[(0x10000000000 * (k + 1), ROW, 2**16 + 2) for k in range(4)], hi=(8, 2**16, 2**15 + 1)), "more than 2^31 rows"),
])
def test_plan_errors(kw, msg):
    rc, err = kcreate(**kw)
    assert rc == -1, (rc, err)
    assert msg in err, err


def test_plan_create_needs_its_arguments():
    """NULL out, lo or hi (through an untyped binding of the same symbol, so NULL can be passed)."""
    raw = C.CDLL(_lib.LIB_PATH).sb_krylov_plan_create
    raw.restype = C.c_int
    raw.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    arr = (Pitched * 4)(*[Pitched(*b) for b in BUFS])
    h, acc, lo, hi = C.c_void_p(), I3(-1, -1, -1), I3(0, 0, 0), I3(8, 8, 8)
    for args in ((None, lo, hi), (C.byref(h), None, hi), (C.byref(h), lo, None)):
        out, l, u = args
        assert raw(out, 0, _lib.KRYLOV_UPDATE, 2, C.cast(arr, C.c_void_p), 4, C.cast(acc, C.c_void_p), l if l is None else C.cast(l, C.c_void_p),
                   u if u is None else C.cast(u, C.c_void_p)) == -1
        assert "needs an output handle, acc_origin, lo and hi" in lib().sb_last_error().decode()


@pytest.mark.parametrize("bufs", [[BUFS[0], BUFS[0], BUFS[0]], [BUFS[0], (0x100008, ROW, ROWS)]])
def test_dot_sources_may_alias(bufs):
    """<r, r> is one source passed twice, and DOT sources may overlap: every check passes, so creation succeeds on a
    machine with a GPU and fails only for want of a device without one."""
    n = C.c_int(0)
    has_gpu = lib().sb_device_count(C.byref(n)) == 0 and n.value > 0
    rc, err = kcreate(mode=_lib.KRYLOV_DOT, bufs=bufs)
    assert rc == (0 if has_gpu else -3), (rc, err)


def test_new_symbols():
    with open(os.path.join(ROOT, "include", "stencil_b200.h")) as f:
        header = f.read()
    for name in ("sb_krylov_plan_create", "sb_krylov_plan_launch", "sb_krylov_plan_bytes", "sb_krylov_plan_destroy"):
        assert re.search(rf"\b{name}\(", header), name
        assert name in _lib._SIGS
        assert getattr(lib(), name) is not None
    assert (_lib.KRYLOV_DOT, _lib.KRYLOV_XPBY, _lib.KRYLOV_UPDATE) == (0, 1, 2)
    assert lib().sb_krylov_plan_bytes(None) == 0 and lib().sb_krylov_plan_destroy(None) == 0
    assert callable(sb.DistributedDomain.dot) and callable(sb.PCG.solve)


# ------------------------------------------------------------------------------------------- BCs
def test_homogeneous_bc():
    assert homogeneous_bc(sb.BC.ODD(0.75)) == sb.BC.ODD(0.0)
    assert homogeneous_bc(sb.BC.EVEN()) == sb.BC.EVEN()
    assert homogeneous_bc(sb.BC.VALUE(2.5)) == sb.BC.VALUE(0.0)
    with pytest.raises(sb.StencilError, match="x needs a boundary condition"):
        homogeneous_bc(sb.BC.NONE())
    assert ko.homogeneous({0: ("odd", 0.5), 1: ("even", 0.0), 2: ("value", 3.0)}) == {0: ("odd", 0.0), 1: ("even", 0.0), 2: ("value", 0.0)}


class _FakeDomain(sb.DistributedDomain):
    """A DistributedDomain that passes PCG's realized check without a GPU: the constructor's refusals come first."""

    def __init__(self, walls_x, walls_p, walls_z):
        super().__init__(8, 8, 8)
        self.x, self.f, self.r, self.z, self.p, self.q = (self.add_data(np.float64, n) for n in "xfrzpq")
        self.set_boundary(sb.Boundary.FIXED)
        for h, w in ((self.x, walls_x), (self.p, walls_p), (self.z, walls_z)):
            for fc, bc in w.items():
                self.set_boundary_condition(h, sb.FACES[fc], bc)
        self.partition_ = object()
        self._plans = [[None]]


ODD_X = {fc: sb.BC.ODD(0.5) for fc in range(6)}
ODD_0 = {fc: sb.BC.ODD(0.0) for fc in range(6)}


@pytest.mark.parametrize("walls_p,walls_z,msg", [
    ({**ODD_0, 3: sb.BC.EVEN()}, ODD_0, "p needs ODD(0.0) on face (0, 1, 0), the homogeneous counterpart of x's ODD(0.5), not EVEN"),
    (ODD_0, {**ODD_0, 5: sb.BC.ODD(0.5)}, "z needs ODD(0.0) on face (0, 0, 1)"),
    ({fc: bc for fc, bc in ODD_0.items() if fc != 0}, ODD_0, "p needs ODD(0.0) on face (-1, 0, 0)"),
])
def test_pcg_refuses_mismatched_bcs(walls_p, walls_z, msg):
    d = _FakeDomain(ODD_X, walls_p, walls_z)
    with pytest.raises(sb.StencilError) as e:
        sb.PCG(d, d.x, d.f, d.r, d.z, d.p, d.q, lambda l: None)
    assert msg.replace("ODD(0.0)", repr(sb.BC.ODD(0.0))).replace("ODD(0.5)", repr(sb.BC.ODD(0.5))).replace("EVEN", repr(sb.BC.EVEN())) in str(e.value), str(e.value)


def test_pcg_refuses_before_building():
    d = _FakeDomain(ODD_X, ODD_0, ODD_0)
    A = lambda l: None  # noqa: E731
    with pytest.raises(sb.StencilError, match="precond must be 'multigrid' or None"):
        sb.PCG(d, d.x, d.f, d.r, d.z, d.p, d.q, A, precond="jacobi")
    with pytest.raises(sb.StencilError, match="pass z=None"):
        sb.PCG(d, d.x, d.f, d.r, d.z, d.p, d.q, A, precond=None)
    with pytest.raises(sb.StencilError, match="must be 6 different quantities"):
        sb.PCG(d, d.x, d.f, d.r, d.p, d.p, d.q, A)
    with pytest.raises(sb.StencilError, match="q must be a DataHandle of dd"):
        sb.PCG(d, d.x, d.f, d.r, d.z, d.p, 3, A)
    with pytest.raises(sb.StencilError, match="x needs a boundary condition"):
        sb.PCG(_FakeDomain({}, ODD_0, ODD_0), d.x, d.f, d.r, d.z, d.p, d.q, A)
    with pytest.raises(sb.StencilError, match="op_at\\(0\\) must be a StencilOp"):
        sb.PCG(d, d.x, d.f, d.r, d.z, d.p, d.q, A)
    with pytest.raises(sb.StencilError, match="realized DistributedDomain"):
        sb.PCG(sb.DistributedDomain(8, 8, 8), d.x, d.f, d.r, d.z, d.p, d.q, A)


# ------------------------------------------------------------------------------------------- the numpy solver
def problem(n, kappa, kind, precond=True, sign=1.0):
    """The problems of test_vmultigrid_host.cycle_factors under PCG: ODD(0) walls with even kappa walls, or periodic
    with a cell field sigma = 10; f uniform in [-1, 1) (seed 0), x = 0."""
    h = 1.0 / n
    levels = int(np.log2(n)) - 1
    if kind == "odd":
        periodic, walls, kinds, sig = (False,) * 3, {f: ("odd", 0.0) for f in range(6)}, ("x", "y", "z"), False
        cw = [{f: ("even", 0.0) for f in range(6)} for _ in range(3)]
    else:
        periodic, walls, kinds, sig = (True,) * 3, {}, ("x", "y", "z", "cell"), True
        cw = [{} for _ in range(4)]

    def A_at(l):
        return [t[:2] + (sign * t[2],) + tuple(t[3:]) for t in vm.helmholtz_div_grad(h * 2**l, sigma_field=sig)]

    lv = vm.hierarchy((n, n, n), levels, A_at, np.float64, periodic, ko.homogeneous(walls), cw)
    for a, b in zip(lv[0].k, vm.kappa_faces(n, h, kappa, np.float64)):
        a[...] = b
    if sig:
        lv[0].k[3][...] = 10.0
    vm.update_coefficients(lv, kinds)
    s = ko.PCG(lv, walls, precond=precond)
    s.I(s.f)[...] = np.random.default_rng(0).uniform(-1, 1, (n, n, n))
    return s


@pytest.mark.parametrize("kind", ["odd", "periodic"])
def test_pcg_smooth_kappa_factor(kind):
    """Smooth kappa: every factor of the residual norm is <= 0.08 (measured 0.021 - 0.057) at 16^3, 32^3 and 64^3, and
    the true residual agrees with the recursive one."""
    for n in (16, 32, 64):
        s = problem(n, "smooth", kind)
        hist = s.solve(0.0, 8 if n == 64 else 12)
        f = [hist[k + 1] / hist[k] for k in range(len(hist) - 1)]
        assert max(f) <= 0.08, (n, f)
        assert abs(s.residual_norm() - hist[-1]) <= 1e-12 * hist[0], (n, s.residual_norm(), hist[-1])


@pytest.mark.parametrize("n", [32, 64])
def test_pcg_jump_kappa_converges(n):
    """A 10^3 jump: <= 1e-3 of the start after 12 iterations and <= 1e-8 within 30 (measured 25 and 23 iterations)."""
    s = problem(n, "jump", "odd")
    hist = s.solve(0.0, 30)
    assert hist[12] <= 1e-3 * hist[0], hist
    assert min(hist) <= 1e-8 * hist[0], [h / hist[0] for h in hist]
    assert s.breakdown is None


def test_vcycle_alone_stalls_on_the_jump():
    """The same 32^3 problem under vm.vcycle alone is still above 1e-3 of the start after 30 cycles (measured 2.2e-3)."""
    s = problem(32, "jump", "odd")
    L = s.L
    L.u[...] = 0
    L.f[...] = s.f
    r0 = L.residual_norm()
    for _ in range(30):
        vm.vcycle(s.lv)
    assert L.residual_norm() > 1e-3 * r0


@pytest.mark.parametrize("precond", [True, False])
def test_indefinite_op_breaks_down_at_once(precond):
    s = problem(16, "smooth", "odd", precond=precond, sign=-1.0)
    hist = s.solve(1e-8, 10)
    assert s.breakdown == 0 and len(hist) == 1
