"""Host-side checks of multigrid-preconditioned BiCGStab (no GPU): the BICG_P and UPDATE-with-c rules of
tests/bicgstab_oracle.py against per-cell loops in both dtypes (with a case FMA contraction would change), <c, r'>
against fractions.Fraction sums with special values, every new error of sb_krylov_plan_create and the new symbols, the
solver's constructor refusals, and the convergence of the numpy BiCGStab preconditioned by one V(2,2) cycle: a 10^3
jump in kappa with convection on ODD(0) walls (where the V-cycle alone stalls), smooth kappa with convection,
constant-coefficient convection-diffusion, periodic with sigma, and the symmetric jump; the true residual against the
recursive one, each breakdown branch, the stop at the half step, and a cycle on another pair."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import bicgstab_oracle as bo
import krylov_oracle as ko
import mg_oracle as mo
import vmg_oracle as vm
import stencil_b200 as sb
from stencil_b200 import _lib
from stencil_b200._lib import I3, Pitched, lib
from test_krylov_host import BUFS, ROW, ROWS, _FakeDomain, fraction_dot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = (4.0, 2.4, 1.2)  # the convection velocity


def same(a, b):
    return a == b or (math.isnan(a) and math.isnan(b))


# ------------------------------------------------------------------------------------------- the per-cell rules
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("beta,omega", [(0.75, -1.0 / 3), (1e-30, 3.5), (0.0, 0.25), (-0.0, -0.0), (1e300, 1e-300), (2.0, 0.0)])
def test_bicg_p_is_the_loop(dtype, beta, omega):
    rng = np.random.default_rng(3)
    p, r, v = (rng.uniform(-2, 2, (3, 4, 5)).astype(dtype) for _ in range(3))
    with np.errstate(over="ignore", invalid="ignore", under="ignore"):
        assert np.array_equal(bo.bicg_p(p, r, v, beta, omega), bo.bicg_p_loop(p, r, v, beta, omega), equal_nan=True)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("s", [0.75, -1.0 / 3, 1e-30, 0.0, 1e300])
def test_update_c_is_the_loop(dtype, s):
    rng = np.random.default_rng(4)
    x, p, r, q, c = (rng.uniform(-2, 2, (3, 4, 5)).astype(dtype) for _ in range(5))
    with np.errstate(over="ignore", invalid="ignore"):
        xn, rn, rr, cr = bo.update_c(x, p, r, q, c, s)
        xl, rl = ko.update_loop(x, p, r, q, s)
        assert np.array_equal(xn, xl, equal_nan=True) and np.array_equal(rn, rl, equal_nan=True)
        assert same(rr, ko.exact_dot(rl, rl)) and same(cr, ko.exact_dot(c, rl))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_bicg_p_rounds_each_operation(dtype):
    """No FMA contraction: with omega = v = 1 + eps and p = 1 + 2 eps, T(omega) v rounds to p and p - T(omega) v is 0,
    where a fused multiply-subtract would give -eps^2."""
    from fractions import Fraction

    T, eps = dtype, float(np.finfo(dtype).eps)
    p, r, v = (np.array([a], T) for a in (1.0 + 2 * eps, 0.0, 1.0 + eps))
    omega, beta = 1.0 + eps, 3.0
    got = bo.bicg_p(p, r, v, beta, omega)[0]
    assert got == 0 and got == bo.bicg_p_loop(p, r, v, beta, omega)[0]
    fused = Fraction(float(p[0])) - Fraction(float(T(omega))) * Fraction(float(v[0]))
    assert fused == -Fraction(eps) ** 2 and T(float(3 * fused)) != 0


@pytest.mark.parametrize("name", ["cancellation", "tiny", "huge", "mixed"])
def test_update_c_dot_is_exact(name):
    from test_krylov_host import ADVERSARIAL

    c, r = ADVERSARIAL[name]
    z = np.zeros_like(r)
    _, rn, _, cr = bo.update_c(z, z, r, z, c, 0.0)
    assert np.array_equal(rn, r) and cr == fraction_dot(c, r)


@pytest.mark.parametrize("c,r,want", [
    ([1.0, np.nan, 2.0], [1.0, 1.0, 1.0], "nan"),
    ([np.inf, 1.0], [1.0, 2.0], math.inf),
    ([np.inf, 1.0], [-1.0, 2.0], -math.inf),
    ([np.inf, np.inf], [1.0, -1.0], "nan"),
    ([1e300, 1e300], [1e10, 1e10], math.inf),
    ([0.0, -0.0], [-1.0, 1.0], 0.0),
])
def test_update_c_dot_special_values(c, r, want):
    c, r = np.array(c), np.array(r)
    got = bo.dot(c, r)
    assert same(got, ko.exact_dot(c, r))
    if want == "nan":
        assert math.isnan(got)
    else:
        assert got == want and math.copysign(1.0, got) == math.copysign(1.0, want)


# ------------------------------------------------------------------------------------------- the C ABI
C5 = BUFS + [(0x600000, ROW, ROWS)]  # UPDATE x, p, r, q, c
P3 = BUFS[:3]  # BICG_P p, r, v


def kcreate(mode=_lib.KRYLOV_UPDATE, dtype=2, bufs=BUFS, nbuf=None, origin=(-1, -1, -1), lo=(0, 0, 0), hi=(8, 8, 8)):
    """test_krylov_host.kcreate with room for six buffers."""
    arr = (Pitched * 6)(*[Pitched(*b) for b in (list(bufs) + [(None, 0, 0)] * 6)[:6]])
    h = C.c_void_p()
    rc = lib().sb_krylov_plan_create(C.byref(h), 0, mode, dtype, arr, len(bufs) if nbuf is None else nbuf, I3(*origin), I3(*lo), I3(*hi))
    err = lib().sb_last_error().decode()
    if rc == 0:
        lib().sb_krylov_plan_destroy(h)
    return rc, err


@pytest.mark.parametrize("kw,msg", [
    (dict(nbuf=6, bufs=C5), "SB_KRYLOV_UPDATE takes 4 buffers, not 6 (5 with c)"),
    (dict(nbuf=3), "SB_KRYLOV_UPDATE takes 4 buffers, not 3 (5 with c)"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=P3, nbuf=2), "SB_KRYLOV_BICG_P takes 3 buffers, not 2"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=BUFS), "SB_KRYLOV_BICG_P takes 3 buffers, not 4"),
    (dict(mode=3, bufs=P3), "unknown krylov mode 3"),
    (dict(mode=5, bufs=P3), "unknown krylov mode 5"),
    (dict(bufs=BUFS + [(None, ROW, ROWS)]), "buffer c is NULL"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], (None, ROW, ROWS), P3[2]]), "buffer r is NULL"),
    (dict(bufs=BUFS + [(0x600000, ROW + 8, ROWS)]), "the buffers have different pitches or row counts"),
    (dict(bufs=BUFS + [(0x600004, ROW, ROWS)]), "buffer c: pointer and pitch must be multiples of the 8-byte element"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], P3[1], (0x300004, ROW, ROWS)]), "buffer v: pointer and pitch must be multiples"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=P3, hi=(24, 8, 8)), "box outside the allocation"),
    (dict(bufs=BUFS + [BUFS[0]]), "SB_KRYLOV_UPDATE: c must not be x or r (c is x)"),
    (dict(bufs=BUFS + [BUFS[2]]), "SB_KRYLOV_UPDATE: c must not be x or r (c is r)"),
    (dict(bufs=BUFS[:2] + [BUFS[0], BUFS[3], C5[4]]), "x, p, r and q must be four distinct buffers (r is x)"),
    (dict(bufs=BUFS + [(0x100008, ROW, ROWS)]), "SB_KRYLOV_UPDATE: buffers x and c overlap over the box"),
    (dict(bufs=BUFS + [(0x300000 + 7 * ROW * ROWS, ROW, ROWS)]), "SB_KRYLOV_UPDATE: buffers r and c overlap over the box"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], P3[0], P3[2]]), "SB_KRYLOV_BICG_P: p must not be r or v (r is p)"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], P3[1], P3[0]]), "SB_KRYLOV_BICG_P: p must not be r or v (v is p)"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], (0x100008, ROW, ROWS), P3[2]]), "SB_KRYLOV_BICG_P: buffers p and r overlap over the box"),
    (dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], P3[1], (0x100000 + ROW * ROWS, ROW, ROWS)]), "SB_KRYLOV_BICG_P: buffers p and v overlap"),
])
def test_new_plan_errors(kw, msg):
    rc, err = kcreate(**kw)
    assert rc == -1, (rc, err)
    assert msg in err, err


def _has_gpu():
    n = C.c_int(0)
    return lib().sb_device_count(C.byref(n)) == 0 and n.value > 0


@pytest.mark.parametrize("kw", [
    dict(bufs=BUFS + [BUFS[1]]),  # c is p
    dict(bufs=BUFS + [BUFS[3]]),  # c is q
    dict(bufs=BUFS + [(0x200008, ROW, ROWS)]),  # c overlaps p
    dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], P3[1], P3[1]]),  # v is r
    dict(mode=_lib.KRYLOV_BICG_P, bufs=[P3[0], P3[1], (0x200008, ROW, ROWS)]),  # v overlaps r
])
def test_read_only_buffers_may_alias(kw):
    """Every check passes: creation succeeds on a machine with a GPU and fails only for want of a device without one."""
    rc, err = kcreate(**kw)
    assert rc == (0 if _has_gpu() else -3), (rc, err)


def test_existing_update_still_refuses_overlapping_p_and_q():
    """The four-buffer UPDATE keeps its rule: p and q, though both only read, must not overlap."""
    rc, err = kcreate(bufs=BUFS[:3] + [(0x200008, ROW, ROWS)])
    assert rc == -1 and "SB_KRYLOV_UPDATE: buffers p and q overlap over the box" in err, err


def test_new_symbols():
    with open(os.path.join(ROOT, "include", "stencil_b200.h")) as f:
        header = f.read()
    assert re.search(r"\bsb_krylov_plan_launch2\(", header)
    assert re.search(r"SB_KRYLOV_BICG_P = 4\b", header)
    assert "sb_krylov_plan_launch2" in _lib._SIGS and lib().sb_krylov_plan_launch2 is not None
    assert lib().sb_krylov_plan_launch2(None, 1.0, 2.0, None, None) == -1 and "null plan" in lib().sb_last_error().decode()
    assert _lib.KRYLOV_BICG_P == 4
    assert callable(sb.BiCGStab.solve) and callable(sb.Multigrid.cycle)


# ------------------------------------------------------------------------------------------- the constructor
class _FakeDomain9(_FakeDomain):
    def __init__(self, walls_x, walls_ph, walls_sh):
        super().__init__(walls_x, {}, {})
        self.r0, self.v, self.ph, self.sh, self.t = (self.add_data(np.float64, n) for n in ("r0", "v", "ph", "sh", "t"))
        for h, w in ((self.ph, walls_ph), (self.sh, walls_sh)):
            for fc, bc in w.items():
                self.set_boundary_condition(h, sb.FACES[fc], bc)

    def args(self, **kw):
        a = dict(x=self.x, f=self.f, r=self.r, r0=self.r0, p=self.p, v=self.v, phat=self.ph, shat=self.sh, t=self.t)
        a.update(kw)
        return a


ODD_X = {fc: sb.BC.ODD(0.5) for fc in range(6)}
ODD_0 = {fc: sb.BC.ODD(0.0) for fc in range(6)}


def test_bicgstab_refuses_before_building():
    d = _FakeDomain9(ODD_X, ODD_0, ODD_0)
    A = lambda l: None  # noqa: E731
    with pytest.raises(sb.StencilError, match="must be 9 different quantities"):
        sb.BiCGStab(d, **d.args(t=d.p), op_at=A)
    with pytest.raises(sb.StencilError, match="r0 must be a DataHandle of dd"):
        sb.BiCGStab(d, **d.args(r0=3), op_at=A)
    with pytest.raises(sb.StencilError, match=r"shat needs .* on face \(0, 0, 1\), the homogeneous counterpart of x's"):
        e = _FakeDomain9(ODD_X, ODD_0, {**ODD_0, 5: sb.BC.ODD(0.5)})
        sb.BiCGStab(e, **e.args(), op_at=A)
    with pytest.raises(sb.StencilError, match=r"phat needs .* on face \(-1, 0, 0\)"):
        e = _FakeDomain9(ODD_X, {fc: bc for fc, bc in ODD_0.items() if fc != 0}, ODD_0)
        sb.BiCGStab(e, **e.args(), op_at=A)
    with pytest.raises(sb.StencilError, match="x needs a boundary condition"):
        e = _FakeDomain9({}, ODD_0, ODD_0)
        sb.BiCGStab(e, **e.args(), op_at=A)
    with pytest.raises(sb.StencilError, match="op_at\\(0\\) must be a StencilOp"):
        sb.BiCGStab(d, **d.args(), op_at=A)
    with pytest.raises(sb.StencilError, match="realized DistributedDomain"):
        sb.BiCGStab(sb.DistributedDomain(8, 8, 8), **d.args(), op_at=A)


# ------------------------------------------------------------------------------------------- the numpy solver
def conv(h, b=B):
    """Central differences of b . grad u on spacing h."""
    t = []
    for a in range(3):
        e = [0, 0, 0]
        e[a] = 1
        t.append((0, tuple(e), b[a] / (2 * h)))
        t.append((0, tuple(-v for v in e), -b[a] / (2 * h)))
    return t


def problem(n, kappa, kind, b=B):
    """-div(kappa grad u) + b . grad u (+ sigma u) as test_krylov_host.problem sets it up: ODD(0) walls with EVEN kappa
    walls, or periodic with a cell field sigma = 10; kappa None: constant-coefficient -lap u + b . grad u through
    mg_oracle; f uniform in [-1, 1) (seed 0), x = 0."""
    h = 1.0 / n
    levels = int(np.log2(n)) - 1
    if kind == "odd":
        periodic, walls, kinds, sig = (False,) * 3, {f: ("odd", 0.0) for f in range(6)}, ("x", "y", "z"), False
        cw = [{f: ("even", 0.0) for f in range(6)} for _ in range(3)]
    else:
        periodic, walls, kinds, sig = (True,) * 3, {}, ("x", "y", "z", "cell"), True
        cw = [{} for _ in range(4)]
    if kappa is None:
        def A_at(l):
            hl = h * 2**l
            return [(0, (0, 0, 0), 6.0 / hl**2)] + [(0, o, -1.0 / hl**2) for o in ((1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1))] + conv(hl, b)

        lv = mo.hierarchy((n, n, n), levels, A_at, np.float64, periodic, ko.homogeneous(walls))
    else:
        lv = vm.hierarchy((n, n, n), levels, lambda l: vm.helmholtz_div_grad(h * 2**l, sigma_field=sig) + conv(h * 2**l, b), np.float64, periodic,
                          ko.homogeneous(walls), cw)
        for a, k in zip(lv[0].k, vm.kappa_faces(n, h, kappa, np.float64)):
            a[...] = k
        if sig:
            lv[0].k[3][...] = 10.0
        vm.update_coefficients(lv, kinds)
    s = bo.BiCGStab(lv, walls)
    s.I(s.f)[...] = np.random.default_rng(0).uniform(-1, 1, (n, n, n))
    return s


@pytest.mark.parametrize("n", [32, 64])
def test_jump_convection_converges(n):
    """The 10^3 jump with convection: <= 1e-8 of the start within 10 iterations (measured 9.1e-11 after 7 at 32^3),
    and the true residual agrees with the recursive one."""
    s = problem(n, "jump", "odd")
    hist = s.solve(1e-8, 10)
    assert s.breakdown is None
    assert hist[-1] <= 1e-8 * hist[0] and len(hist) - 1 <= 10, [v / hist[0] for v in hist]
    assert abs(s.residual_norm() - hist[-1]) <= 1e-10 * hist[0]


def test_vcycle_alone_stalls_on_jump_convection():
    """The same 32^3 problem under vm.vcycle alone is still above 1e-3 of the start after 24 cycles (measured 5.8e-3)."""
    s = problem(32, "jump", "odd")
    L = s.L
    L.u[...] = 0
    L.f[...] = s.f
    r0 = L.residual_norm()
    for _ in range(24):
        vm.vcycle(s.lv)
    assert L.residual_norm() > 1e-3 * r0


@pytest.mark.parametrize("kappa,kind", [("smooth", "odd"), (None, "odd"), ("smooth", "periodic"), ("jump-symmetric", "odd")])
def test_other_problems_converge(kappa, kind):
    """Smooth kappa with convection, constant-coefficient convection-diffusion (mg_oracle), periodic with sigma and
    convection, and the symmetric jump (b = 0): <= 1e-8 within 10 iterations at 32^3, true residual as recursive."""
    b = (0.0, 0.0, 0.0) if kappa == "jump-symmetric" else B
    s = problem(32, "jump" if kappa == "jump-symmetric" else kappa, kind, b)
    hist = s.solve(1e-8, 10)
    assert s.breakdown is None
    assert hist[-1] <= 1e-8 * hist[0], [v / hist[0] for v in hist]
    assert abs(s.residual_norm() - hist[-1]) <= 1e-10 * hist[0]


class _Zero:
    """Replaces the solver's apply_A by zeros from call `after` on (0: v = 0; 1: t = 0)."""

    def __init__(self, s, after):
        self.s, self.after, self.calls, self.apply = s, after, 0, s.apply_A

    def __call__(self, p):
        self.calls += 1
        return np.zeros_like(p) if self.calls > self.after else self.apply(p)


def test_breakdown_sigma():
    s = problem(16, "smooth", "odd")
    s.apply_A = _Zero(s, 0)
    hist = s.solve(1e-8, 10)
    assert s.breakdown == 0 and len(hist) == 1 and not s.I(s.x).any()


def test_breakdown_omega():
    """t = 0: <t, t> = 0 after the half step, which is kept and reported."""
    s = problem(16, "smooth", "odd")
    s.apply_A = _Zero(s, 1)
    hist = s.solve(1e-8, 10)
    assert s.breakdown == 0 and len(hist) == 2 and hist[1] == math.sqrt(ko.dot(s.I(s.r), s.I(s.r)))


def test_breakdown_rho(monkeypatch):
    """A new <r0, r> of exactly zero after the first iteration (the full step's dot replaced by zero)."""
    s = problem(16, "smooth", "odd")
    orig = bo.update_c

    def update_c_zero_rho(*a):
        xn, rn, rr, _ = orig(*a)
        return xn, rn, rr, 0.0

    monkeypatch.setattr(bo, "update_c", update_c_zero_rho)
    hist = s.solve(1e-8, 10)
    assert s.breakdown == 0 and len(hist) == 2 and hist[1] > 1e-8 * hist[0]


def test_stop_at_the_half_step():
    """When sqrt(<s, s>) reaches the target the solve stops with the half-step iterate, whose residual is the last
    entry: a large rtol is met after the half step of iteration 0."""
    s = problem(16, "smooth", "odd")
    ref = problem(16, "smooth", "odd")
    h_ref = [math.sqrt(ref.start())]
    ref.iterate(0, 0.0, h_ref)  # the full iteration; its half-step residual:
    I = ref.I
    xn, rn = ko.update(np.zeros_like(I(ref.x)), I(ref.ph), I(ref.f), I(ref.v), ref.alpha)
    ss = math.sqrt(ko.dot(rn, rn))
    rtol = ss / math.sqrt(ko.dot(I(ref.f), I(ref.f)))
    hist = s.solve(rtol, 10)
    assert s.breakdown is None and len(hist) == 2 and hist[1] == ss
    assert np.array_equal(s.I(s.x), xn) and s.residual_norm() <= 1e-12 + 1.01 * ss


def test_cycle_pair_is_a_hierarchy_on_the_pair():
    """A cycle of lv on another pair (u2, f2) is the bits of a cycle of a hierarchy built with (u2, f2) on level 0."""
    n, h = 16, 1.0 / 16
    A_at = lambda l: vm.helmholtz_div_grad(h * 2**l) + conv(h * 2**l)  # noqa: E731
    walls = {f: ("odd", 0.0) for f in range(6)}
    cw = [{f: ("even", 0.0) for f in range(6)} for _ in range(3)]
    lvs = []
    for _ in range(2):
        lv = vm.hierarchy((n,) * 3, 3, A_at, np.float64, (False,) * 3, walls, cw)
        for a, k in zip(lv[0].k, vm.kappa_faces(n, h, "jump", np.float64)):
            a[...] = k
        vm.update_coefficients(lv, ("x", "y", "z"))
        lvs.append(lv)
    rng = np.random.default_rng(9)
    lvs[0][0].f[...] = rng.uniform(-1, 1, lvs[0][0].f.shape)  # the constructor pair holds other data
    u2 = rng.uniform(-1, 1, lvs[0][0].u.shape)
    f2 = rng.uniform(-1, 1, lvs[0][0].f.shape)
    keep_u, keep_f = lvs[0][0].u.copy(), lvs[0][0].f.copy()
    lvs[1][0].u[...], lvs[1][0].f[...] = u2, f2
    bo.cycle_pair(lvs[0], u2, f2, vm.vcycle)
    vm.vcycle(lvs[1])
    assert np.array_equal(u2, lvs[1][0].u)
    assert np.array_equal(lvs[0][0].u, keep_u) and np.array_equal(lvs[0][0].f, keep_f)
