"""The numpy oracles' walled operators and solvers against an independently assembled matrix (CPU, DESIGN.md section
2.14).  The bit-for-bit GPU tests tie the CUDA kernels and the Python and C++ solvers to tests/mg_oracle.py,
vmg_oracle.py, krylov_oracle.py and bicgstab_oracle.py, but kernel and oracle restate the same rule; here the fine
operator of every case of test_gpu_multigrid.py, test_gpu_vmultigrid.py, test_gpu_krylov.py and test_gpu_bicgstab.py is
built at 16^3 as a dense float64 matrix M and wall vector g straight from its definition,

    A u = -sum_a [kappa_a(p + e_a) (u(p + e_a) - u(p)) - kappa_a(p) (u(p) - u(p - e_a))] / h^2
          + sigma u + sum_a b_a (u(p + e_a) - u(p - e_a)) / (2 h),

kappa_a(p) on the face between p - e_a and p (kappa_a at the high wall is the field's ghost cell n, from its own BC),
sigma a constant or a cell field, and the ghost cells behind a wall ODD(c): 2c - mirror, EVEN: mirror, VALUE(c): c
(periodic axes wrap); the 27-point op, which discretises no PDE, from its term list.  Nothing here goes through
stencil_op_oracle, vm.helmholtz_div_grad or fill_ghosts.  Then:
1. the oracle's residual f - A u (its ghost fill, then its op, in float64) equals f - (M u + g) cell by cell within a few
   ulps of the sum of the magnitudes of the terms (the two sum in different orders);
2. each case's own numpy solver in float64 (Multigrid, PCG or BiCGStab as its table says; PCG without a preconditioner
   for noprec; float32 cases as the same case in float64) reaches rtol 1e-10, its true residual ||f - (M x + g)|| is
   within 10 rtol ||f||, and x agrees with np.linalg.solve(M, f - g)."""
import numpy as np
import pytest

import bicgstab_oracle as bo
import krylov_oracle as ko
import mg_oracle as mo
import vmg_oracle as vm
from test_gpu_bicgstab import B, CASES as BICG_CASES, conv
from test_gpu_krylov import CASES as PCG_CASES, poisson
from test_gpu_multigrid import CASES as MG_CASES, helmholtz_at, twenty_seven_at
from test_gpu_vmultigrid import CASES as VMG_CASES, fields

N = 16
SIZE = (N, N, N)
LEVELS = 3  # 16^3 .. 4^3
RTOL = 1e-10
# the operator check: |difference| <= ULPS * eps * sum |terms| per cell; measured at most 3.0 eps (the 27-point op)
ULPS = 8
# x against np.linalg.solve(M, f - g): ||x - x*|| / ||x*||, measured at 16^3 once the solvers reach 1e-10: 1.0e-7 and
# 8.0e-8 on the periodic and EVEN-walled coefficient cases (cond(M) 1.5e4, sigma of order 1 against 1/h^2 = 1024), at
# most 2.5e-8 on the others, 3e-14 .. 5e-10 where cond(M) is about 100; the bound leaves a factor 10
SOLUTION_RTOL = 1e-6


# ----------------------------------------------------------------------------------------------- the definition
class Problem:
    """One fine operator as the matrix is assembled from it: spacing, walls of u, kappa and its walls, sigma, b, or the
    term list of an op that discretises no PDE."""

    def __init__(self, h, periodic, walls, kappa=None, kwalls=None, sigma=0.0, b=(0.0, 0.0, 0.0), terms=None):
        self.h, self.periodic, self.walls = h, periodic, dict(walls or {})
        self.kappa = kappa  # None (kappa = 1) or three [z, y, x] interior face fields
        self.kwalls = dict(kwalls or {})
        self.sigma, self.b, self.terms = sigma, tuple(b), terms


def cell(p):
    return (p[2] * N + p[1]) * N + p[0]


def ghost(kind, c):
    """(factor of the mirror value, constant) of the ghost cell behind a wall"""
    if kind == "odd":
        return -1.0, 2.0 * c
    if kind == "even":
        return 1.0, 0.0
    assert kind == "value"
    return 0.0, c


def add_u(M, g, P, q, w, pr):
    """row P gets w * u(q): q inside, wrapped on a periodic axis, or the ghost cell behind a wall (reach 1)"""
    q = list(q)
    out = [a for a in range(3) if not 0 <= q[a] < N]
    if pr.periodic:
        M[P, cell([v % N for v in q])] += w
        return
    assert len(out) <= 1, "a walled op reaches one axis out at a time"
    if not out:
        M[P, cell(q)] += w
        return
    a = out[0]
    face = 2 * a + (q[a] >= N)
    q[a] = 0 if q[a] < 0 else N - 1  # the mirror: the cell next to the wall
    fac, const = ghost(*pr.walls[face])
    M[P, cell(q)] += w * fac
    g[P] += w * const


def kappa_at(pr, a, p):
    """kappa_a at the face between p - e_a and p; p_a = N is the ghost cell of the high wall"""
    if pr.kappa is None:
        return 1.0
    k = pr.kappa[a]
    if p[a] < N:
        return float(k[p[2], p[1], p[0]])
    q = list(p)
    q[a] = 0 if pr.periodic else N - 1
    if pr.periodic:
        return float(k[q[2], q[1], q[0]])
    fac, const = ghost(*pr.kwalls[2 * a + 1])
    return fac * float(k[q[2], q[1], q[0]]) + const


def assemble(pr):
    """M, g with A u = M u + g for every u of the interior"""
    M, g = np.zeros((N**3, N**3)), np.zeros(N**3)
    ih2, ih = 1.0 / pr.h**2, 1.0 / (2.0 * pr.h)
    for z in range(N):
        for y in range(N):
            for x in range(N):
                p = (x, y, z)
                P = cell(p)
                if pr.terms is not None:
                    for _, o, w in pr.terms:
                        add_u(M, g, P, [p[i] + o[i] for i in range(3)], w, pr)
                    continue
                for a in range(3):
                    e = [int(i == a) for i in range(3)]
                    hi, lo = [p[i] + e[i] for i in range(3)], [p[i] - e[i] for i in range(3)]
                    kh, kl = kappa_at(pr, a, hi), kappa_at(pr, a, p)
                    add_u(M, g, P, hi, -kh * ih2 + pr.b[a] * ih, pr)
                    add_u(M, g, P, p, (kh + kl) * ih2, pr)
                    add_u(M, g, P, lo, -kl * ih2 - pr.b[a] * ih, pr)
                s = pr.sigma if np.isscalar(pr.sigma) else float(pr.sigma[z, y, x])
                if s:
                    M[P, P] += s
    return M, g


# ----------------------------------------------------------------------------------------------- the cases
def interior(a):
    return np.ascontiguousarray(a[1:-1, 1:-1, 1:-1])


def solve_cycles(lv, cycle, fh):
    """cycles of the hierarchy until its residual is within RTOL ||f||; u.  The EVEN-walled and periodic coefficient
    cases with a small sigma are nearly singular, and 30 sweeps on 4^3 leave their smoothest mode: about 0.75 per cycle
    there, 0.1 - 0.3 elsewhere."""
    L = lv[0]
    L.interior(L.f)[...] = fh
    target = RTOL * np.linalg.norm(fh)
    for _ in range(200):
        if L.residual_norm() <= target:
            break
        cycle(lv)
    return interior(L.u)


def mg_setup(name):
    _, periodic, walls, sigma, p27 = MG_CASES[name]
    A_at = twenty_seven_at(SIZE) if p27 else helmholtz_at(SIZE, sigma)
    pr = Problem(1.0 / N, periodic, walls, sigma=sigma, terms=A_at(0) if p27 else None)

    def oracle():
        return mo.hierarchy(SIZE, LEVELS, A_at, np.float64, (periodic,) * 3, walls or {}, m=8 if p27 else 2)

    def residual(u, f):
        L = oracle()[0]
        L.interior(L.u)[...] = u
        L.interior(L.f)[...] = f
        L.residual_norm()
        return interior(L.r)

    return pr, residual, lambda fh, x0: solve_cycles(oracle(), mo.vcycle, fh)


def vmg_setup(name):
    _, periodic, walls, cw, kind, sig = VMG_CASES[name]
    ncoef = 4 if sig else 3
    kinds = ("x", "y", "z", "cell")[:ncoef]
    A_at = lambda l: vm.helmholtz_div_grad(2.0**l / 32, sigma_field=sig)  # noqa: E731
    kp = fields(SIZE, np.dtype(np.float64), kind, ncoef)
    pr = Problem(1.0 / 32, periodic, walls, [interior(k) for k in kp[:3]], cw, interior(kp[3]) if sig else 0.0)

    def oracle():
        lv = vm.hierarchy(SIZE, LEVELS, A_at, np.float64, (periodic,) * 3, walls or {}, [dict(cw) for _ in range(ncoef)])
        for a, k in zip(lv[0].k, kp):
            a[...] = k
        vm.update_coefficients(lv, kinds)
        return lv

    def residual(u, f):
        L = oracle()[0]
        L.interior(L.u)[...] = u
        L.interior(L.f)[...] = f
        L.residual_norm()
        return interior(L.r)

    return pr, residual, lambda fh, x0: solve_cycles(oracle(), vm.vcycle, fh)


def krylov_setup(periodic, walls, cw, kappa, sigma, conv_b, precond, bicg):
    """The fine operator of test_gpu_krylov.Setup / test_gpu_bicgstab.Setup (h = 1/32, their kappa and sigma fields)"""
    cw = {} if periodic or cw is None else cw
    h = 1.0 / 32
    ncoef = 0 if kappa is None else 4 if sigma == "field" else 3
    kinds = ("x", "y", "z", "cell")[:ncoef]
    kp = []
    if ncoef:
        kp = vm.kappa_faces(SIZE, h, kappa, np.float64)
        if ncoef == 4:
            kp.append(np.random.default_rng(7 + 11).uniform(0.5, 2.0, tuple(n + 2 for n in SIZE)))
    cv = (lambda l: conv(h * 2**l)) if conv_b else (lambda l: [])
    if kappa is None:
        A_at = lambda l: poisson(h * 2**l, sigma) + cv(l)  # noqa: E731
    else:
        A_at = lambda l: vm.helmholtz_div_grad(h * 2**l, sigma_field=sigma == "field") + cv(l)  # noqa: E731
    sig = interior(kp[3]) if ncoef == 4 else (sigma or 0.0)
    pr = Problem(h, periodic, walls, [interior(k) for k in kp[:3]] if ncoef else None, cw, sig, B if conv_b else (0.0, 0.0, 0.0))

    def oracle():
        per, hom = (periodic,) * 3, ko.homogeneous(walls)
        if not kp:
            lv = mo.hierarchy(SIZE, LEVELS, A_at, np.float64, per, hom)
        else:
            lv = vm.hierarchy(SIZE, LEVELS, A_at, np.float64, per, hom, [dict(cw) for _ in kp])
            for a, k in zip(lv[0].k, kp):
                a[...] = k
            vm.update_coefficients(lv, kinds)
        return bo.BiCGStab(lv, walls) if bicg else ko.PCG(lv, walls, precond=precond)

    def residual(u, f):
        s = oracle()
        s.I(s.x)[...] = u
        s.I(s.f)[...] = f
        return interior(s.residual())

    def solve(fh, x0):
        s = oracle()
        s.I(s.x)[...] = x0
        s.I(s.f)[...] = fh
        s.solve(RTOL, 300)
        assert s.breakdown is None
        return interior(s.x)

    return pr, residual, solve


SETUPS = {"mg-" + n: (mg_setup, n) for n in MG_CASES}
SETUPS.update({"vmg-" + n: (vmg_setup, n) for n in VMG_CASES})
SETUPS.update({"pcg-" + n: (lambda n: krylov_setup(*PCG_CASES[n][1:6], False, PCG_CASES[n][6], False), n) for n in PCG_CASES})
SETUPS.update({"bicgstab-" + n: (lambda n: krylov_setup(*BICG_CASES[n][1:], True, True, True), n) for n in BICG_CASES})
NAMES = sorted(SETUPS)


def setup(name):
    make, arg = SETUPS[name]
    return make(arg)


_MATRICES = {}


def matrix(name, pr):
    if name not in _MATRICES:
        _MATRICES[name] = assemble(pr)
    return _MATRICES[name]


def data(seed=7):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1, 1, SIZE), rng.uniform(-0.5, 0.5, SIZE)


@pytest.mark.parametrize("name", NAMES)
def test_operator(name):
    pr, residual, _ = setup(name)
    M, g = matrix(name, pr)
    rng = np.random.default_rng(3)
    u, f = rng.uniform(-1, 1, SIZE), rng.uniform(-1, 1, SIZE)
    got = residual(u, f).ravel()
    want = f.ravel() - (M @ u.ravel() + g)
    scale = np.abs(f.ravel()) + np.abs(M) @ np.abs(u.ravel()) + np.abs(g)
    err = np.abs(got - want)
    assert np.all(err <= ULPS * np.finfo(np.float64).eps * scale), (name, float(np.max(err / scale)) / np.finfo(np.float64).eps)


@pytest.mark.parametrize("name", NAMES)
def test_solution(name):
    pr, _, solve = setup(name)
    M, g = matrix(name, pr)
    fh, x0 = data()
    x = solve(fh, x0).ravel()
    f = fh.ravel()
    res = np.linalg.norm(f - (M @ x + g))
    assert res <= 10 * RTOL * np.linalg.norm(f), (name, res / np.linalg.norm(f))
    exact = np.linalg.solve(M, f - g)
    assert np.linalg.norm(x - exact) <= SOLUTION_RTOL * np.linalg.norm(exact), (name, np.linalg.norm(x - exact) / np.linalg.norm(exact))
