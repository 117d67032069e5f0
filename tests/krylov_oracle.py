"""numpy restatement of the Krylov vector kernels (include/stencil_b200.h: sb_krylov_plan_*; DESIGN.md section 2.13) and
of the flexible CG stencil_b200.PCG runs, preconditioned by one V-cycle of tests/vmg_oracle.py.

Arrays are [z, y, x]; the solver's arrays are padded by one ghost cell (origin (-1, -1, -1)) as in vmg_oracle.  Every
per-cell operation is one numpy operation in the array's dtype, so each is rounded separately, as on the GPU; a dot is
math.fsum of the double products, the exact sum rounded once."""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Dict, List, Optional

import numpy as np

import mg_oracle as mo
import vmg_oracle as vm
import vstencil_oracle as vo


# --------------------------------------------------------------------------------------------- the per-cell modes
def dot(a: np.ndarray, b: np.ndarray) -> float:
    """<a, b>: the exact sum of fl64(double(a) * double(b)), rounded once (finite terms)."""
    return math.fsum((a.astype(np.float64) * b.astype(np.float64)).ravel())


def xpby(p: np.ndarray, z: np.ndarray, s: float) -> np.ndarray:
    """p = z + T(s) * p; T(s) = +-0: p = z (p is not read)."""
    T = p.dtype.type
    t = T(s)
    if t == 0:
        return z.copy()
    return np.add(z, np.multiply(t, p, dtype=p.dtype), dtype=p.dtype)


def update(x: np.ndarray, p: np.ndarray, r: np.ndarray, q: np.ndarray, s: float):
    """x + T(s) * p, r - T(s) * q."""
    t = x.dtype.type(s)
    return (np.add(x, np.multiply(t, p, dtype=x.dtype), dtype=x.dtype), np.subtract(r, np.multiply(t, q, dtype=x.dtype), dtype=x.dtype))


def xpby_loop(p: np.ndarray, z: np.ndarray, s: float) -> np.ndarray:
    T = p.dtype.type
    t = T(s)
    out = np.empty_like(p)
    for i in np.ndindex(p.shape):
        out[i] = z[i] if t == 0 else T(z[i] + T(t * p[i]))
    return out


def update_loop(x, p, r, q, s):
    T = x.dtype.type
    t = T(s)
    xo, ro = np.empty_like(x), np.empty_like(r)
    for i in np.ndindex(x.shape):
        xo[i] = T(x[i] + T(t * p[i]))
        ro[i] = T(r[i] - T(t * q[i]))
    return xo, ro


def exact_sum(terms) -> float:
    """The sb_reduce_exact rule for a sum with special values: a NaN term or both infinities give NaN, one infinity
    gives it, else the exact rational sum rounded once to double (beyond the range: +-inf; an exact zero: +0.0)."""
    terms = [float(t) for t in terms]
    if any(t != t for t in terms) or (math.inf in terms and -math.inf in terms):
        return math.nan
    if math.inf in terms:
        return math.inf
    if -math.inf in terms:
        return -math.inf
    s = sum((Fraction(t) for t in terms), Fraction(0))
    if s == 0:
        return 0.0
    try:
        return float(s)  # Fraction -> float rounds to nearest, ties to even
    except OverflowError:
        return math.inf if s > 0 else -math.inf


def exact_dot(a: np.ndarray, b: np.ndarray) -> float:
    """<a, b> by exact_sum: the reference of dot() with special values."""
    with np.errstate(over="ignore", invalid="ignore"):
        return exact_sum((a.astype(np.float64) * b.astype(np.float64)).ravel())


def ordered_min_max(v: np.ndarray):
    """min / max of v by sb_reduce_exact_combine's order-independent rule: a NaN wins (the larger bit pattern of two);
    of +0 and -0 min takes -0 and max +0; empty: +inf, -inf."""
    v = np.asarray(v, np.float64).ravel()
    if v.size == 0:
        return math.inf, -math.inf
    nan = v[np.isnan(v)]
    if nan.size:
        x = nan.view(np.uint64).max().view(np.float64)
        return float(x), float(x)
    mn, mx = v.min(), v.max()
    if mn == 0 and np.any((v == 0) & np.signbit(v)):
        mn = -0.0
    if mx == 0 and np.any((v == 0) & ~np.signbit(v)):
        mx = 0.0
    return float(mn), float(mx)


# --------------------------------------------------------------------------------------------- the solver
def homogeneous(walls: Dict[int, vm.Wall]) -> Dict[int, vm.Wall]:
    """The walls of a Krylov vector for x's walls: ODD(c) -> ODD(0), EVEN -> EVEN, VALUE(c) -> VALUE(0)."""
    return {f: (k, 0.0) for f, (k, c) in walls.items()}


class PCG:
    """stencil_b200.PCG on one grid: lv is the preconditioner's hierarchy (vm.hierarchy with the homogeneous walls on
    level 0 and its coefficient fields set, or mg_oracle.hierarchy for a constant-coefficient op), x_walls x's own
    walls; precond=False: z is r and lv[0] only gives A and the fields.  x and f are padded arrays of lv[0]'s shape; x
    holds the first guess."""

    def __init__(self, lv: List[vm.Level], x_walls: Dict[int, vm.Wall], precond: bool = True, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30):
        self.lv, self.L = lv, lv[0]
        self.x_walls = dict(x_walls)
        self.hom = homogeneous(x_walls)
        self.precond, self.nu1, self.nu2, self.coarse_sweeps = precond, nu1, nu2, coarse_sweeps
        shape, dtype = self.L.u.shape, self.L.u.dtype
        self.x, self.f, self.r, self.p, self.q = (np.zeros(shape, dtype) for _ in range(5))
        self.breakdown: Optional[int] = None
        self.k, self.coef_walls = getattr(self.L, "k", []), getattr(self.L, "coef_walls", [])
        self.vcycle = vm.vcycle if hasattr(self.L, "k") else mo.vcycle

    def I(self, a):
        return a[1:-1, 1:-1, 1:-1]

    def _fill_coefs(self):
        for k, w in zip(self.k, self.coef_walls):
            vm.fill_ghosts(k, self.L.periodic, w)

    def apply_A(self, p: np.ndarray) -> np.ndarray:
        """q = A p, p's ghosts from the homogeneous walls."""
        vm.fill_ghosts(p, self.L.periodic, self.hom)
        self._fill_coefs()
        q = np.zeros_like(p)
        vo.apply_box(self.L.A, p, None, self.k, q, (1, 1, 1), self.L.size)
        return q

    def residual(self) -> np.ndarray:
        """f - A x with x's own walls."""
        vm.fill_ghosts(self.x, self.L.periodic, self.x_walls)
        self._fill_coefs()
        r = np.zeros_like(self.x)
        vo.apply_box(self.L.res, self.x, self.f, self.k, r, (1, 1, 1), self.L.size)
        return r

    def M(self, r: np.ndarray) -> np.ndarray:
        if not self.precond:
            return r
        self.L.u[...] = 0
        self.I(self.L.f)[...] = self.I(r)
        self.vcycle(self.lv, 0, self.nu1, self.nu2, self.coarse_sweeps)
        return self.L.u.copy()

    def start(self) -> float:
        self.r = self.residual()
        return dot(self.I(self.r), self.I(self.r))

    def iterate(self, k: int) -> Optional[float]:
        I = self.I
        z = self.M(self.r)
        gamma = dot(I(z), I(self.r))
        delta = dot(I(z), I(self.q)) if k else 0.0
        if not math.isfinite(gamma):
            self.breakdown = k
            return None
        beta = 0.0 if k == 0 else -delta / self.eta
        p = self.p.copy()
        I(p)[...] = xpby(I(self.p), I(z), beta)
        self.p = p
        self.q = self.apply_A(self.p)
        eta = dot(I(self.p), I(self.q))
        if not (math.isfinite(eta) and eta > 0.0):
            self.breakdown = k
            return None
        self.eta = eta
        xn, rn = update(I(self.x), I(self.p), I(self.r), I(self.q), gamma / eta)
        I(self.x)[...] = xn
        I(self.r)[...] = rn
        return dot(I(self.r), I(self.r))

    def solve(self, rtol: float, max_iters: int) -> List[float]:
        target = rtol * math.sqrt(dot(self.I(self.f), self.I(self.f)))
        self.breakdown = None
        hist = [math.sqrt(self.start())]
        k = 0
        while hist[-1] > target and k < max_iters:
            rho = self.iterate(k)
            if rho is None:
                break
            hist.append(math.sqrt(rho))
            k += 1
        return hist

    def residual_norm(self) -> float:
        r = self.residual()
        return math.sqrt(dot(self.I(r), self.I(r)))
