"""numpy restatement of the BiCGStab Krylov modes (include/stencil_b200.h: SB_KRYLOV_BICG_P and SB_KRYLOV_UPDATE with c;
DESIGN.md section 2.14) and of the right-preconditioned BiCGStab stencil_b200.BiCGStab runs, with one V-cycle of
tests/vmg_oracle.py (or tests/mg_oracle.py for a constant-coefficient op) from zero as the preconditioner.

Arrays are [z, y, x]; the solver's arrays are padded by one ghost cell (origin (-1, -1, -1)) as in krylov_oracle.  Every
per-cell operation is one numpy operation in the array's dtype, so each is rounded separately, as on the GPU; a dot is
the exact sum of the double products, rounded once."""
from __future__ import annotations

import math
from typing import List, Optional

import numpy as np

import krylov_oracle as ko


# --------------------------------------------------------------------------------------------- the per-cell modes
def bicg_p(p: np.ndarray, r: np.ndarray, v: np.ndarray, beta: float, omega: float) -> np.ndarray:
    """p = r + T(beta) * (p - T(omega) * v)."""
    T = p.dtype.type
    b, w = T(beta), T(omega)
    dt = p.dtype
    return np.add(r, np.multiply(b, np.subtract(p, np.multiply(w, v, dtype=dt), dtype=dt), dtype=dt), dtype=dt)


def bicg_p_loop(p, r, v, beta, omega):
    T = p.dtype.type
    b, w = T(beta), T(omega)
    out = np.empty_like(p)
    for i in np.ndindex(p.shape):
        out[i] = T(r[i] + T(b * T(p[i] - T(w * v[i]))))
    return out


def dot(a: np.ndarray, b: np.ndarray) -> float:
    """<a, b> by the exact rule, special values included (krylov_oracle.dot where every term is finite)."""
    with np.errstate(over="ignore", invalid="ignore"):
        terms = a.astype(np.float64) * b.astype(np.float64)
    return ko.dot(a, b) if np.isfinite(terms).all() else ko.exact_sum(terms.ravel())


def update_c(x, p, r, q, c, s):
    """UPDATE with c: x + T(s) p, r - T(s) q, <r', r'>, <c, r'> of the new r'."""
    xn, rn = ko.update(x, p, r, q, s)
    return xn, rn, dot(rn, rn), dot(c, rn)


# --------------------------------------------------------------------------------------------- M on another pair
def cycle_pair(lv, u: np.ndarray, f: np.ndarray, cycle, *args) -> None:
    """One cycle of the hierarchy lv on the fine pair (u, f) in place: lv[0]'s u and f swapped for the pair, the coarse
    levels shared (stencil_b200.Multigrid.cycle(u=, f=))."""
    L = lv[0]
    keep = L.u, L.f
    L.u, L.f = u, f
    try:
        cycle(lv, *args)
    finally:
        L.u, L.f = keep


# --------------------------------------------------------------------------------------------- the solver
class BiCGStab(ko.PCG):
    """stencil_b200.BiCGStab on one grid: lv is the preconditioner's hierarchy (as for krylov_oracle.PCG, with the
    homogeneous walls on level 0), x_walls x's own walls.  x and f are padded arrays of lv[0]'s shape; x holds the first
    guess.  <t, r> and <t, t> are exact, so one two-pair dot and two one-pair dots give the same values."""

    def __init__(self, lv, x_walls, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30):
        super().__init__(lv, x_walls, True, nu1, nu2, coarse_sweeps)
        shape, dtype = self.L.u.shape, self.L.u.dtype
        self.r0, self.v, self.t = (np.zeros(shape, dtype) for _ in range(3))
        self.ph, self.sh = (np.zeros(shape, dtype) for _ in range(2))

    def start(self) -> float:
        self.r = self.residual()
        self.r0 = self.r.copy()
        self.rho = ko.dot(self.I(self.r0), self.I(self.r))
        return self.rho

    def iterate(self, k: int, target: float, hist: List[float]) -> bool:
        """Iteration k of stencil_b200.BiCGStab._iterate, step for step."""
        I = self.I
        if k == 0:
            I(self.p)[...] = ko.xpby(I(self.p), I(self.r), 0.0)
        else:
            beta = (self.rho / self.rho_prev) * (self.alpha / self.omega)
            I(self.p)[...] = bicg_p(I(self.p), I(self.r), I(self.v), beta, self.omega)
        self.ph = self.M(self.p)
        self.v = self.apply_A(self.ph)
        sigma = ko.dot(I(self.r0), I(self.v))
        if sigma == 0.0 or not math.isfinite(sigma):
            self.breakdown = k
            return False
        alpha = self.rho / sigma
        xn, rn = ko.update(I(self.x), I(self.ph), I(self.r), I(self.v), alpha)
        I(self.x)[...] = xn
        I(self.r)[...] = rn
        ss = ko.dot(I(self.r), I(self.r))
        self.sh = self.M(self.r)
        self.t = self.apply_A(self.sh)
        t_r, t_t = ko.dot(I(self.t), I(self.r)), ko.dot(I(self.t), I(self.t))
        hist.append(math.sqrt(ss))
        if hist[-1] <= target:
            return False
        omega = t_r / t_t if t_t != 0.0 else 0.0
        if t_t == 0.0 or omega == 0.0 or not math.isfinite(omega):
            self.breakdown = k
            return False
        xn, rn, rr, rho = update_c(I(self.x), I(self.sh), I(self.r), I(self.t), I(self.r0), omega)
        I(self.x)[...] = xn
        I(self.r)[...] = rn
        hist[-1] = math.sqrt(rr)
        self.rho_prev, self.rho, self.alpha, self.omega = self.rho, rho, alpha, omega
        if hist[-1] <= target:
            return False
        if rho == 0.0 or not math.isfinite(rho):
            self.breakdown = k
            return False
        return True

    def solve(self, rtol: float, max_iters: int) -> List[float]:
        target = rtol * math.sqrt(ko.dot(self.I(self.f), self.I(self.f)))
        self.breakdown: Optional[int] = None
        hist = [math.sqrt(self.start())]
        k = 0
        while hist[-1] > target and k < max_iters:
            if not self.iterate(k, target, hist):
                break
            k += 1
        return hist
