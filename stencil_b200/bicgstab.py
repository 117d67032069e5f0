"""Multigrid-preconditioned BiCGStab for A x = f on a DistributedDomain (DESIGN.md section 2.14): right-preconditioned
BiCGStab for non-symmetric operators such as advection-diffusion, -div(kappa grad x) + b . grad x (+ sigma x), with one
V-cycle of stencil_b200.Multigrid from zero as the preconditioner, the vector algebra in the fused sm_90a Krylov kernels
and every inner product exact, so the iterates are the same bits on every partition and rank count.

    A_at = lambda l: sb.StencilOp(diffusion(h * 2**l) + convection(b, h * 2**l), np.float64)
    bi = sb.BiCGStab(dd, x, f, r, r0, p, v, phat, shat, t, A_at, coefs=[kx, ky, kz])   # nine quantities, then kappa
    history = bi.solve(1e-8, 30)                                                      # sqrt(<r, r>) per step
    bi.close()

phat and shat must carry the homogeneous counterpart of x's wall BC on every FIXED face (homogeneous_bc), as PCG's p
and z do; x keeps its own BC, which enters through the first residual.  A breakdown (<r0, v> zero or not finite, <t, t>
zero, omega zero or not finite, or a new <r0, r> zero or not finite) stops the solve and is recorded in .breakdown.
dd.swap() may be called between solves: every pass looks its buffers up for the current swap parity."""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib
from .domain import DataHandle, DistributedDomain
from .krylov import _KrylovSolver
from .multigrid import Multigrid
from .stencil_op import StencilOp


class BiCGStab(_KrylovSolver):
    """Right-preconditioned BiCGStab for A x = f on the realized domain dd.  x, f, r, r0, p, v, phat, shat and t are nine
    distinct float32 or float64 quantities of dd (curr buffers): x the solution (its initial value is the first guess),
    f the right-hand side, r the residual (s from the half step on), r0 the shadow residual, p the direction, v = A phat,
    phat = M p, shat = M s and t = A shat.  op_at(l) returns A on level l as Multigrid takes it; an internal
    Multigrid(dd, phat, p, v, op_at, nu1, nu2, coarse_sweeps, levels, coefs, coef_kinds) is M, run on the pair (phat, p)
    and, by Multigrid.cycle(u=shat, f=r), on (shat, r) (v is only the scratch of its residual_norm, which BiCGStab never
    calls).  coefs / coef_kinds: as for Multigrid.  Building, solve(), residual_norm() and update_coefficients() are
    collective under torchrun.  The solver never calls dd.swap(); a caller may swap between solves.
    Each exchange of a solve moves only what the pass reads at an offset (x for the residual, the vector A is applied to,
    u on each V-cycle level; the coefficient fields once per solve), so after a solve the ghost cells of the solver's
    scratch quantities are no longer refreshed as a side effect (DESIGN.md section 2.15)."""

    NAMES = ("x", "f", "r", "r0", "p", "v", "phat", "shat", "t")

    def __init__(self, dd: DistributedDomain, x: DataHandle, f: DataHandle, r: DataHandle, r0: DataHandle, p: DataHandle, v: DataHandle,
                 phat: DataHandle, shat: DataHandle, t: DataHandle, op_at: Callable[[int], StencilOp], coefs: Optional[Sequence[DataHandle]] = None,
                 coef_kinds: Optional[Sequence[str]] = None, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30, levels: Optional[int] = None):
        super().__init__("BiCGStab", dd, dict(zip(self.NAMES, (x, f, r, r0, p, v, phat, shat, t))), ("phat", "shat"), op_at, coefs)
        self.r0, self.p, self.v, self.phat, self.shat, self.t = r0, p, v, phat, shat, t
        self.mg = Multigrid(dd, phat, p, v, op_at, nu1=nu1, nu2=nu2, coarse_sweeps=coarse_sweeps, levels=levels, coefs=self.coefs,
                            coef_kinds=coef_kinds)
        try:
            self.mg._fine_level(shat, r)  # the second pair's checks, now rather than at the first solve
        except Exception:
            self.close()
            raise
        # <t, r> and <t, t> by one two-pair DOT in FP64; in FP32 by two one-pair DOTs, the faster form there (section
        # 2.13).  The sums are exact either way, so the choice changes no bit.
        self._split_tr_tt = dd.dtypes_[x.id] == np.dtype(np.float32)

    def _start(self) -> float:
        """r = f - A x with x's own BC through the exchange, r0 = r; returns rho = <r0, r> (= <r, r>)."""
        self._residual()
        self._queue(self._plans(_lib.KRYLOV_XPBY, self.r0, self.r), 0.0)
        rr = self._plans(_lib.KRYLOV_DOT, self.r0, self.r)
        self._queue(rr)
        return self._combine(rr)[0]

    def _iterate(self, k: int, target: float, hist: List[float]) -> bool:
        """Iteration k (from 0); appends sqrt(<r, r>) of each new x to hist.  Returns True to go on, False to stop (the
        half-step or full-step residual reached target, or a breakdown, recorded in .breakdown)."""
        K = _lib
        if k == 0:
            self._queue(self._plans(K.KRYLOV_XPBY, self.p, self.r), 0.0)
        else:
            beta = (self._rho / self._rho_prev) * (self._alpha / self._omega)
            self._queue(self._plans(K.KRYLOV_BICG_P, self.p, self.r, self.v), beta, self._omega)
        self._precondition(self.phat, self.p)
        self._apply_A(self.v, self.phat)
        rv = self._plans(K.KRYLOV_DOT, self.r0, self.v)
        self._queue(rv)
        sigma = self._combine(rv)[0]
        if sigma == 0.0 or not math.isfinite(sigma):
            self.breakdown = k
            return False
        alpha = self._rho / sigma
        half = self._plans(K.KRYLOV_UPDATE, self.x, self.phat, self.r, self.v)
        self._queue(half, alpha)
        self._precondition(self.shat, self.r)
        self._apply_A(self.t, self.shat)
        if self._split_tr_tt:
            tr, tt = self._plans(K.KRYLOV_DOT, self.t, self.r), self._plans(K.KRYLOV_DOT, self.t, self.t)
            self._queue(tr)
            self._queue(tt)
            ss, t_r, t_t = self._combine(half, tr, tt)
        else:
            trt = self._plans(K.KRYLOV_DOT, self.t, self.r, self.t)
            self._queue(trt)
            ss, t_r, t_t = self._combine(half, trt)
        hist.append(math.sqrt(ss))
        if hist[-1] <= target:
            return False
        omega = t_r / t_t if t_t != 0.0 else 0.0
        if t_t == 0.0 or omega == 0.0 or not math.isfinite(omega):
            self.breakdown = k
            return False
        full = self._plans(K.KRYLOV_UPDATE, self.x, self.shat, self.r, self.t, self.r0)
        self._queue(full, omega)
        rr, rho = self._combine(full)
        hist[-1] = math.sqrt(rr)
        self._rho_prev, self._rho, self._alpha, self._omega = self._rho, rho, alpha, omega
        if hist[-1] <= target:
            return False
        if rho == 0.0 or not math.isfinite(rho):
            self.breakdown = k
            return False
        return True

    def solve(self, rtol: float, max_iters: int) -> List[float]:
        """Iterations from the current x until sqrt(<r, r>) <= rtol ||f||_2 (||f||_2 exact, as Multigrid.solve) or
        max_iters iterations; returns sqrt(<r, r>) before the first iteration and after each, the last entry being that
        of the x left behind: the half-step iterate when the half step reached the target or omega broke down.  r is
        the recursive residual (residual_norm() gives the true one).  A breakdown stops the solve with the history so far
        and sets .breakdown to its iteration (None otherwise).  Every rank calls it."""
        target = float(rtol) * self.dd.reduce(self.f, "curr", exact=True).l2()
        self.breakdown = None
        self._rho = self._start()
        hist = [math.sqrt(self._rho)]
        k = 0
        while hist[-1] > target and k < int(max_iters):
            if not self._iterate(k, target, hist):
                break
            k += 1
        return hist
