"""Multigrid-preconditioned conjugate gradients for A x = f on a DistributedDomain (DESIGN.md section 2.13): flexible CG
(the Polak-Ribiere form, which tolerates the V-cycle's slight asymmetry) with one V-cycle of stencil_b200.Multigrid as
the preconditioner, the vector algebra in the fused sm_90a Krylov kernels and every inner product exact, so the
iterates are the same bits on every partition and rank count.

    A_at = lambda l: sb.StencilOp.div_grad((h * 2**l,) * 3, np.float64).scaled(-1.0)   # -div(kappa grad x) on level l
    cg = sb.PCG(dd, x, f, r, z, p, q, A_at, coefs=[kx, ky, kz])               # six quantities of dd, then kappa
    history = cg.solve(1e-8, 50)                                               # sqrt(<r, r>) per iteration
    cg.close()

p and z must carry the homogeneous counterpart of x's wall BC on every FIXED face (ODD(c) -> ODD(0), EVEN -> EVEN,
VALUE(c) -> VALUE(0)), so that A sees them as a linear operator does; x keeps its own BC, which enters through the first
residual.  A must be symmetric positive definite for CG; a breakdown (a non-positive or non-finite <p, A p>, or a
non-finite <z, r>) stops the solve and is recorded in .breakdown.  dd.swap() may be called between solves: every pass
looks its buffers up for the current swap parity."""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np

from . import _lib
from .domain import FACES, BC, BCKind, Boundary, DataHandle, DistributedDomain
from .multigrid import Multigrid, residual_op
from .stencil_op import StencilOp


def homogeneous_bc(bc: BC) -> BC:
    """The BC a Krylov vector (p, z) needs for a wall BC of x: ODD(c) -> ODD(0), EVEN -> EVEN, VALUE(c) -> VALUE(0).
    NONE has none (StencilError)."""
    if bc.kind == BCKind.ODD:
        return BC.ODD(0.0)
    if bc.kind == BCKind.EVEN:
        return BC.EVEN()
    if bc.kind == BCKind.VALUE:
        return BC.VALUE(0.0)
    raise _lib.StencilError("PCG: x needs a boundary condition (ODD, EVEN or VALUE) on every FIXED face")


class _KrylovSolver:
    """What PCG and BiCGStab share: the refusals of their vectors, A and its residual on the fine level, the
    preconditioner's handle and the queued schedule's passes and host waits.  A subclass builds self.mg on its own pair
    and keeps its solve() and _iterate()."""

    def __init__(self, who: str, dd: DistributedDomain, named: Dict[str, DataHandle], applied: Sequence[str], op_at: Callable[[int], StencilOp],
                 coefs: Optional[Sequence[DataHandle]]):
        """named: every vector by name, x, f and r among them; applied: the names of the vectors A is applied to, which
        must carry the homogeneous counterpart of x's BC on every FIXED face.  Refusals name the solver `who`."""
        self.mg: Optional[Multigrid] = None
        self.breakdown: Optional[int] = None
        if not isinstance(dd, DistributedDomain) or dd.partition_ is None or not dd._plans:
            raise _lib.StencilError(f"{who}: dd must be a realized DistributedDomain")
        for name, h in named.items():
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(dd.dtypes_):
                raise _lib.StencilError(f"{who}: {name} must be a DataHandle of dd, not {h!r}")
        names = ", ".join(named)
        if len({h.id for h in named.values()}) != len(named):
            raise _lib.StencilError(f"{who}: {names} must be {len(named)} different quantities")
        x = named["x"]
        dtype = dd.dtypes_[x.id]
        if dtype not in (np.dtype(np.float32), np.dtype(np.float64)) or any(dd.dtypes_[h.id] != dtype for h in named.values()):
            raise _lib.StencilError(f"{who}: {names} must all be float32 or all float64")
        coefs = list(coefs) if coefs is not None else []
        for k, h in enumerate(coefs):
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(dd.dtypes_):
                raise _lib.StencilError(f"{who}: coefficient {k} must be a DataHandle of dd, not {h!r}")
            if any(h.id == g.id for g in named.values()) or dd.dtypes_[h.id] != dtype:
                raise _lib.StencilError(f"{who}: coefficient {k} must be a quantity of x's type other than {names}")
        for fc in range(6):
            if dd.boundary_[fc // 2] != Boundary.FIXED:
                continue
            bx = dd.bcs_.get((x.id, fc), BC.NONE())
            if bx.kind == BCKind.NONE:
                raise _lib.StencilError(f"{who}: x needs a boundary condition (ODD, EVEN or VALUE) on every FIXED face (face {FACES[fc]})")
            want = homogeneous_bc(bx)
            for name in applied:
                got = dd.bcs_.get((named[name].id, fc), BC.NONE())
                if got != want:
                    raise _lib.StencilError(f"{who}: {name} needs {want!r} on face {FACES[fc]}, the homogeneous counterpart of x's {bx!r}, not {got!r}")
        A = op_at(0)
        if not isinstance(A, StencilOp) or A.dtype != dtype:
            raise _lib.StencilError(f"{who}: op_at(0) must be a StencilOp in {dtype}, not {A!r}")
        if A.has_aux:
            raise _lib.StencilError(f"{who}: op_at(0) has an aux term; A reads x only")
        if A.ncoef != len(coefs):
            raise _lib.StencilError(f"{who}: op_at(0) reads {A.ncoef} coefficient fields, but {len(coefs)} were given")
        A.check(dd.radius_)
        self.dd, self.x, self.f, self.r = dd, x, named["f"], named["r"]
        self.A, self.res = A, residual_op(A)
        self.coefs = coefs or None
        dd._ensure_apply_streams()

    # -- the queued schedule
    def _plans(self, mode: int, *handles: DataHandle):
        """The pass's plans on the curr buffers of the current swap parity (dd's cache)."""
        return self.dd.krylov_plans(mode, handles)

    def _queue(self, plans, s: float = 0.0, t: float = 0.0) -> None:
        for pl in plans:
            pl.s, pl.t = float(s), float(t)
        self.dd._run_plans([(pl,) for pl in plans], False, queued=True)

    def _combine(self, *launched) -> List[float]:
        """Host wait: each subdomain's parts of the last launch of each plan list in launched, on its interior apply
        stream (where _queue put them), gathered across ranks in one exchange, combined and rounded once."""
        dd = self.dd
        mine = []
        for di, (idx, (si, _)) in enumerate(zip(dd.domain_idx_, dd._apply_streams)):
            mine.append((idx, [part for plans in launched for part in plans[di].parts(si)]))
        return [red.sum for red in dd._exact_gather(mine, sum(plans[0].n for plans in launched))]

    def _apply_A(self, out: DataHandle, src: DataHandle) -> None:
        self.dd._run_plans(*self.dd._apply_plans(self.A, (out, "curr"), src, None, (src,), self.coefs), queued=True)

    def _residual(self) -> None:
        """r = f - A x with x's own BC through the exchange, queued after the work on the caller's stream.  The first pass
        of a solve: the coefficient fields are exchanged here, once per solve, as every later exchange moves only the
        vector A reads (DESIGN.md section 2.15)."""
        dd = self.dd
        dd._follow_caller()
        if self.coefs:
            dd._queue_exchange(dd._exchange_sel(type(self).__name__, tuple(self.coefs), ()))
        dd._run_plans(*dd._apply_plans(self.res, (self.r, "curr"), self.x, (self.f, "curr"), (self.x,), self.coefs), queued=True)

    def _precondition(self, u: DataHandle, f: DataHandle) -> None:
        """u = M f: u set to +0, then one cycle on the pair (u, f), queued."""
        self.dd._queue_clear(u)
        self.mg.cycle(wait=False, u=u, f=f)

    def residual_norm(self) -> float:
        """The true ||f - A x||_2 over dd's compute region (the residual into r, then an exact dot)."""
        self.dd.apply(self.res, (self.r, "curr"), self.x, (self.f, "curr"), coefs=self.coefs)
        return math.sqrt(self.dd.dot(self.r, self.r))

    def update_coefficients(self) -> None:
        """Re-coarsen the preconditioner's coefficient fields after they change (Multigrid.update_coefficients); A on
        the fine level reads the fields directly."""
        if self.mg is not None:
            self.mg.update_coefficients()

    def close(self) -> None:
        """Release the preconditioner's coarse domains (the Krylov plans stay in dd's cache until dd.close())."""
        if self.mg is not None:
            self.mg.close()
            self.mg = None


class PCG(_KrylovSolver):
    """Flexible preconditioned CG for A x = f on the realized domain dd.  x, f, r, z, p and q are distinct float32 or
    float64 quantities of dd (curr buffers): x the solution (its initial value is the first guess), f the right-hand side,
    r the residual, z the preconditioned residual, p the search direction and q = A p.  op_at(l) returns A on level l as
    Multigrid takes it; with precond="multigrid" an internal Multigrid(dd, z, r, q, op_at, nu1, nu2, coarse_sweeps, levels,
    coefs, coef_kinds) is the preconditioner (its u is z, its f is r; q is only the scratch of its residual_norm, which
    PCG never calls).  With precond=None, z must be None, z is r, and only op_at(0) is used.  coefs / coef_kinds: as for
    Multigrid.  Building, solve(), residual_norm() and update_coefficients() are collective under torchrun.  The solver
    never calls dd.swap(); a caller may swap between solves (the passes follow the current curr buffers).
    Each exchange of a solve moves only what the pass reads at an offset (x for the residual, the vector A is applied to,
    u on each V-cycle level; the coefficient fields once per solve), so after a solve the ghost cells of the solver's
    scratch quantities are no longer refreshed as a side effect (DESIGN.md section 2.15)."""

    def __init__(self, dd: DistributedDomain, x: DataHandle, f: DataHandle, r: DataHandle, z: Optional[DataHandle], p: DataHandle, q: DataHandle,
                 op_at: Callable[[int], StencilOp], precond: Optional[str] = "multigrid", coefs: Optional[Sequence[DataHandle]] = None,
                 coef_kinds: Optional[Sequence[str]] = None, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30, levels: Optional[int] = None):
        if precond not in ("multigrid", None):
            raise _lib.StencilError(f"PCG: precond must be 'multigrid' or None, not {precond!r}")
        if precond is None and z is not None:
            raise _lib.StencilError("PCG: without a preconditioner z is r; pass z=None")
        named = dict(x=x, f=f, r=r, p=p, q=q, **({"z": z} if precond else {}))
        super().__init__("PCG", dd, named, ("p", "z") if precond else ("p",), op_at, coefs)
        self.p, self.q = p, q
        self.z = z if precond else r
        self.precond = precond
        if precond:
            self.mg = Multigrid(dd, z, r, q, op_at, nu1=nu1, nu2=nu2, coarse_sweeps=coarse_sweeps, levels=levels, coefs=self.coefs,
                                coef_kinds=coef_kinds)
        # <z, r> and <z, q> by one two-pair DOT in FP64 (3 reads instead of 4); in FP32 the two-pair kernel is bound by its
        # per-cell work and two one-pair launches are faster (DESIGN.md section 2.13).  The sums are exact either way.
        self._split_gamma_delta = dd.dtypes_[x.id] == np.dtype(np.float32)

    def _start(self) -> float:
        """r = f - A x, with x's own BC through the exchange; returns rho = <r, r>."""
        self._residual()
        rr = self._plans(_lib.KRYLOV_DOT, self.r, self.r)
        self._queue(rr)
        return self._combine(rr)[0]

    def _iterate(self, k: int) -> Optional[float]:
        """Iteration k (from 0): returns rho = <r, r> of the new r, or None at a breakdown (recorded in .breakdown)."""
        if self.mg is not None:
            self._precondition(self.z, self.r)
        K = _lib
        if k == 0:
            zr = self._plans(K.KRYLOV_DOT, self.z, self.r)
            self._queue(zr)
            gamma, delta = self._combine(zr)[0], 0.0
        elif self._split_gamma_delta:
            zr, zq = self._plans(K.KRYLOV_DOT, self.z, self.r), self._plans(K.KRYLOV_DOT, self.z, self.q)
            self._queue(zr)
            self._queue(zq)
            gamma, delta = self._combine(zr, zq)
        else:
            zrq = self._plans(K.KRYLOV_DOT, self.z, self.r, self.q)
            self._queue(zrq)
            gamma, delta = self._combine(zrq)
        if not math.isfinite(gamma):
            self.breakdown = k
            return None
        beta = 0.0 if k == 0 else -delta / self._eta
        self._queue(self._plans(K.KRYLOV_XPBY, self.p, self.z), beta)
        self._apply_A(self.q, self.p)
        pq = self._plans(K.KRYLOV_DOT, self.p, self.q)
        self._queue(pq)
        eta = self._combine(pq)[0]
        if not (math.isfinite(eta) and eta > 0.0):
            self.breakdown = k
            return None
        self._eta = eta
        up = self._plans(K.KRYLOV_UPDATE, self.x, self.p, self.r, self.q)
        self._queue(up, gamma / eta)
        return self._combine(up)[0]

    def solve(self, rtol: float, max_iters: int) -> List[float]:
        """Iterations from the current x until sqrt(<r, r>) <= rtol ||f||_2 (||f||_2 exact, as Multigrid.solve) or
        max_iters iterations; returns sqrt(<r, r>) before the first iteration and after each.  r is the recursive
        residual (residual_norm() gives the true one).  A breakdown stops the solve with the history so far and sets
        .breakdown to its iteration (None otherwise).  Every rank calls it."""
        target = float(rtol) * self.dd.reduce(self.f, "curr", exact=True).l2()
        self.breakdown = None
        hist = [math.sqrt(self._start())]
        k = 0
        while hist[-1] > target and k < int(max_iters):
            rho = self._iterate(k)
            if rho is None:
                break
            hist.append(math.sqrt(rho))
            k += 1
        return hist
