"""Geometric multigrid for A u = f on a DistributedDomain (DESIGN.md section 2.11): V(nu1, nu2) cycles over a hierarchy
of coarsenings by 2, built from the coloured sweeps (section 2.9), the fused residual-restriction and the prolongation
(sections 2.10, 2.11), with no host synchronisation inside a cycle.

    A = sb.StencilOp.laplacian(2, (h, h, h), np.float64).scaled(-1.0)          # -lap u = f
    mg = sb.Multigrid(dd, u, f, r, lambda l: A if l == 0 else coarse_A(l))     # A on level l, l = 0 finest
    history = mg.solve(1e-8, 20)                                                # ||f - A u||_2 per cycle
    mg.close()

Periodic Poisson (A singular) needs f of zero mean; the solver does not project.

Variable coefficients (DESIGN.md section 2.12): with coefs= the ops may have coefficient terms, such as -div(kappa grad u)
with kappa on faces in three fields; each level gets its own coarsened copy of every field and is smoothed by the
diagonal relaxation (DistributedDomain.relax) instead of A.relax(1):

    A_at = lambda l: sb.StencilOp.div_grad((h * 2**l,) * 3, np.float64).scaled(-1.0)
    mg = sb.Multigrid(dd, u, f, r, A_at, coefs=[kx, ky, kz], coef_kinds=("x", "y", "z"))
    ...                                    # kappa changes (a variable-density projection: kappa = 1 / rho)
    mg.update_coefficients()               # every coarse level re-coarsened from kx, ky, kz"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence

import numpy as np

from . import _lib
from .domain import FACES, BC, BCKind, Boundary, DataHandle, DistributedDomain, Partition, PlacementStrategy, Radius, wait_queued
from .stencil_op import StencilOp


def residual_op(A: StencilOp) -> StencilOp:
    """r = f - A u as one op on src u and aux f: (aux, 0, 1), then each term of A with its weight negated (a coefficient
    term keeps its field and coefficient offset)."""
    return StencilOp([(1, (0, 0, 0), 1.0)] + [(0, t[1], -t[2]) + tuple(t[3:]) for t in A.terms], A.dtype)


COEF_KINDS = {"x": 0, "y": 1, "z": 2, "cell": None}  # a face field's axis; None: a cell-centred field


def coarse_bc(bc: BC) -> BC:
    """The coarse correction's BC for a wall BC of u: ODD(c) -> ODD(0) (the correction of a solution pinned to c at the
    wall vanishes there), EVEN -> EVEN.  VALUE and NONE have none (StencilError)."""
    if bc.kind == BCKind.ODD:
        return BC.ODD(0.0)
    if bc.kind == BCKind.EVEN:
        return BC.EVEN()
    if bc.kind == BCKind.VALUE:
        raise _lib.StencilError("Multigrid: VALUE walls are not consistent across levels (DESIGN.md section 2.10); use ODD(c), "
                                "which pins the same value at the wall face")
    raise _lib.StencilError("Multigrid: u needs a boundary condition (ODD or EVEN) on every FIXED face")


def level_count(sizes, levels: Optional[int] = None) -> int:
    """The number of grids: halve while every subdomain extent is even and its half is >= 2, capped at levels."""
    n, cur = 1, [tuple(s) for s in sizes]
    while (levels is None or n < levels) and all(v % 2 == 0 and v // 2 >= 2 for s in cur for v in s):
        cur = [tuple(v // 2 for v in s) for s in cur]
        n += 1
    return n


class _Level:
    def __init__(self, dd: DistributedDomain, u: DataHandle, f: DataHandle, A: StencilOp, coefs: List[DataHandle]):
        self.dd, self.u, self.f, self.A, self.coefs = dd, u, f, A, coefs
        # coefficient ops: the diagonal relaxation (relax); plain ops: the SOR table, as before
        self.gs = None if A.has_coef else A.relax(1.0)
        self.res = residual_op(A)


class Multigrid:
    """V(nu1, nu2) cycles for A u = f on the realized domain dd.  u, f and r are float32 or float64 quantities of dd
    (curr buffers); r is scratch for the residual norm of solve().  op_at(l) returns A on level l (0 = dd): a StencilOp
    of dd's type with plain src terms of reach <= 1 and one centre term.  Each coarse level is a DistributedDomain of u
    and f on the same GPUs, placement and boundary kinds as dd, with dd's radius raised to >= 1 in all 26 directions;
    the grid is halved while every subdomain extent is even and its half >= 2, at most `levels` grids.  The smoother is
    red-black Gauss-Seidel if every level's A passes check(radius, colours=2), else 8-colour Gauss-Seidel.  With coefs=
    the ops may have coefficient terms (DESIGN.md section 2.12): each level holds its own coarsened fields, the smoother
    is the diagonal relaxation and the residual goes through the fused coefficient kernel.  Building the hierarchy is
    collective under torchrun, and so are cycle(), update_coefficients() and solve().  The solver never calls
    dd.swap()."""

    def __init__(self, dd: DistributedDomain, u: DataHandle, f: DataHandle, r: DataHandle, op_at: Callable[[int], StencilOp], nu1: int = 2,
                 nu2: int = 2, coarse_sweeps: int = 30, levels: Optional[int] = None, coefs: Optional[Sequence[DataHandle]] = None,
                 coef_kinds: Optional[Sequence[str]] = None):
        """coefs: the coefficient quantities of dd the ops read (field k = coefs[k], every op_at(l) with ncoef equal to
        len(coefs)); coef_kinds: one per field, "x", "y" or "z" for a field on the faces normal to that axis (coarsened by
        the face restriction) or "cell" for a cell-centred field (the 8-cell restriction); by default ("x", "y", "z")
        for three fields.  Each coarse level holds one quantity per field with the fine field's BC on every FIXED face,
        which must be set.  Coefficient ops are smoothed by the diagonal relaxation with omega = 1 and their residual is
        restricted by the fused coefficient kernel; plain ops run as without coefs."""
        if not isinstance(dd, DistributedDomain) or dd.partition_ is None or not dd._plans:
            raise _lib.StencilError("Multigrid: dd must be a realized DistributedDomain")
        for name, h in (("u", u), ("f", f), ("r", r)):
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(dd.dtypes_):
                raise _lib.StencilError(f"Multigrid: {name} must be a DataHandle of dd, not {h!r}")
        if len({u.id, f.id, r.id}) != 3:
            raise _lib.StencilError("Multigrid: u, f and r must be three different quantities")
        dtype = dd.dtypes_[u.id]
        if dtype not in (np.dtype(np.float32), np.dtype(np.float64)) or dd.dtypes_[f.id] != dtype or dd.dtypes_[r.id] != dtype:
            raise _lib.StencilError("Multigrid: u, f and r must all be float32 or all float64")
        coefs = list(coefs) if coefs is not None else []
        if coef_kinds is None:
            coef_kinds = ("x", "y", "z") if len(coefs) == 3 else ()
        coef_kinds = tuple(coef_kinds)
        if len(coefs) > 4:
            raise _lib.StencilError(f"Multigrid: at most 4 coefficient fields, not {len(coefs)}")
        if len(coef_kinds) != len(coefs) or any(k not in COEF_KINDS for k in coef_kinds):
            raise _lib.StencilError(f"Multigrid: coef_kinds must name one of 'x', 'y', 'z', 'cell' per coefficient field, not {coef_kinds!r}")
        for k, h in enumerate(coefs):
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(dd.dtypes_):
                raise _lib.StencilError(f"Multigrid: coefficient {k} must be a DataHandle of dd, not {h!r}")
            if h.id in (u.id, f.id, r.id) or dd.dtypes_[h.id] != dtype:
                raise _lib.StencilError(f"Multigrid: coefficient {k} must be a quantity of u's type other than u, f and r")
        if len({h.id for h in coefs}) != len(coefs):
            raise _lib.StencilError("Multigrid: the coefficient fields must be different quantities")
        if int(nu1) < 0 or int(nu2) < 0 or int(coarse_sweeps) < 1:
            raise _lib.StencilError("Multigrid: nu1 and nu2 must be >= 0 and coarse_sweeps >= 1")
        if levels is not None and int(levels) < 2:
            raise _lib.StencilError("Multigrid: levels must be >= 2 (or None)")
        self.nu1, self.nu2, self.coarse_sweeps = int(nu1), int(nu2), int(coarse_sweeps)
        walls, coef_walls = {}, [{} for _ in coefs]
        for fc in range(6):
            if dd.boundary_[fc // 2] == Boundary.FIXED:
                walls[fc] = coarse_bc(dd.bcs_.get((u.id, fc), BC.NONE()))
                for k, h in enumerate(coefs):
                    bc = dd.bcs_.get((h.id, fc), BC.NONE())
                    if bc.kind == BCKind.NONE:
                        raise _lib.StencilError(f"Multigrid: coefficient {k} needs a boundary condition on every FIXED face (face {FACES[fc]})")
                    coef_walls[k][fc] = bc
        part = dd.partition_
        nlev = level_count([part.subdomain_size(i) for i in part.indices()], levels)
        if nlev < 2:
            raise _lib.StencilError(f"Multigrid: the grid cannot be coarsened once: every subdomain extent must be even and >= 4, "
                                    f"not {[part.subdomain_size(i) for i in part.indices()]}")
        coarse_radius = Radius()
        for d in coarse_radius._r:
            coarse_radius.set_dir(d, dd.radius_.dir(d) if d == (0, 0, 0) else max(1, dd.radius_.dir(d)))
        # each coarse domain partitions its own grid: check now, before any domain is built, that it splits as dd does
        n_sub = len(dd.gpus_) * dd._world.size
        trivial = dd.strategy_ == PlacementStrategy.Trivial
        for l in range(1, nlev):
            size_l = tuple(v >> l for v in dd.size())
            cp = Partition(size_l, coarse_radius, 1, n_sub, trivial=trivial)
            if cp.dim != part.dim or any(tuple(v * (1 << l) for v in cp.subdomain_size(i)) != tuple(part.subdomain_size(i)) for i in part.indices()):
                raise _lib.StencilError(f"Multigrid: the {size_l} grid of level {l} is split as {cp.dim} subdomains, not as dd's {part.dim} "
                                        f"halved {l} times; pass levels={l} or choose a grid whose coarsenings split alike")
        ops = []
        for l in range(nlev):
            A = op_at(l)
            if not isinstance(A, StencilOp) or A.dtype != dtype:
                raise _lib.StencilError(f"Multigrid: op_at({l}) must be a StencilOp in {dtype}, not {A!r}")
            if A.has_aux or (A.has_coef and not coefs):
                raise _lib.StencilError(f"Multigrid: op_at({l}) has coefficient or aux terms; the smoother takes src terms, and coefficient "
                                        "terms only with coefs=")
            if coefs and A.ncoef != len(coefs):
                raise _lib.StencilError(f"Multigrid: op_at({l}) reads {A.ncoef} coefficient fields, but {len(coefs)} were given")
            if A.has_coef and not any(t[0] == 0 and t[1] == (0, 0, 0) for t in A.terms):
                raise _lib.StencilError(f"Multigrid: op_at({l}) has no term at offset (0, 0, 0)")
            if A.reach() > 1:
                raise _lib.StencilError(f"Multigrid: op_at({l}) reaches {A.reach()} cells; the fused residual-restriction takes reach <= 1")
            ops.append(A)
        self.colours = 0
        for m in (2, 8):
            try:
                for l, A in enumerate(ops):
                    A.check(dd.radius_ if l == 0 else coarse_radius, colours=m)
            except _lib.StencilError:
                continue
            self.colours = m
            break
        if not self.colours:
            raise _lib.StencilError("Multigrid: A reads its own colour under both red-black and 8-colour orderings (or leaves the "
                                    "radius); no Gauss-Seidel smoother applies")
        self.levels: List[_Level] = [_Level(dd, u, f, ops[0], coefs)]
        self._walls = {fc: dd.bcs_.get((u.id, fc), BC.NONE()) for fc in walls}  # u's own wall BCs, for cycle(u=, f=)
        self._pairs = {}  # (u, f) ids -> the fine _Level of another pair (cycle(u=, f=))
        self.r = r
        self.coef_kinds = coef_kinds
        self._coef_parity = None
        # every level queues on dd's apply streams, so stream order alone orders the work of consecutive levels
        dd._ensure_apply_streams()
        size = dd.size()
        try:
            for l in range(1, nlev):
                size = tuple(v // 2 for v in size)
                cd = DistributedDomain(*size)
                if dd.gpus_ is not None:
                    cd.set_gpus(dd.gpus_)
                cd.set_placement(dd.strategy_)
                cd.set_methods(dd.flags_)
                cd.set_radius(coarse_radius)
                cu, cf = cd.add_data(dtype, "u"), cd.add_data(dtype, "f")
                ck = [cd.add_data(dtype, f"coef{k}") for k in range(len(coefs))]
                cd.set_boundary(*dd.boundary_)
                for fc, bc in walls.items():
                    cd.set_boundary_condition(cu, FACES[fc], bc)
                for h, w in zip(ck, coef_walls):
                    for fc, bc in w.items():
                        cd.set_boundary_condition(h, FACES[fc], bc)
                cd.realize()
                cd._apply_streams = dd._apply_streams
                self.levels.append(_Level(cd, cu, cf, ops[l], ck))
            for l in range(nlev - 1):
                self.levels[l].dd._check_pairing(self.levels[l + 1].dd, True)
            if coefs:
                self.update_coefficients()
        except Exception:
            self.close()
            raise

    def _smooth(self, L: _Level, sweeps: int) -> None:
        for _ in range(sweeps):
            for c in range(self.colours):
                if L.gs is None:
                    plans = L.dd._apply_plans(L.A, (L.u, "curr"), L.u, (L.f, "curr"), (L.u,), L.coefs, (self.colours, c), omega=1.0)
                else:
                    plans = L.dd._apply_plans(L.gs, (L.u, "curr"), L.u, (L.f, "curr"), (L.u,), colour=(self.colours, c))
                L.dd._run_plans(*plans, queued=True)

    def update_coefficients(self, wait: bool = True) -> None:
        """Re-coarsen every level's coefficient fields from the current fine ones, level by level: face fields by the
        face restriction, cell fields by the 8-cell restriction.  Queued like a cycle, after the work on the caller's
        stream, with one host wait (none with wait=False).  The constructor calls it once; call it again whenever the
        fine fields change.  It then exchanges the fields of every level, fine and coarse: the cycles exchange only the
        vector each call reads at an offset (DESIGN.md section 2.15), never a coefficient field.  A cycle after dd.swap()
        exchanges the fine fields once more, as their curr buffers are then the other allocation."""
        self.levels[0].dd._follow_caller()
        for F, Cl in zip(self.levels[:-1], self.levels[1:]):
            for kf, kc, kind in zip(F.coefs, Cl.coefs, self.coef_kinds):
                F.dd._transfer(Cl.dd, _lib.TRANSFER_RESTRICT, (kc, "curr"), (kf, "curr"), None, False, queued=True, face=COEF_KINDS[kind])
        for L in self.levels:
            if L.coefs:
                L.dd._queue_exchange(L.dd._exchange_sel("Multigrid", tuple(L.coefs), ()))
        self._coef_parity = self.levels[0].dd._parity
        if wait:
            self.wait()

    def _fine_coefs_current(self) -> None:
        """After dd.swap() the fine coefficient fields' curr buffers are the other allocation: exchange them once."""
        L0 = self.levels[0]
        if L0.coefs and self._coef_parity != L0.dd._parity:
            L0.dd._queue_exchange(L0.dd._exchange_sel("Multigrid", tuple(L0.coefs), ()))
            self._coef_parity = L0.dd._parity

    def _vcycle(self, l: int, L: Optional[_Level] = None) -> None:
        L = self.levels[l] if L is None else L
        if l == len(self.levels) - 1:
            self._smooth(L, self.coarse_sweeps)
            return
        self._smooth(L, self.nu1)
        Cl = self.levels[l + 1]
        L.dd._transfer(Cl.dd, _lib.TRANSFER_RESTRICT, (Cl.f, "curr"), (L.u, "curr"), (L.f, "curr"), (L.u,), op=L.res, queued=True,
                       coefs=L.coefs if L.res.has_coef else None)
        Cl.dd._queue_clear(Cl.u)
        self._vcycle(l + 1)
        L.dd._transfer(Cl.dd, _lib.TRANSFER_PROLONG, (L.u, "curr"), (Cl.u, "curr"), (L.u, "curr"), (Cl.u,), queued=True)
        self._smooth(L, self.nu2)

    def _fine_level(self, u: DataHandle, f: DataHandle) -> _Level:
        """The fine level of the pair (u, f): the constructor's, or one that shares A, the coefficient fields and every
        coarse level (checked and built on first use)."""
        L0 = self.levels[0]
        if u is None and f is None:
            return L0
        key = (getattr(u, "id", None), getattr(f, "id", None))
        if key == (L0.u.id, L0.f.id):
            return L0
        if key in self._pairs:
            return self._pairs[key]
        dd = L0.dd
        for name, h in (("u", u), ("f", f)):
            if not isinstance(h, DataHandle) or not 0 <= h.id < len(dd.dtypes_):
                raise _lib.StencilError(f"Multigrid.cycle: {name} must be a DataHandle of dd, not {h!r}")
        if u.id == f.id:
            raise _lib.StencilError("Multigrid.cycle: u and f must be two different quantities")
        dtype = dd.dtypes_[L0.u.id]
        if dd.dtypes_[u.id] != dtype or dd.dtypes_[f.id] != dtype:
            raise _lib.StencilError(f"Multigrid.cycle: u and f must be {dtype} quantities, like the constructor's u")
        if any(h.id in {k.id for k in L0.coefs} for h in (u, f)):
            raise _lib.StencilError("Multigrid.cycle: u and f must not be coefficient fields")
        # the coarse walls were derived from the constructor u's BCs, so the new u must carry the same ones
        for fc, want in self._walls.items():
            got = dd.bcs_.get((u.id, fc), BC.NONE())
            if got != want:
                raise _lib.StencilError(f"Multigrid.cycle: u needs {want!r} on face {FACES[fc]}, the constructor u's BC, not {got!r}")
        L = self._pairs[key] = _Level(dd, u, f, L0.A, L0.coefs)
        return L

    def cycle(self, wait: bool = True, u: Optional[DataHandle] = None, f: Optional[DataHandle] = None) -> None:
        """One V(nu1, nu2) cycle: per level nu1 sweeps, the fused residual-restriction into the coarse f, the coarse u set
        to +0, the recursion, the in-place prolongation u <- u + P e and nu2 sweeps; coarse_sweeps sweeps on the coarsest
        level.  Queued after the work on the caller's stream; returns when the cycle is complete (one host wait), or,
        with wait=False, as soon as it is queued (call wait() before touching u).

        With u= and f=, the cycle runs on that fine-level pair instead of the constructor's, through the same coarse
        levels and coarse coefficient fields: u and f are two different quantities of dd of the constructor u's type,
        not coefficient fields, and u carries the constructor u's BC on every FIXED face (the coarse walls derive from
        it).  The cycle is then the bits of one on a Multigrid built on (u, f).  Give both or neither.
        Each exchange inside a cycle moves only the vector the call reads at an offset (u on each level), so after a cycle
        the ghost cells of the other quantities, the solver's scratch included, are no longer refreshed as a side effect."""
        if (u is None) != (f is None):
            raise _lib.StencilError("Multigrid.cycle: give both u and f, or neither")
        L = self._fine_level(u, f)
        self.levels[0].dd._follow_caller()
        self._fine_coefs_current()
        self._vcycle(0, L)
        if wait:
            self.wait()

    def wait(self) -> None:
        """Return when every queued cycle is complete."""
        wait_queued([L.dd for L in self.levels])

    def residual_norm(self) -> float:
        """||f - A u||_2 over dd's compute region: the residual into r (apply) and an exact reduction, so every rank and
        every partition reach the same value."""
        L = self.levels[0]
        L.dd.apply(L.res, (self.r, "curr"), L.u, (L.f, "curr"), coefs=L.coefs if L.res.has_coef else None)
        return L.dd.reduce(self.r, "curr", exact=True).l2()

    def solve(self, rtol: float, max_cycles: int) -> List[float]:
        """Cycles until ||f - A u||_2 <= rtol ||f||_2 or max_cycles cycles; returns the residual norm before the first
        cycle and after each.  Every rank calls it."""
        L = self.levels[0]
        target = float(rtol) * L.dd.reduce(L.f, "curr", exact=True).l2()
        hist = [self.residual_norm()]
        while hist[-1] > target and len(hist) - 1 < int(max_cycles):
            self.cycle()
            hist.append(self.residual_norm())
        return hist

    def close(self) -> None:
        """Release the coarse domains and dd's transfer plans to them."""
        dd = self.levels[0].dd
        coarse = [L.dd for L in self.levels[1:]]
        for fine in [dd] + coarse[:-1]:
            for key in [k for k in fine._transfer_plans if any(k[0] is cd for cd in coarse)]:
                for per_dom in fine._transfer_plans.pop(key):
                    for p in per_dom:
                        p.destroy()
            fine._paired = {k for k in fine._paired if not any(k[0] is cd for cd in coarse)}
        for cd in coarse:
            cd.close()
        self.levels = self.levels[:1]
        self._pairs = {}
