"""numpy restatement of the fused residual-restriction (include/stencil_b200.h, sb_transfer_oplan_create; DESIGN.md
section 2.11) and of the cycle stencil_b200.Multigrid runs.

Arrays are [z, y, x]; origin is the global coordinate of element (0, 0, 0); boxes are [lo, hi) in global coordinates.
Every multiply and add is one numpy operation in the array's dtype, so each is rounded separately, as on the GPU."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import colour_oracle as co
import stencil_op_oracle as so
import transfer_oracle as to


def restrict_op_box(dst: np.ndarray, dst_origin, terms, src: np.ndarray, aux: Optional[np.ndarray], src_origin, lo, hi) -> None:
    """dst[I] = the restriction of op(src, aux) over the coarse cells I of [lo, hi): the op on the fine footprint
    [2 lo, 2 hi) into a scratch array, then transfer_oracle.restrict_box (aux shares src's layout)."""
    n = [hi[a] - lo[a] for a in range(3)]
    if min(n) <= 0:
        return
    scratch = np.full(src.shape, np.nan, dst.dtype)  # src's layout
    so.apply_box(terms, src, aux, scratch, [2 * lo[a] - src_origin[a] for a in range(3)], [2 * v for v in n])
    to.restrict_box(dst, dst_origin, scratch, src_origin, lo, hi)


def restrict_op_loop(dst: np.ndarray, dst_origin, terms, src: np.ndarray, aux: Optional[np.ndarray], src_origin, lo, hi) -> None:
    """The same rule one coarse cell at a time with numpy scalars: for each of the eight fine cells in the restriction's
    order, the op in list order, then the running sum and T(0.125) times it."""
    T = dst.dtype.type
    for z in range(lo[2], hi[2]):
        for y in range(lo[1], hi[1]):
            for x in range(lo[0], hi[0]):
                acc = None
                for d in to.RESTRICT_ORDER:
                    p = (2 * z + d[2] - src_origin[2], 2 * y + d[1] - src_origin[1], 2 * x + d[0] - src_origin[0])
                    v = None
                    for s, o, w in terms:
                        val = src[p[0] + o[2], p[1] + o[1], p[2] + o[0]] if s == 0 else aux[p]
                        m = T(T(w) * T(val))
                        v = m if v is None else T(v + m)
                    acc = v if acc is None else T(acc + v)
                dst[z - dst_origin[2], y - dst_origin[1], x - dst_origin[0]] = T(T(0.125) * acc)


# ----------------------------------------------------------------------------------------------- the solver's cycle
Wall = Tuple[str, float]  # ("odd", c) or ("even", 0)


def fill_ghosts(u: np.ndarray, periodic: Sequence[bool], walls: Dict[int, Wall]) -> None:
    """The one-cell ghost layer of a padded [z, y, x] array: periodic axes wrap (the exchange), then on the walled axes in
    order x, y, z, face - then +, ODD(c): T(2) * T(c) - mirror, EVEN: the mirror (tests/bc_oracle.py)."""
    T = u.dtype.type
    for a in range(3):
        if periodic[a]:
            ax = 2 - a
            u[(slice(None),) * ax + (0,)] = u[(slice(None),) * ax + (-2,)]
            u[(slice(None),) * ax + (-1,)] = u[(slice(None),) * ax + (1,)]
    for a in range(3):
        if periodic[a]:
            continue
        ax = 2 - a
        for side, g, m in ((0, 0, 1), (1, -1, -2)):
            kind, c = walls[2 * a + side]
            mirror = u[(slice(None),) * ax + (m,)]
            u[(slice(None),) * ax + (g,)] = T(2) * T(c) - mirror if kind == "odd" else mirror


def coarse_walls(walls: Dict[int, Wall]) -> Dict[int, Wall]:
    """ODD(c) -> ODD(0), EVEN -> EVEN (stencil_b200.multigrid.coarse_bc)."""
    return {f: (k, 0.0) for f, (k, _) in walls.items()}


class Level:
    """One grid: padded u, f and r (ghost width 1, origin (-1, -1, -1)), the operator A (a term list), its Gauss-Seidel
    update (relax(A, 1)) and the residual op; m colours."""

    def __init__(self, size, A, dtype, periodic: Sequence[bool], walls: Dict[int, Wall], m: int = 2):
        self.size, self.periodic, self.walls, self.m = tuple(size), tuple(periodic), dict(walls), m
        shape = tuple(n + 2 for n in self.size[::-1])
        self.u, self.f, self.r = (np.zeros(shape, dtype) for _ in range(3))
        self.A = A
        self.gs = co.relax(A, 1.0)
        self.res = to.residual_terms(A)

    def interior(self, a: np.ndarray) -> np.ndarray:
        return a[1:-1, 1:-1, 1:-1]

    def smooth(self, sweeps: int) -> None:
        for _ in range(sweeps):
            for c in range(self.m):
                fill_ghosts(self.u, self.periodic, self.walls)
                co.apply_box(self.gs, self.u, self.f, [], self.u, (1, 1, 1), self.size, (-1, -1, -1), self.m, c)

    def residual_norm(self) -> float:
        fill_ghosts(self.u, self.periodic, self.walls)
        so.apply_box(self.res, self.u, self.f, self.r, (1, 1, 1), self.size)
        return float(np.linalg.norm(self.interior(self.r).astype(np.float64)))


def hierarchy(size, levels: int, A_at, dtype, periodic: Sequence[bool], walls: Dict[int, Wall], m: int = 2) -> List[Level]:
    """levels grids from size down by 2 per axis; A_at(l) the term list of level l; walls on the finest, coarse_walls
    below."""
    out = []
    for l in range(levels):
        out.append(Level(size, A_at(l), dtype, periodic, walls if l == 0 else coarse_walls(walls), m))
        size = tuple(n // 2 for n in size)
    return out


def vcycle(lv: List[Level], l: int = 0, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30) -> None:
    """Multigrid.cycle(): the fused residual-restriction into the coarse f, the coarse u set to +0."""
    L = lv[l]
    if l == len(lv) - 1:
        L.smooth(coarse_sweeps)
        return
    L.smooth(nu1)
    Cl = lv[l + 1]
    fill_ghosts(L.u, L.periodic, L.walls)
    restrict_op_box(Cl.f, (-1, -1, -1), L.res, L.u, L.f, (-1, -1, -1), (0, 0, 0), Cl.size)
    Cl.u[...] = 0
    vcycle(lv, l + 1, nu1, nu2, coarse_sweeps)
    fill_ghosts(Cl.u, Cl.periodic, Cl.walls)
    to.prolong_box(L.u, (-1, -1, -1), Cl.u, (-1, -1, -1), (0, 0, 0), L.size, aux=L.u)
    L.smooth(nu2)
