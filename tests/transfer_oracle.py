"""numpy restatement of the multigrid transfers (include/stencil_b200.h, sb_transfer_*; DESIGN.md section 2.10), and a
V-cycle composed from it, tests/colour_oracle.py and the ODD / periodic ghost rule of tests/bc_oracle.py.

Arrays are [z, y, x]; origin is the global coordinate of element (0, 0, 0); boxes are [lo, hi) in global coordinates.
Every multiply and add is one numpy operation in the array's dtype, so each is rounded separately, as on the GPU."""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

import colour_oracle as co
import vstencil_oracle as vo

RESTRICT_ORDER = [(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0), (0, 0, 1), (1, 0, 1), (0, 1, 1), (1, 1, 1)]
# (weight numerator over 64, which axes step to the side s) in the order of the prolongation rule
PROLONG_ORDER = [(27, (0, 0, 0)), (9, (1, 0, 0)), (9, (0, 1, 0)), (9, (0, 0, 1)), (3, (1, 1, 0)), (3, (1, 0, 1)), (3, (0, 1, 1)), (1, (1, 1, 1))]


def _sl(lo, n, origin, step=1):
    return tuple(slice(lo[a] - origin[a], lo[a] - origin[a] + step * n[a], step) for a in (2, 1, 0))


def restrict_box(dst: np.ndarray, dst_origin, src: np.ndarray, src_origin, lo, hi) -> None:
    """dst[I] = T(0.125) * (the 8 fine cells 2I + d summed in RESTRICT_ORDER) for the coarse cells I of [lo, hi)."""
    T = dst.dtype.type
    n = [hi[a] - lo[a] for a in range(3)]
    if min(n) <= 0:
        return
    acc = None
    for d in RESTRICT_ORDER:
        f = src[_sl([2 * lo[a] + d[a] for a in range(3)], n, src_origin, 2)]
        acc = f.copy() if acc is None else acc + f
    dst[_sl(lo, n, dst_origin)] = T(0.125) * acc


def prolong_box(dst: np.ndarray, dst_origin, src: np.ndarray, src_origin, lo, hi, aux: Optional[np.ndarray] = None) -> None:
    """dst[p] = aux[p] + acc (or acc) for the fine cells p of [lo, hi), acc the trilinear rule; aux has dst's layout and
    may be dst."""
    T = dst.dtype.type
    n = [hi[a] - lo[a] for a in range(3)]
    if min(n) <= 0:
        return
    P, S = [], []
    for a in range(3):
        p = np.arange(lo[a], hi[a])
        P.append(p // 2 - src_origin[a])  # floor
        S.append(np.where(p % 2 == 1, 1, -1))
    acc = None
    for w, st in PROLONG_ORDER:
        ix = [P[a] + st[a] * S[a] for a in range(3)]
        m = T(w / 64.0) * src[np.ix_(ix[2], ix[1], ix[0])]
        acc = m if acc is None else acc + m
    box = _sl(lo, n, dst_origin)
    dst[box] = acc if aux is None else aux[box] + acc


def restrict_loop(dst, dst_origin, src, src_origin, lo, hi) -> None:
    """restrict_box one coarse cell at a time with numpy scalars."""
    T = dst.dtype.type
    for z in range(lo[2], hi[2]):
        for y in range(lo[1], hi[1]):
            for x in range(lo[0], hi[0]):
                acc = None
                for d in RESTRICT_ORDER:
                    v = src[2 * z + d[2] - src_origin[2], 2 * y + d[1] - src_origin[1], 2 * x + d[0] - src_origin[0]]
                    acc = v if acc is None else T(acc + v)
                dst[z - dst_origin[2], y - dst_origin[1], x - dst_origin[0]] = T(T(0.125) * acc)


def prolong_loop(dst, dst_origin, src, src_origin, lo, hi, aux=None) -> None:
    """prolong_box one fine cell at a time with numpy scalars."""
    T = dst.dtype.type
    for z in range(lo[2], hi[2]):
        for y in range(lo[1], hi[1]):
            for x in range(lo[0], hi[0]):
                p = (x, y, z)
                par = [p[a] // 2 for a in range(3)]
                s = [1 if p[a] % 2 else -1 for a in range(3)]
                acc = None
                for w, st in PROLONG_ORDER:
                    q = [par[a] + st[a] * s[a] - src_origin[a] for a in range(3)]
                    m = T(T(w / 64.0) * src[q[2], q[1], q[0]])
                    acc = m if acc is None else T(acc + m)
                at = (z - dst_origin[2], y - dst_origin[1], x - dst_origin[0])
                dst[at] = acc if aux is None else T(aux[at] + acc)


# ----------------------------------------------------------------------------------------------- a V(nu1, nu2) cycle
def fill_ghosts(u: np.ndarray, periodic: Sequence[bool]) -> None:
    """The one-cell ghost layer of a padded [z, y, x] array: periodic axes wrap (the exchange), then on the walled axes in
    order x, y, z the ODD(0) rule v = T(2) * T(0) - mirror (bc_oracle.apply_regions)."""
    T = u.dtype.type
    for a in range(3):
        if periodic[a]:
            ax = 2 - a
            u[(slice(None),) * ax + (0,)] = u[(slice(None),) * ax + (-2,)]
            u[(slice(None),) * ax + (-1,)] = u[(slice(None),) * ax + (1,)]
    for a in range(3):
        if not periodic[a]:
            ax = 2 - a
            u[(slice(None),) * ax + (0,)] = T(2) * T(0) - u[(slice(None),) * ax + (1,)]
            u[(slice(None),) * ax + (-1,)] = T(2) * T(0) - u[(slice(None),) * ax + (-2,)]


def residual_terms(A) -> list:
    """r = f - A u as one op: (aux, 0, 1), then each term of A with its weight negated."""
    return [(1, (0, 0, 0), 1.0)] + [(0, tuple(o), -w) for _, o, w in A]


ZERO_TERMS = [(0, (0, 0, 0), 0.0)]  # u = 0 * f: how a cycle clears the coarse correction with one apply


class Level:
    """One grid of a cycle: padded u, f and r (ghost width 1, origin (-1, -1, -1)), its operator A = -lap + sigma on
    spacing h, the red-black Gauss-Seidel update and the residual op."""

    def __init__(self, size, h: float, sigma: float, dtype, periodic: Sequence[bool]):
        self.size, self.periodic = tuple(size), tuple(periodic)
        shape = tuple(n + 2 for n in self.size[::-1])
        self.u, self.f, self.r = (np.zeros(shape, dtype) for _ in range(3))
        self.A = co.helmholtz(h, sigma)
        self.gs = co.relax(self.A, 1.0)
        self.res = residual_terms(self.A)

    def interior(self, a: np.ndarray) -> np.ndarray:
        return a[1:-1, 1:-1, 1:-1]

    def smooth(self, sweeps: int) -> None:
        for _ in range(sweeps):
            for c in range(2):
                fill_ghosts(self.u, self.periodic)
                co.apply_box(self.gs, self.u, self.f, [], self.u, (1, 1, 1), self.size, (-1, -1, -1), 2, c)

    def residual(self) -> None:
        fill_ghosts(self.u, self.periodic)
        vo.apply_box(self.res, self.u, self.f, [], self.r, (1, 1, 1), self.size)


def hierarchy(size, levels: int, sigma: float, dtype, periodic: Sequence[bool]) -> List[Level]:
    """levels grids from size down by 2 per axis; spacing 1 / n_x on the finest, doubled per level."""
    out, h = [], 1.0 / size[0]
    for _ in range(levels):
        out.append(Level(size, h, sigma, dtype, periodic))
        size, h = tuple(n // 2 for n in size), 2 * h
    return out


def vcycle(lv: List[Level], l: int = 0, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30) -> None:
    L = lv[l]
    if l == len(lv) - 1:
        L.smooth(coarse_sweeps)
        return
    L.smooth(nu1)
    L.residual()
    C = lv[l + 1]
    restrict_box(C.f, (-1, -1, -1), L.r, (-1, -1, -1), (0, 0, 0), C.size)
    vo.apply_box(ZERO_TERMS, C.f, None, [], C.u, (1, 1, 1), C.size)
    vcycle(lv, l + 1, nu1, nu2, coarse_sweeps)
    fill_ghosts(C.u, C.periodic)
    prolong_box(L.u, (-1, -1, -1), C.u, (-1, -1, -1), (0, 0, 0), L.size, aux=L.u)
    L.smooth(nu2)


def residual_norm(L: Level) -> float:
    L.residual()
    return float(np.linalg.norm(L.interior(L.r).astype(np.float64)))
