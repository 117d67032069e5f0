"""numpy restatement of multigrid for variable-coefficient operators (include/stencil_b200.h: sb_stencil_dplan_create,
sb_transfer_fplan_create, sb_transfer_voplan_create; DESIGN.md section 2.12) and of the cycle stencil_b200.Multigrid
runs with coefficient fields.

Arrays are [z, y, x].  Boxes are (lo, ext) in (x, y, z) allocation coordinates for the diagonal rule (as in
tests/colour_oracle.py) and [lo, hi) in global coordinates for the transfers (as in tests/transfer_oracle.py).  Every
operation is one numpy operation in the array's dtype, so each is rounded separately, as on the GPU."""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

import colour_oracle as co
import mg_oracle as mo
import transfer_oracle as to
import vstencil_oracle as vo
from stencil_op_oracle import _view


# --------------------------------------------------------------------------------------------- diagonal relaxation
def diag_box(terms, omega: float, u: np.ndarray, f: np.ndarray, coefs: Sequence[np.ndarray], dst: np.ndarray, lo, ext, origin, m: int,
             c: int) -> None:
    """dst = u + T(omega) ((f - A u) / d) on the cells of the box of colour c under m, evaluated on a snapshot of the
    buffers taken before (dst may be u or f); d = the sum of the factors of A's terms at offset 0, in list order."""
    T = dst.dtype.type
    u0, f0, ks = u.copy(), f.copy(), [k.copy() for k in coefs]
    acc = d = None
    for t in terms:
        s, o, w, k, cc = vo.split(t)
        assert s == 0
        wt = T(w) if k < 0 else np.multiply(T(w), _view(ks[k], lo, ext, cc), dtype=dst.dtype)
        mm = np.multiply(wt, _view(u0, lo, ext, o), dtype=dst.dtype)
        acc = mm if acc is None else np.add(acc, mm, dtype=dst.dtype)
        if not any(o):
            d = wt if d is None else np.add(d, wt, dtype=dst.dtype)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.divide(np.subtract(_view(f0, lo, ext, (0, 0, 0)), acc, dtype=dst.dtype), d, dtype=dst.dtype)
    new = dst.copy()
    _view(new, lo, ext, (0, 0, 0))[...] = np.add(_view(u0, lo, ext, (0, 0, 0)), np.multiply(T(omega), q, dtype=dst.dtype), dtype=dst.dtype)
    mk = co.box_mask(dst.shape, lo, ext, origin, m, c)
    dst[mk] = new[mk]


def diag_loop(terms, omega: float, u: np.ndarray, f: np.ndarray, coefs: Sequence[np.ndarray], dst: np.ndarray, lo, ext, origin, m: int,
              c: int) -> None:
    """The same rule one cell at a time with numpy scalars (out of place: dst is neither u nor f)."""
    T = dst.dtype.type
    for z in range(lo[2], lo[2] + ext[2]):
        for y in range(lo[1], lo[1] + ext[1]):
            for x in range(lo[0], lo[0] + ext[0]):
                gx, gy, gz = x + origin[0], y + origin[1], z + origin[2]
                col = 0 if m == 1 else (gx + gy + gz) & 1 if m == 2 else (gx & 1) | (gy & 1) << 1 | (gz & 1) << 2
                if col != c:
                    continue
                a = d = None
                for t in terms:
                    s, o, w, k, cc = vo.split(t)
                    wt = T(w) if k < 0 else T(T(w) * coefs[k][z + cc[2], y + cc[1], x + cc[0]])
                    mm = T(wt * u[z + o[2], y + o[1], x + o[0]])
                    a = mm if a is None else T(a + mm)
                    if not any(o):
                        d = wt if d is None else T(d + wt)
                with np.errstate(divide="ignore", invalid="ignore"):
                    dst[z, y, x] = T(u[z, y, x] + T(T(omega) * T(T(f[z, y, x] - a) / d)))


# --------------------------------------------------------------------------------------------- face restriction
def other_axes(axis: int) -> Tuple[int, int]:
    b, c = [a for a in range(3) if a != axis]
    return b, c


def face_restrict_box(dst: np.ndarray, dst_origin, src: np.ndarray, src_origin, axis: int, lo, hi) -> None:
    """dst[I] = T(0.25) * (((F(2I) + F(2I + e_b)) + F(2I + e_c)) + F(2I + e_b + e_c)), b < c the axes other than axis."""
    T = dst.dtype.type
    n = [hi[a] - lo[a] for a in range(3)]
    if min(n) <= 0:
        return
    b, c = other_axes(axis)
    acc = None
    for st in ((), (b,), (c,), (b, c)):
        f = src[to._sl([2 * lo[a] + (1 if a in st else 0) for a in range(3)], n, src_origin, 2)]
        acc = f.copy() if acc is None else acc + f
    dst[to._sl(lo, n, dst_origin)] = T(0.25) * acc


def face_restrict_loop(dst: np.ndarray, dst_origin, src: np.ndarray, src_origin, axis: int, lo, hi) -> None:
    T = dst.dtype.type
    b, c = other_axes(axis)
    for z in range(lo[2], hi[2]):
        for y in range(lo[1], hi[1]):
            for x in range(lo[0], hi[0]):
                p = [2 * x - src_origin[0], 2 * y - src_origin[1], 2 * z - src_origin[2]]
                vals = []
                for st in ((), (b,), (c,), (b, c)):
                    q = [p[a] + (1 if a in st else 0) for a in range(3)]
                    vals.append(src[q[2], q[1], q[0]])
                dst[z - dst_origin[2], y - dst_origin[1], x - dst_origin[0]] = T(T(0.25) * T(T(T(vals[0] + vals[1]) + vals[2]) + vals[3]))


# --------------------------------------------------------------------------------------------- fused, with coefficients
def restrict_vop_box(dst: np.ndarray, dst_origin, terms, src: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray], src_origin,
                     lo, hi) -> None:
    """dst[I] = the restriction of op(src, aux, coefs) over the coarse cells I of [lo, hi): the op on the fine footprint
    into a scratch array (vstencil_oracle), then transfer_oracle.restrict_box; aux and coefs share src's layout."""
    n = [hi[a] - lo[a] for a in range(3)]
    if min(n) <= 0:
        return
    scratch = np.full(src.shape, np.nan, dst.dtype)
    vo.apply_box(terms, src, aux, coefs, scratch, [2 * lo[a] - src_origin[a] for a in range(3)], [2 * v for v in n])
    to.restrict_box(dst, dst_origin, scratch, src_origin, lo, hi)


def restrict_vop_loop(dst: np.ndarray, dst_origin, terms, src: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray], src_origin,
                      lo, hi) -> None:
    T = dst.dtype.type
    for z in range(lo[2], hi[2]):
        for y in range(lo[1], hi[1]):
            for x in range(lo[0], hi[0]):
                acc = None
                for dd in to.RESTRICT_ORDER:
                    p = (2 * z + dd[2] - src_origin[2], 2 * y + dd[1] - src_origin[1], 2 * x + dd[0] - src_origin[0])
                    v = None
                    for t in terms:
                        s, o, w, k, c = vo.split(t)
                        val = src[p[0] + o[2], p[1] + o[1], p[2] + o[0]] if s == 0 else aux[p]
                        wt = T(w) if k < 0 else T(T(w) * coefs[k][p[0] + c[2], p[1] + c[1], p[2] + c[0]])
                        mm = T(wt * T(val))
                        v = mm if v is None else T(v + mm)
                    acc = v if acc is None else T(acc + v)
                dst[z - dst_origin[2], y - dst_origin[1], x - dst_origin[0]] = T(T(0.125) * acc)


def vresidual_terms(A) -> list:
    """r = f - A u: (aux, 0, 1), then each term of A with its weight negated and its coefficient kept."""
    out = [(1, (0, 0, 0), 1.0)]
    for t in A:
        s, o, w, k, c = vo.split(t)
        out.append((0, tuple(o), -float(w), k, tuple(c)) if k >= 0 else (0, tuple(o), -float(w)))
    return out


def helmholtz_div_grad(h: float, sigma_field: bool = False, sigma: float = 0.0) -> list:
    """-div(kappa grad u) (+ sigma u): sb_stencil_div_grad negated, then (src, 0, 1, field 3) for a cell field sigma or
    (src, 0, sigma) for a constant."""
    A = [(0, o, -w, k, c) for _, o, w, k, c in vo.div_grad((h, h, h))]
    if sigma_field:
        A.append((0, (0, 0, 0), 1.0, 3, (0, 0, 0)))
    elif sigma:
        A.append((0, (0, 0, 0), float(sigma)))
    return A


# --------------------------------------------------------------------------------------------- the solver's cycle
Wall = Tuple[str, float]  # ("odd", c), ("even", 0) or ("value", c)
KINDS = {"x": 0, "y": 1, "z": 2, "cell": -1}


def fill_ghosts(u: np.ndarray, periodic: Sequence[bool], walls: Dict[int, Wall]) -> None:
    """mg_oracle.fill_ghosts with VALUE walls as well (ghost = T(c))."""
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
            if kind == "odd":
                u[(slice(None),) * ax + (g,)] = T(2) * T(c) - mirror
            elif kind == "even":
                u[(slice(None),) * ax + (g,)] = mirror
            else:
                u[(slice(None),) * ax + (g,)] = T(c)


class Level:
    """One grid: padded u, f, r and coefficient fields (ghost width 1, origin (-1, -1, -1)); A (a term list) smoothed by
    the diagonal relaxation with omega = 1 under m colours."""

    def __init__(self, size, A, dtype, periodic, walls, coef_walls: List[Dict[int, Wall]], m: int = 2):
        self.size, self.periodic, self.walls, self.coef_walls, self.m = tuple(size), tuple(periodic), dict(walls), coef_walls, m
        shape = tuple(n + 2 for n in self.size[::-1])
        self.u, self.f, self.r = (np.zeros(shape, dtype) for _ in range(3))
        self.k = [np.zeros(shape, dtype) for _ in coef_walls]
        self.A = A
        self.res = vresidual_terms(A)

    def interior(self, a: np.ndarray) -> np.ndarray:
        return a[1:-1, 1:-1, 1:-1]

    def fill(self) -> None:
        fill_ghosts(self.u, self.periodic, self.walls)
        for k, w in zip(self.k, self.coef_walls):
            fill_ghosts(k, self.periodic, w)

    def smooth(self, sweeps: int) -> None:
        for _ in range(sweeps):
            for c in range(self.m):
                self.fill()
                diag_box(self.A, 1.0, self.u, self.f, self.k, self.u, (1, 1, 1), self.size, (-1, -1, -1), self.m, c)

    def residual_norm(self) -> float:
        self.fill()
        vo.apply_box(self.res, self.u, self.f, self.k, self.r, (1, 1, 1), self.size)
        return float(np.linalg.norm(self.interior(self.r).astype(np.float64)))


def hierarchy(size, levels: int, A_at, dtype, periodic, walls: Dict[int, Wall], coef_walls: List[Dict[int, Wall]], m: int = 2) -> List[Level]:
    """levels grids from size down by 2 per axis; A_at(l) the term list of level l; u's walls on the finest and
    mg_oracle.coarse_walls below; every level's coefficient fields keep the fine fields' walls."""
    out = []
    for l in range(levels):
        out.append(Level(size, A_at(l), dtype, periodic, walls if l == 0 else mo.coarse_walls(walls), coef_walls, m))
        size = tuple(n // 2 for n in size)
    return out


def update_coefficients(lv: List[Level], kinds: Sequence[str]) -> None:
    """Multigrid.update_coefficients(): each level's fields from the level above, face fields by face_restrict_box and
    cell fields by the 8-cell restriction."""
    for l in range(len(lv) - 1):
        F, Cl = lv[l], lv[l + 1]
        for kf, kc, kind in zip(F.k, Cl.k, kinds):
            if KINDS[kind] >= 0:
                face_restrict_box(kc, (-1, -1, -1), kf, (-1, -1, -1), KINDS[kind], (0, 0, 0), Cl.size)
            else:
                to.restrict_box(kc, (-1, -1, -1), kf, (-1, -1, -1), (0, 0, 0), Cl.size)


def vcycle(lv: List[Level], l: int = 0, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30) -> None:
    """Multigrid.cycle() with coefficient fields."""
    L = lv[l]
    if l == len(lv) - 1:
        L.smooth(coarse_sweeps)
        return
    L.smooth(nu1)
    Cl = lv[l + 1]
    L.fill()
    restrict_vop_box(Cl.f, (-1, -1, -1), L.res, L.u, L.f, L.k, (-1, -1, -1), (0, 0, 0), Cl.size)
    Cl.u[...] = 0
    vcycle(lv, l + 1, nu1, nu2, coarse_sweeps)
    fill_ghosts(Cl.u, Cl.periodic, Cl.walls)
    to.prolong_box(L.u, (-1, -1, -1), Cl.u, (-1, -1, -1), (0, 0, 0), L.size, aux=L.u)
    L.smooth(nu2)


# --------------------------------------------------------------------------------------------- test problems
def kappa_faces(size, h: float, kind: str, dtype) -> List[np.ndarray]:
    """Padded face fields kx, ky, kz on a grid of size (nx, ny, nz) and spacing h (origin (-1, -1, -1)): field a at cell p
    is kappa at the face between p - e_a and p, x_f = p_a h on axis a and cell centres on the others.  kind "smooth":
    exp(0.5 sin(2 pi x) sin(2 pi y) sin(2 pi z)) (contrast about e on the unit cube); "jump": 1000 inside the cube
    [1/4, 3/4)^3, else 1 (aligned with every grid of the unit cube down to 4^3)."""
    size = (size,) * 3 if np.isscalar(size) else tuple(size)
    out = []
    for a in range(3):
        coords = []
        for b in range(3):
            idx = np.arange(-1, size[b] + 1, dtype=np.float64)
            c = idx * h if b == a else (idx + 0.5) * h
            coords.append(c)
        Z, Y, X = np.meshgrid(coords[2], coords[1], coords[0], indexing="ij")
        if kind == "smooth":
            k = np.exp(0.5 * np.sin(2 * np.pi * X) * np.sin(2 * np.pi * Y) * np.sin(2 * np.pi * Z))
        else:
            # a face is inside when both cells it separates are: on its own axis strictly between 1/4 and 3/4
            inside = [((V > 0.25) & (V < 0.75)) if b == a else ((V >= 0.25) & (V < 0.75)) for b, V in enumerate((X, Y, Z))]
            k = np.where(inside[0] & inside[1] & inside[2], 1000.0, 1.0)
        out.append(k.astype(dtype))
    return out
