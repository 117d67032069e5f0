"""numpy restatement of coloured application (include/stencil_b200.h, sb_stencil_cplan_create; DESIGN.md section 2.9)
and of the relaxation table sb_stencil_relax, for the CPU and GPU tests.

A colouring m is 1, 2 or 8; a cell's colour comes from its GLOBAL coordinates: 0 for m = 1, (x + y + z) mod 2 for
m = 2, (x mod 2) + 2 (y mod 2) + 4 (z mod 2) for m = 8.  A coloured launch evaluates the op on the buffers as they were
before it (the ghost cells filled first, by periodic wrap or by tests/bc_oracle.py) and writes only the cells of the box
of colour c; every other cell keeps its bits.  Arrays are [z, y, x]; boxes are (lo, ext) in (x, y, z) allocation
coordinates; origin is the global coordinate of allocation element (0, 0, 0)."""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np

import stencil_op_oracle as so
import vstencil_oracle as vo


def colours(shape, origin, m: int) -> np.ndarray:
    """The colour of every element of a [z, y, x] array whose element (0, 0, 0) has global coordinate origin."""
    z, y, x = np.indices(shape)
    gx, gy, gz = x + origin[0], y + origin[1], z + origin[2]
    if m == 1:
        return np.zeros(shape, np.int64)
    if m == 2:
        return (gx + gy + gz) & 1
    return (gx & 1) | ((gy & 1) << 1) | ((gz & 1) << 2)


def colour_ok(terms, m: int) -> bool:
    """The colour condition: every src term with o != 0 reads a cell of another colour (m = 2: o_x + o_y + o_z odd;
    m = 8: some o_a odd)."""
    for t in terms:
        s, o = t[0], t[1]
        if s != 0 or not any(o) or m == 1:
            continue
        if m == 2 and sum(o) % 2 == 0:
            return False
        if m == 8 and not any(v % 2 for v in o):
            return False
    return True


def box_mask(shape, lo, ext, origin, m: int, c: int) -> np.ndarray:
    """The cells of the box [lo, lo + ext) of colour c."""
    inbox = np.zeros(shape, bool)
    so._view(inbox, lo, ext, (0, 0, 0))[...] = True
    return inbox & (colours(shape, origin, m) == c)


def apply_box(terms, src: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray], dst: np.ndarray, lo, ext, origin, m: int,
              c: int) -> None:
    """dst = the coloured op, in place; dst may be src or aux (the op is evaluated on a snapshot taken before)."""
    new = dst.copy()
    vo.apply_box(terms, src.copy(), None if aux is None else aux.copy(), [k.copy() for k in coefs], new, lo, ext)
    mk = box_mask(dst.shape, lo, ext, origin, m, c)
    dst[mk] = new[mk]


def apply_periodic(terms, u: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray], dst: np.ndarray, m: int, c: int) -> np.ndarray:
    """The coloured op on a periodic [z, y, x] grid with no ghost cells (global origin 0): the cells of colour c take
    op(u), the others dst's values.  In place, dst is u."""
    new = vo.apply_periodic(terms, u, aux, coefs)
    return np.where(colours(u.shape, (0, 0, 0), m) == c, new, dst)


def sweep_loop(terms, u: np.ndarray, aux: Optional[np.ndarray], lo, ext, origin, m: int, c: int) -> None:
    """The literal Gauss-Seidel loop: the box's cells of colour c in lexicographic (z, y, x) order, each updated in
    place by the op reading u as it is at that moment (numpy scalars, every operation rounded)."""
    T = u.dtype.type
    for z in range(lo[2], lo[2] + ext[2]):
        for y in range(lo[1], lo[1] + ext[1]):
            for x in range(lo[0], lo[0] + ext[0]):
                gx, gy, gz = x + origin[0], y + origin[1], z + origin[2]
                col = 0 if m == 1 else (gx + gy + gz) & 1 if m == 2 else (gx & 1) | (gy & 1) << 1 | (gz & 1) << 2
                if col != c:
                    continue
                acc = None
                for s, o, w in terms:
                    v = u[z + o[2], y + o[1], x + o[0]] if s == 0 else aux[z, y, x]
                    mm = T(T(w) * T(v))
                    acc = mm if acc is None else T(acc + mm)
                u[z, y, x] = acc


def relax(A, omega: float):
    """sb_stencil_relax restated: (src, 0, 1 - omega), each off-centre src term (src, o, (-omega * w) / a_c) in A's order,
    then (aux, 0, omega / a_c); None where the C call refuses A or omega."""
    omega = float(omega)
    if not np.isfinite(omega) or any(t[0] != 0 for t in A):
        return None
    centre = [t for t in A if not any(t[1])]
    if len(centre) != 1 or centre[0][2] == 0.0:
        return None
    ac = float(centre[0][2])
    out = [(0, (0, 0, 0), 1.0 - omega)]
    out += [(0, tuple(t[1]), (-omega * float(t[2])) / ac) for t in A if any(t[1])]
    return out + [(1, (0, 0, 0), omega / ac)]


def helmholtz(h: float, sigma: float):
    """A of -lap(u) + sigma u = f (order-2 Laplacian, spacing h on every axis): the centre first."""
    lap = so.laplacian(2, (h, h, h))
    return [(0, (0, 0, 0), -lap[0][2] + sigma)] + [(0, o, -w) for _, o, w in lap[1:]]
