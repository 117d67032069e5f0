"""numpy restatement of the linear stencil rule of include/stencil_b200.h (sb_stencil_*), for the CPU and GPU tests.

An op is a list of terms (source, (dx, dy, dz), weight): source 0 reads src at p + o, source 1 reads aux at p.  For
every cell p of a box, in the array's type T, every multiply and every add rounded separately, in list order:
    acc = T(w_0) * S_0(p + o_0);  acc = acc + T(w_k) * S_k(p + o_k);  dst[p] = acc
Arrays are [z, y, x]; boxes are (lo, ext) in (x, y, z) allocation coordinates."""
from __future__ import annotations

from fractions import Fraction
from typing import List, Optional, Sequence, Tuple

import numpy as np

Term = Tuple[int, Tuple[int, int, int], float]

# c_0 .. c_R of the central second difference, exact
LAPLACIAN_COEFFS = {
    2: [Fraction(-2), Fraction(1)],
    4: [Fraction(-5, 2), Fraction(4, 3), Fraction(-1, 12)],
    6: [Fraction(-49, 18), Fraction(3, 2), Fraction(-3, 20), Fraction(1, 90)],
    8: [Fraction(-205, 72), Fraction(8, 5), Fraction(-1, 5), Fraction(8, 315), Fraction(-1, 560)],
}


def laplacian(order: int, spacing: Sequence[float]) -> List[Term]:
    """The term list sb_stencil_laplacian returns: centre, then for k = 1..R the axes x, y, z, side - then side +; in
    double, i_a = 1 / (h_a * h_a), an axis term c_k * i_a, the centre (c_0 * i_x + c_0 * i_y) + c_0 * i_z."""
    c = [float(v) for v in LAPLACIAN_COEFFS[order]]
    inv = [1.0 / (float(h) * float(h)) for h in spacing]
    terms: List[Term] = [(0, (0, 0, 0), (c[0] * inv[0] + c[0] * inv[1]) + c[0] * inv[2])]
    for k in range(1, order // 2 + 1):
        for a in range(3):
            for side in (-1, 1):
                o = [0, 0, 0]
                o[a] = side * k
                terms.append((0, tuple(o), c[k] * inv[a]))
    return terms


def _view(a: np.ndarray, lo, ext, o) -> np.ndarray:
    return a[lo[2] + o[2] : lo[2] + o[2] + ext[2], lo[1] + o[1] : lo[1] + o[1] + ext[1], lo[0] + o[0] : lo[0] + o[0] + ext[0]]


def apply_box(terms: Sequence[Term], src: np.ndarray, aux: Optional[np.ndarray], dst: np.ndarray, lo, ext) -> None:
    """dst[box] = op(src, aux) in dst's dtype, in place.  aux may be dst (its box is read before it is written)."""
    T = dst.dtype.type
    acc = None
    for s, o, w in terms:
        v = _view(src, lo, ext, o) if s == 0 else _view(aux, lo, ext, (0, 0, 0))
        m = np.multiply(T(w), v, dtype=dst.dtype)
        acc = m if acc is None else np.add(acc, m, dtype=dst.dtype)
    _view(dst, lo, ext, (0, 0, 0))[...] = acc


def apply_cell_loop(terms: Sequence[Term], src: np.ndarray, aux: Optional[np.ndarray], dst: np.ndarray, lo, ext) -> None:
    """The same rule one cell at a time with numpy scalars (the slow restatement the array form is checked against)."""
    T = dst.dtype.type
    for z in range(lo[2], lo[2] + ext[2]):
        for y in range(lo[1], lo[1] + ext[1]):
            for x in range(lo[0], lo[0] + ext[0]):
                acc = None
                for s, o, w in terms:
                    v = src[z + o[2], y + o[1], x + o[0]] if s == 0 else aux[z, y, x]
                    m = T(T(w) * T(v))
                    acc = m if acc is None else T(acc + m)
                dst[z, y, x] = acc


def apply_periodic(terms: Sequence[Term], u: np.ndarray, aux: Optional[np.ndarray]) -> np.ndarray:
    """The op on a periodic [z, y, x] grid with no ghost cells (reads wrap around)."""
    T = u.dtype.type
    acc = None
    for s, o, w in terms:
        v = np.roll(u, (-o[2], -o[1], -o[0]), axis=(0, 1, 2)) if s == 0 else aux
        m = np.multiply(T(w), v, dtype=u.dtype)
        acc = m if acc is None else np.add(acc, m, dtype=u.dtype)
    return acc


def reach(terms: Sequence[Term]) -> Tuple[Tuple[int, int, int], Tuple[int, int, int]]:
    """(below, above) per axis: how far the op reads on each side of a cell."""
    rm = tuple(max([0] + [-o[a] for _, o, _ in terms]) for a in range(3))
    rp = tuple(max([0] + [o[a] for _, o, _ in terms]) for a in range(3))
    return rm, rp


def check_rule(terms: Sequence[Term], radius27: Sequence[int]) -> bool:
    """sb_stencil_check restated: the limits, then per term with o != 0 the ghost box of sign(o) is exchanged and each
    non-zero component fits the face radius on its side."""
    if not 1 <= len(terms) <= 64:
        return False
    for s, o, _ in terms:
        if s not in (0, 1) or any(abs(c) > 4 for c in o) or (s == 1 and any(o)):
            return False
    for s, o, _ in terms:
        if not any(o):
            continue
        sg = [(c > 0) - (c < 0) for c in o]
        if radius27[(sg[2] + 1) * 9 + (sg[1] + 1) * 3 + (sg[0] + 1)] <= 0:
            return False
        for a in range(3):
            if o[a]:
                d = [0, 0, 0]
                d[a] = sg[a]
                if abs(o[a]) > radius27[(d[2] + 1) * 9 + (d[1] + 1) * 3 + (d[0] + 1)]:
                    return False
    return True
