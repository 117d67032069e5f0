"""numpy restatement of the variable-coefficient stencil rule of include/stencil_b200.h (sb_stencil_vterm), for the CPU
and GPU tests.  A term is (source, offset, weight) or (source, offset, weight, k, coef_offset).  For every cell p of a box,
in the array's type T, every multiply and add rounded separately, in list order:
    coefficient term  m = (T(w) * C_k(p + c)) * S(p + o)
    plain term        m = T(w) * S(p + o)
    acc = m_0;  acc = acc + m_t;  dst[p] = acc
Arrays are [z, y, x]; boxes are (lo, ext) in (x, y, z) allocation coordinates."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from stencil_op_oracle import _view

MAX_COEFS, COEF_REACH = 4, 1


def split(t) -> Tuple[int, tuple, float, int, tuple]:
    """(source, offset, weight, k, coef_offset) of a 3- or 5-tuple term; k = -1 for a plain term."""
    return tuple(t) if len(t) == 5 else (t[0], t[1], t[2], -1, (0, 0, 0))


def div_grad(spacing: Sequence[float]) -> List[tuple]:
    """The term list sb_stencil_div_grad returns: for the axes x, y, z, with i_a = 1 / (h_a * h_a) in double,
    (src +e_a, i_a, C_a at +e_a), (src 0, -i_a, C_a at +e_a), (src 0, -i_a, C_a at 0), (src -e_a, i_a, C_a at 0)."""
    out = []
    for a in range(3):
        i = 1.0 / (float(spacing[a]) * float(spacing[a]))
        e = [0, 0, 0]
        e[a] = 1
        e, m, z = tuple(e), tuple(-v for v in e), (0, 0, 0)
        out += [(0, e, i, a, e), (0, z, -i, a, e), (0, z, -i, a, z), (0, m, i, a, z)]
    return out


def apply_box(terms, src: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray], dst: np.ndarray, lo, ext) -> None:
    """dst[box] = op(src, aux, coefs) in dst's dtype, in place.  aux may be dst (its box is read before it is written)."""
    T = dst.dtype.type
    acc = None
    for t in terms:
        s, o, w, k, c = split(t)
        v = _view(src, lo, ext, o) if s == 0 else _view(aux, lo, ext, (0, 0, 0))
        wt = T(w) if k < 0 else np.multiply(T(w), _view(coefs[k], lo, ext, c), dtype=dst.dtype)
        m = np.multiply(wt, v, dtype=dst.dtype)
        acc = m if acc is None else np.add(acc, m, dtype=dst.dtype)
    _view(dst, lo, ext, (0, 0, 0))[...] = acc


def apply_cell_loop(terms, src: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray], dst: np.ndarray, lo, ext) -> None:
    """The same rule one cell at a time with numpy scalars."""
    T = dst.dtype.type
    for z in range(lo[2], lo[2] + ext[2]):
        for y in range(lo[1], lo[1] + ext[1]):
            for x in range(lo[0], lo[0] + ext[0]):
                acc = None
                for t in terms:
                    s, o, w, k, c = split(t)
                    v = src[z + o[2], y + o[1], x + o[0]] if s == 0 else aux[z, y, x]
                    wt = T(w) if k < 0 else T(T(w) * coefs[k][z + c[2], y + c[1], x + c[0]])
                    m = T(wt * T(v))
                    acc = m if acc is None else T(acc + m)
                dst[z, y, x] = acc


def apply_periodic(terms, u: np.ndarray, aux: Optional[np.ndarray], coefs: Sequence[np.ndarray]) -> np.ndarray:
    """The op on a periodic [z, y, x] grid with no ghost cells (reads wrap around)."""
    T = u.dtype.type
    acc = None
    for t in terms:
        s, o, w, k, c = split(t)
        v = np.roll(u, (-o[2], -o[1], -o[0]), axis=(0, 1, 2)) if s == 0 else aux
        wt = T(w) if k < 0 else np.multiply(T(w), np.roll(coefs[k], (-c[2], -c[1], -c[0]), axis=(0, 1, 2)), dtype=u.dtype)
        m = np.multiply(wt, v, dtype=u.dtype)
        acc = m if acc is None else np.add(acc, m, dtype=u.dtype)
    return acc


def reach(terms) -> Tuple[Tuple[int, int, int], Tuple[int, int, int]]:
    """(below, above) per axis over every src offset and every coefficient offset."""
    offs = []
    for t in terms:
        s, o, w, k, c = split(t)
        offs.append(o)
        if k >= 0:
            offs.append(c)
    rm = tuple(max([0] + [-o[a] for o in offs]) for a in range(3))
    rp = tuple(max([0] + [o[a] for o in offs]) for a in range(3))
    return rm, rp


def _in_reach(o, radius27) -> bool:
    if not any(o):
        return True
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


def check_rule(terms, radius27: Sequence[int]) -> bool:
    """sb_stencil_vcheck restated: the limits, then the reach test on every src offset and every coefficient offset."""
    if not 1 <= len(terms) <= 64:
        return False
    for t in terms:
        s, o, w, k, c = split(t)
        if s not in (0, 1) or any(abs(v) > 4 for v in o) or (s == 1 and any(o)):
            return False
        if not -1 <= k < MAX_COEFS or any(abs(v) > COEF_REACH for v in c) or (k == -1 and any(c)):
            return False
    for t in terms:
        s, o, w, k, c = split(t)
        if not _in_reach(o, radius27) or (k >= 0 and not _in_reach(c, radius27)):
            return False
    return True
