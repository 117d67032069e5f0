"""numpy restatement of the linear stencil system rule of include/stencil_b200.h (sb_stencil_sys_term), for the CPU and GPU
tests.  A term is (output, input, offset, weight) or (output, input, offset, weight, coef, coef_offset).  For every cell
p of a box and every output j, over the terms of output j in list order, in the arrays' type T, every multiply and add
rounded separately:
    coefficient term  m = (T(w) * I_coef(p + c)) * I_in(p + o)
    plain term        m = T(w) * I_in(p + o)
    acc = m_first;  acc = acc + m;  O_j[p] = acc
Every output is computed before any is written, so an output may be an input read at offset 0.
Arrays are [z, y, x]; boxes are (lo, ext) in (x, y, z) allocation coordinates."""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np

from stencil_op_oracle import _view

MAX_INPUTS, MAX_OUTPUTS, MAX_TERMS, MAX_REACH, COEF_REACH = 8, 4, 128, 4, 1


def split(t) -> Tuple[int, int, tuple, float, int, tuple]:
    """(output, input, offset, weight, coef, coef_offset) of a 4- or 6-tuple term; coef = -1 for a plain term."""
    return tuple(t) if len(t) == 6 else (t[0], t[1], t[2], t[3], -1, (0, 0, 0))


def _diff(stagger: int, a: int, h: float, out: int, inp: int, sign: float) -> List[tuple]:
    w = 0.5 / h if stagger == 0 else 1.0 / h
    hi, lo = (1 if stagger >= 0 else 0), (-1 if stagger <= 0 else 0)
    e = lambda k: tuple(k if b == a else 0 for b in range(3))  # noqa: E731
    return [(out, inp, e(hi), sign * w), (out, inp, e(lo), -(sign * w))]


def grad(stagger: int, spacing: Sequence[float]) -> List[tuple]:
    """sb_stencil_grad: input 0 -> outputs x, y, z."""
    return [t for a in range(3) for t in _diff(stagger, a, float(spacing[a]), a, 0, 1.0)]


def div(stagger: int, spacing: Sequence[float]) -> List[tuple]:
    """sb_stencil_div: inputs 0, 1, 2 -> output 0, axes in order."""
    return [t for a in range(3) for t in _diff(stagger, a, float(spacing[a]), 0, a, 1.0)]


def curl(stagger: int, spacing: Sequence[float]) -> List[tuple]:
    """sb_stencil_curl: output j = D_{j+1} in_{j+2} - D_{j+2} in_{j+1}, the positive part first."""
    out = []
    for j in range(3):
        a, b = (j + 1) % 3, (j + 2) % 3
        out += _diff(stagger, a, float(spacing[a]), j, b, 1.0) + _diff(stagger, b, float(spacing[b]), j, a, -1.0)
    return out


def shifted(terms, ib: int = 0, ob: int = 0) -> List[tuple]:
    out = []
    for t in terms:
        j, i, o, w, k, c = split(t)
        out.append((j + ob, i + ib, o, w, k + ib, c) if k >= 0 else (j + ob, i + ib, o, w))
    return out


def scaled(terms, f: float) -> List[tuple]:
    return [tuple(t[:3]) + (t[3] * float(f),) + tuple(t[4:]) for t in terms]


def nout_of(terms) -> int:
    return max(split(t)[0] for t in terms) + 1


def apply_box(terms, inputs: Sequence[Optional[np.ndarray]], outputs: Sequence[np.ndarray], lo, ext) -> None:
    """outputs[j][box] = the rule, in place; outputs may be inputs read at offset 0."""
    T = outputs[0].dtype
    accs = {}
    for t in terms:
        j, i, o, w, k, c = split(t)
        wt = T.type(w) if k < 0 else np.multiply(T.type(w), _view(inputs[k], lo, ext, c), dtype=T)
        m = np.multiply(wt, _view(inputs[i], lo, ext, o), dtype=T)
        accs[j] = m if j not in accs else np.add(accs[j], m, dtype=T)
    for j, acc in accs.items():
        _view(outputs[j], lo, ext, (0, 0, 0))[...] = acc


def apply_cell_loop(terms, inputs, outputs, lo, ext) -> None:
    """The same rule one cell at a time with numpy scalars."""
    T = outputs[0].dtype.type
    for z in range(lo[2], lo[2] + ext[2]):
        for y in range(lo[1], lo[1] + ext[1]):
            for x in range(lo[0], lo[0] + ext[0]):
                accs = {}
                for t in terms:
                    j, i, o, w, k, c = split(t)
                    wt = T(w) if k < 0 else T(T(w) * inputs[k][z + c[2], y + c[1], x + c[0]])
                    m = T(wt * T(inputs[i][z + o[2], y + o[1], x + o[0]]))
                    accs[j] = m if j not in accs else T(accs[j] + m)
                for j, v in accs.items():
                    outputs[j][z, y, x] = v


def apply_periodic(terms, inputs: Sequence[np.ndarray]) -> List[np.ndarray]:
    """The system on periodic [z, y, x] grids with no ghost cells (reads wrap around); returns the outputs."""
    T = inputs[0].dtype
    roll = lambda a, o: np.roll(a, (-o[2], -o[1], -o[0]), axis=(0, 1, 2))  # noqa: E731
    accs = {}
    for t in terms:
        j, i, o, w, k, c = split(t)
        wt = T.type(w) if k < 0 else np.multiply(T.type(w), roll(inputs[k], c), dtype=T)
        m = np.multiply(wt, roll(inputs[i], o), dtype=T)
        accs[j] = m if j not in accs else np.add(accs[j], m, dtype=T)
    return [accs[j] for j in range(nout_of(terms))]


def reach(terms, i: int) -> Tuple[Tuple[int, int, int], Tuple[int, int, int]]:
    """(below, above) per axis of input i's reads, as a source and as a coefficient."""
    offs = [(0, 0, 0)]
    for t in terms:
        j, ii, o, w, k, c = split(t)
        if ii == i:
            offs.append(o)
        if k == i:
            offs.append(c)
    return tuple(max(-o[a] for o in offs) for a in range(3)), tuple(max(o[a] for o in offs) for a in range(3))


def reads(terms) -> set:
    return {split(t)[1] for t in terms} | {split(t)[4] for t in terms if split(t)[4] >= 0}


def check_rule(terms, nin: int, nout: int, radius27: Sequence[int]) -> bool:
    """sb_stencil_sys_check restated: the limits, then the reach test of sb_stencil_check on every offset."""
    from vstencil_oracle import _in_reach

    if not (1 <= nin <= MAX_INPUTS and 1 <= nout <= MAX_OUTPUTS and 1 <= len(terms) <= MAX_TERMS):
        return False
    for t in terms:
        j, i, o, w, k, c = split(t)
        if not (0 <= j < nout and 0 <= i < nin) or any(abs(v) > MAX_REACH for v in o):
            return False
        if not -1 <= k < nin or any(abs(v) > COEF_REACH for v in c) or (k == -1 and any(c)):
            return False
    return all(_in_reach(split(t)[2], radius27) and (split(t)[4] < 0 or _in_reach(split(t)[5], radius27)) for t in terms)
