"""Constant-coefficient linear stencil operators over the C ABI (sb_stencil_*, DESIGN.md section 2.7).

    op = StencilOp.laplacian(4, (hx, hy, hz), np.float64)          # or StencilOp([(source, (dx, dy, dz), w), ...], dtype)
    heat = StencilOp([(s, o, dt * w) for s, o, w in op.terms] + [(0, (0, 0, 0), 1.0)], np.float64)
    dd.apply(heat, h)                                               # next = heat(curr), overlapped with the exchange
    dd.swap()

A term reads src (source 0) at p + offset or aux (source 1) at p.  Per cell, in the quantity's type with every multiply
and add rounded separately: acc = T(w_0) * S_0; acc = acc + T(w_k) * S_k in list order; dst[p] = acc.  The rule, the
reach check against a domain's radius and the Laplacian table live in the C library; this module only carries them.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import I27, Pitched, StencilTerm, check, i3, lib, stream_ptr

Term = Tuple[int, Tuple[int, int, int], float]


def _dtype_code(dtype) -> int:
    dt = np.dtype(dtype)
    if dt == np.float32:
        return 1  # SB_DTYPE_F32
    if dt == np.float64:
        return 2  # SB_DTYPE_F64
    raise _lib.StencilError(f"a stencil operator computes in float32 or float64, not {dt}")


class StencilOp:
    """An operator: terms (source, (dx, dy, dz), weight) applied in list order, in dtype (float32 or float64)."""

    def __init__(self, terms: Iterable[Sequence], dtype):
        out: List[Term] = []
        for t in terms:
            s, o, w = t
            out.append((int(s), (int(o[0]), int(o[1]), int(o[2])), float(w)))
        self.terms: Tuple[Term, ...] = tuple(out)
        self.dtype = np.dtype(dtype)
        self.dtype_code = _dtype_code(self.dtype)
        # the limits of a term list, whatever the domain: every ghost box at the largest radius
        check(lib().sb_stencil_check(self.c_terms(), len(self.terms), I27(*([_lib.STENCIL_MAX_REACH] * 27))))

    @staticmethod
    def laplacian(order: int, spacing: Sequence[float], dtype) -> "StencilOp":
        """The central-difference Laplacian of order 2, 4, 6 or 8 (sb_stencil_laplacian): centre first, then for
        k = 1..order/2 the axes x, y, z, side - then side +."""
        h = (C.c_double * 3)(*[float(v) for v in spacing])
        n = check(lib().sb_stencil_laplacian(int(order), h, None, 0))
        buf = (StencilTerm * n)()
        check(lib().sb_stencil_laplacian(int(order), h, buf, n))
        return StencilOp([(t.source, tuple(t.offset), t.weight) for t in buf], dtype)

    def c_terms(self):
        arr = (StencilTerm * max(1, len(self.terms)))()
        for k, (s, o, w) in enumerate(self.terms):
            arr[k] = StencilTerm(s, (C.c_int32 * 3)(*o), w)
        return arr

    @property
    def has_aux(self) -> bool:
        return any(s == 1 for s, _, _ in self.terms)

    def reach(self) -> int:
        return max(max(abs(c) for c in o) for _, o, _ in self.terms)

    def check(self, radius) -> None:
        """Raise StencilError unless a domain with this Radius exchanges every ghost cell the op reads."""
        check(lib().sb_stencil_check(self.c_terms(), len(self.terms), radius.c27()))

    def key(self) -> tuple:
        return (self.terms, self.dtype.str)

    def __eq__(self, o) -> bool:
        return isinstance(o, StencilOp) and self.key() == o.key()

    def __hash__(self) -> int:
        return hash(self.key())

    def __repr__(self) -> str:
        return f"StencilOp({len(self.terms)} terms, {self.dtype})"


class StencilPlan:
    """sb_stencil_plan: the op over a list of boxes [lo, hi) (global coordinates) of three allocations of one subdomain."""

    def __init__(self, device: int, op: StencilOp, dst: Pitched, src: Pitched, aux: Pitched, acc_origin, zsize: int,
                 boxes: Sequence[Tuple[Sequence[int], Sequence[int]]]):
        nb = len(boxes)
        lo = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[0]])
        hi = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[1]])
        h = C.c_void_p()
        check(lib().sb_stencil_plan_create(C.byref(h), device, op.dtype_code, op.c_terms(), len(op.terms), dst, src, aux,
                                           i3(acc_origin), int(zsize), nb, lo, hi))
        self._h = h
        self.device = device
        self.bytes = int(lib().sb_stencil_plan_bytes(h))

    def launch(self, stream=None) -> None:
        check(lib().sb_stencil_plan_launch(self._h, stream_ptr(stream)))

    def destroy(self) -> None:
        if getattr(self, "_h", None):
            lib().sb_stencil_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass
