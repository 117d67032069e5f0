"""Linear stencil operators, constant and variable coefficients, over the C ABI (sb_stencil_*, DESIGN.md section 2.7).

    op = StencilOp.laplacian(4, (hx, hy, hz), np.float64)          # or StencilOp([(source, (dx, dy, dz), w), ...], dtype)
    heat = StencilOp([(s, o, dt * w) for s, o, w in op.terms] + [(0, (0, 0, 0), 1.0)], np.float64)
    dd.apply(heat, h)                                               # next = heat(curr), overlapped with the exchange
    dd.swap()

A term reads src (source 0) at p + offset or aux (source 1) at p.  Per cell, in the quantity's type with every multiply
and add rounded separately: acc = T(w_0) * S_0; acc = acc + T(w_k) * S_k in list order; dst[p] = acc.  A coefficient term
(source, offset, weight, k, coef_offset) also reads coefficient field k (0..3) at p + coef_offset (|c_a| <= 1) and
contributes (T(w) * C_k) * S instead:

    kdt = StencilOp.div_grad((hx, hy, hz), np.float64).scaled(dt)    # dt div(kappa grad u), kappa on faces in 3 fields
    heat = StencilOp(list(kdt.terms) + [(0, (0, 0, 0), 1.0)], np.float64)
    dd.apply(heat, h, h, coefs=[kx, ky, kz])

A system (DESIGN.md section 2.8) has several outputs over several inputs, one launch for all of them.  A term
(output, input, offset, weight) or (output, input, offset, weight, coef, coef_offset) adds to output `output`; each
output sums its own terms in list order by the same rule:

    curl_h = StencilSystem.curl(-1, (h, h, h), np.float64).scaled(dt / eps)    # inputs 0-2: H, outputs 0-2
    ident = StencilSystem([(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)], np.float64, nin=6)   # inputs 3-5: E
    E = [(q, "curr") for q in (ex, ey, ez)]
    dd.apply_system(ident + curl_h, E, [hx, hy, hz] + E)                       # E = E + dt/eps curl H, in place

A coloured apply (DESIGN.md section 2.9) writes only the cells of one colour and may run in place; one apply per colour
is a Gauss-Seidel or SOR sweep.  For A u = f with f in the quantity f:

    sor = StencilOp.laplacian(2, (h, h, h), np.float64).scaled(-1.0).relax(omega)   # u + omega (f - A u) / a_c
    for c in range(2):                                                               # red, then black
        dd.apply(sor, (u, "curr"), u, f, colour=(2, c))

The rule, the reach and colour checks against a domain's radius and the Laplacian, div-grad, relaxation, grad, div and
curl tables live in the C library; this module only carries them.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import I27, Pitched, StencilSysTerm, StencilTerm, StencilVTerm, check, i3, lib, stream_ptr

Term = Tuple  # (source, offset, weight) or (source, offset, weight, coef, coef_offset)


def _dtype_code(dtype) -> int:
    dt = np.dtype(dtype)
    if dt == np.float32:
        return 1  # SB_DTYPE_F32
    if dt == np.float64:
        return 2  # SB_DTYPE_F64
    raise _lib.StencilError(f"a stencil operator computes in float32 or float64, not {dt}")


class StencilOp:
    """An operator: terms (source, (dx, dy, dz), weight) or coefficient terms (source, (dx, dy, dz), weight, coef,
    (cx, cy, cz)) applied in list order, in dtype (float32 or float64).  A 5-tuple with coef -1 is a plain term and is
    kept as the 3-tuple."""

    def __init__(self, terms: Iterable[Sequence], dtype):
        out: List[Term] = []
        for t in terms:
            if len(t) == 5 and int(t[3]) != -1:
                s, o, w, k, c = t
                out.append((int(s), (int(o[0]), int(o[1]), int(o[2])), float(w), int(k), (int(c[0]), int(c[1]), int(c[2]))))
                continue
            if len(t) == 5 and any(int(v) for v in t[4]):
                raise _lib.StencilError(f"term {t!r}: a term without a coefficient field has coefficient offset (0, 0, 0)")
            if len(t) not in (3, 5):
                raise _lib.StencilError(f"term {t!r}: (source, offset, weight) or (source, offset, weight, coef, coef_offset)")
            s, o, w = t[:3]
            out.append((int(s), (int(o[0]), int(o[1]), int(o[2])), float(w)))
        self.terms: Tuple[Term, ...] = tuple(out)
        self.dtype = np.dtype(dtype)
        self.dtype_code = _dtype_code(self.dtype)
        # the limits of a term list, whatever the domain: every ghost box at the largest radius
        self._check(I27(*([_lib.STENCIL_MAX_REACH] * 27)))

    def _check(self, r27, colours: int = 1) -> None:
        if colours != 1:
            check(lib().sb_stencil_ccheck(self.c_vterms(), len(self.terms), r27, int(colours)))
        elif self.has_coef:
            check(lib().sb_stencil_vcheck(self.c_vterms(), len(self.terms), r27))
        else:
            check(lib().sb_stencil_check(self.c_terms(), len(self.terms), r27))

    @staticmethod
    def laplacian(order: int, spacing: Sequence[float], dtype) -> "StencilOp":
        """The central-difference Laplacian of order 2, 4, 6 or 8 (sb_stencil_laplacian): centre first, then for
        k = 1..order/2 the axes x, y, z, side - then side +."""
        h = (C.c_double * 3)(*[float(v) for v in spacing])
        n = check(lib().sb_stencil_laplacian(int(order), h, None, 0))
        buf = (StencilTerm * n)()
        check(lib().sb_stencil_laplacian(int(order), h, buf, n))
        return StencilOp([(t.source, tuple(t.offset), t.weight) for t in buf], dtype)

    @staticmethod
    def div_grad(spacing: Sequence[float], dtype) -> "StencilOp":
        """The conservative second-order div(kappa grad u) (sb_stencil_div_grad): 12 terms; coefficient field a holds
        kappa on the faces normal to axis a, C_a(p) on the face between p - e_a and p."""
        h = (C.c_double * 3)(*[float(v) for v in spacing])
        n = check(lib().sb_stencil_div_grad(h, None, 0))
        buf = (StencilVTerm * n)()
        check(lib().sb_stencil_div_grad(h, buf, n))
        return StencilOp([(t.source, tuple(t.offset), t.weight, t.coef, tuple(t.coef_offset)) for t in buf], dtype)

    def relax(self, omega: float) -> "StencilOp":
        """The SOR update of A u = f for this op A, f on aux (sb_stencil_relax): u + omega (f - A u) / a_c, with a_c the
        weight of A's one centre term.  Terms: (src, 0, 1 - omega), each off-centre term of A as (src, o, (-omega w) / a_c),
        then (aux, 0, omega / a_c).  omega = 1 in a coloured sweep is Gauss-Seidel, out of place Jacobi; omega outside
        (0, 2) diverges for a symmetric positive definite A.  A must have constant coefficients and no aux term."""
        if self.has_coef:
            raise _lib.StencilError("relax: the op has coefficient terms; the relaxation table takes constant coefficients")
        n = len(self.terms)
        buf = (StencilTerm * (n + 1))()
        n = check(lib().sb_stencil_relax(self.c_terms(), n, float(omega), buf, n + 1))
        return StencilOp([(t.source, tuple(t.offset), t.weight) for t in buf[:n]], self.dtype)

    def scaled(self, f: float) -> "StencilOp":
        """The same op with every weight multiplied by f (in double)."""
        return StencilOp([(t[0], t[1], t[2] * float(f)) + tuple(t[3:]) for t in self.terms], self.dtype)

    def c_terms(self):
        arr = (StencilTerm * max(1, len(self.terms)))()
        for k, t in enumerate(self.terms):
            arr[k] = StencilTerm(t[0], (C.c_int32 * 3)(*t[1]), t[2])
        return arr

    def c_vterms(self):
        arr = (StencilVTerm * max(1, len(self.terms)))()
        for k, t in enumerate(self.terms):
            coef, co = (t[3], t[4]) if len(t) == 5 else (-1, (0, 0, 0))
            arr[k] = StencilVTerm(t[0], (C.c_int32 * 3)(*t[1]), coef, (C.c_int32 * 3)(*co), t[2])
        return arr

    @property
    def has_aux(self) -> bool:
        return any(t[0] == 1 for t in self.terms)

    @property
    def has_coef(self) -> bool:
        return any(len(t) == 5 for t in self.terms)

    @property
    def ncoef(self) -> int:
        """The number of coefficient fields apply() takes: the highest field a term names, plus one (0: none)."""
        return max([t[3] + 1 for t in self.terms if len(t) == 5] + [0])

    def reach(self) -> int:
        return max(max(abs(c) for c in t[1]) for t in self.terms)

    def check(self, radius, colours: int = 1) -> None:
        """Raise StencilError unless a domain with this Radius exchanges every ghost cell the op reads (src cells and
        coefficient cells alike) and, for colours 2 or 8, every src term with a non-zero offset reads a cell of another
        colour (sb_stencil_ccheck)."""
        self._check(radius.c27(), colours)

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
                 boxes: Sequence[Tuple[Sequence[int], Sequence[int]]], coefs: Optional[Sequence[Pitched]] = None,
                 colour: Optional[Tuple[int, int]] = None, omega: Optional[float] = None):
        """coefs: the coefficient allocations (sb_stencil_vplan_create), field k = coefs[k]; None for a plain op.
        colour: (m, c), write only the cells of colour c under the colouring m (sb_stencil_cplan_create); dst may then be
        src.  omega: the diagonal relaxation u + omega ((f - A u) / d) of the op A with f on aux (sb_stencil_dplan_create;
        colour None means m = 1)."""
        nb = len(boxes)
        lo = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[0]])
        hi = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[1]])
        h = C.c_void_p()
        if omega is not None:
            cs = list(coefs or [])
            carr = (Pitched * max(1, len(cs)))(*cs)
            m, c = colour if colour is not None else (1, 0)
            check(lib().sb_stencil_dplan_create(C.byref(h), device, op.dtype_code, op.c_vterms(), len(op.terms), dst, src, aux, carr, len(cs),
                                                float(omega), int(m), int(c), i3(acc_origin), int(zsize), nb, lo, hi))
        elif colour is not None:
            cs = list(coefs or [])
            carr = (Pitched * max(1, len(cs)))(*cs)
            check(lib().sb_stencil_cplan_create(C.byref(h), device, op.dtype_code, op.c_vterms(), len(op.terms), dst, src, aux, carr,
                                                len(cs), int(colour[0]), int(colour[1]), i3(acc_origin), int(zsize), nb, lo, hi))
        elif coefs is None and not op.has_coef:
            check(lib().sb_stencil_plan_create(C.byref(h), device, op.dtype_code, op.c_terms(), len(op.terms), dst, src, aux,
                                               i3(acc_origin), int(zsize), nb, lo, hi))
        else:
            cs = list(coefs or [])
            carr = (Pitched * max(1, len(cs)))(*cs)
            check(lib().sb_stencil_vplan_create(C.byref(h), device, op.dtype_code, op.c_vterms(), len(op.terms), dst, src, aux, carr,
                                                len(cs), i3(acc_origin), int(zsize), nb, lo, hi))
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


SysTerm = Tuple  # (output, input, offset, weight) or (output, input, offset, weight, coef, coef_offset)


class StencilSystem:
    """A system: terms (output, input, (dx, dy, dz), weight) or (output, input, (dx, dy, dz), weight, coef, (cx, cy, cz)),
    in dtype (float32 or float64), over nin inputs and nout outputs (by default one more than the highest index a term
    names).  A 6-tuple with coef -1 is a plain term and is kept as the 4-tuple."""

    def __init__(self, terms: Iterable[Sequence], dtype, nin: Optional[int] = None, nout: Optional[int] = None):
        out: List[SysTerm] = []
        for t in terms:
            if len(t) not in (4, 6):
                raise _lib.StencilError(f"term {t!r}: (output, input, offset, weight) or (output, input, offset, weight, coef, coef_offset)")
            j, i, o, w = int(t[0]), int(t[1]), (int(t[2][0]), int(t[2][1]), int(t[2][2])), float(t[3])
            if len(t) == 6 and int(t[4]) != -1:
                c = t[5]
                out.append((j, i, o, w, int(t[4]), (int(c[0]), int(c[1]), int(c[2]))))
                continue
            if len(t) == 6 and any(int(v) for v in t[5]):
                raise _lib.StencilError(f"term {t!r}: a term without a coefficient field has coefficient offset (0, 0, 0)")
            out.append((j, i, o, w))
        self.terms: Tuple[SysTerm, ...] = tuple(out)
        self.dtype = np.dtype(dtype)
        self.dtype_code = _dtype_code(self.dtype)
        reads = [t[1] for t in out] + [t[4] for t in out if len(t) == 6]
        self.nin = int(nin) if nin is not None else max(reads, default=-1) + 1
        self.nout = int(nout) if nout is not None else max([t[0] for t in out], default=-1) + 1
        self._check(I27(*([_lib.STENCIL_MAX_REACH] * 27)))

    def _check(self, r27) -> None:
        check(lib().sb_stencil_sys_check(self.c_terms(), len(self.terms), self.nin, self.nout, r27))

    @staticmethod
    def _table(fn, stagger: int, spacing: Sequence[float], dtype) -> "StencilSystem":
        h = (C.c_double * 3)(*[float(v) for v in spacing])
        n = check(fn(int(stagger), h, None, 0))
        buf = (StencilSysTerm * n)()
        check(fn(int(stagger), h, buf, n))
        return StencilSystem([(t.output, t.input, tuple(t.offset), t.weight) for t in buf], dtype)

    @staticmethod
    def grad(stagger: int, spacing: Sequence[float], dtype) -> "StencilSystem":
        """Input 0 -> outputs x, y, z (sb_stencil_grad).  stagger +1: forward differences, -1: backward, 0: central."""
        return StencilSystem._table(lib().sb_stencil_grad, stagger, spacing, dtype)

    @staticmethod
    def div(stagger: int, spacing: Sequence[float], dtype) -> "StencilSystem":
        """Inputs 0, 1, 2 -> output 0 (sb_stencil_div)."""
        return StencilSystem._table(lib().sb_stencil_div, stagger, spacing, dtype)

    @staticmethod
    def curl(stagger: int, spacing: Sequence[float], dtype) -> "StencilSystem":
        """Inputs 0, 1, 2 -> outputs 0, 1, 2 (sb_stencil_curl)."""
        return StencilSystem._table(lib().sb_stencil_curl, stagger, spacing, dtype)

    def scaled(self, f: float) -> "StencilSystem":
        """The same system with every weight multiplied by f (in double)."""
        return StencilSystem([t[:3] + (t[3] * float(f),) + tuple(t[4:]) for t in self.terms], self.dtype, self.nin, self.nout)

    def shifted(self, input_base: int = 0, output_base: int = 0) -> "StencilSystem":
        """The same system reading inputs input_base + i (coefficients included) and writing outputs output_base + j."""
        ib, ob = int(input_base), int(output_base)
        out = []
        for t in self.terms:
            u = (t[0] + ob, t[1] + ib) + t[2:4]
            out.append(u + (t[4] + ib, t[5]) if len(t) == 6 else u)
        return StencilSystem(out, self.dtype, self.nin + ib, self.nout + ob)

    def __add__(self, o: "StencilSystem") -> "StencilSystem":
        """Concatenation: self's terms, then o's; each output still sums its terms in this order."""
        if not isinstance(o, StencilSystem) or o.dtype != self.dtype:
            raise _lib.StencilError(f"cannot concatenate {self!r} and {o!r}")
        return StencilSystem(self.terms + o.terms, self.dtype, max(self.nin, o.nin), max(self.nout, o.nout))

    def c_terms(self):
        arr = (StencilSysTerm * max(1, len(self.terms)))()
        for k, t in enumerate(self.terms):
            coef, co = (t[4], t[5]) if len(t) == 6 else (-1, (0, 0, 0))
            arr[k] = StencilSysTerm(t[0], t[1], (C.c_int32 * 3)(*t[2]), coef, (C.c_int32 * 3)(*co), t[3])
        return arr

    def moved_inputs(self) -> set:
        """The inputs some term reads at a non-zero offset (as a source or a coefficient)."""
        return {t[1] for t in self.terms if any(t[2])} | {t[4] for t in self.terms if len(t) == 6 and any(t[5])}

    def read_inputs(self) -> set:
        return {t[1] for t in self.terms} | {t[4] for t in self.terms if len(t) == 6}

    def check(self, radius) -> None:
        """Raise StencilError unless a domain with this Radius exchanges every ghost cell the system reads."""
        self._check(radius.c27())

    def key(self) -> tuple:
        return (self.terms, self.dtype.str, self.nin, self.nout)

    def __eq__(self, o) -> bool:
        return isinstance(o, StencilSystem) and self.key() == o.key()

    def __hash__(self) -> int:
        return hash(self.key())

    def __repr__(self) -> str:
        return f"StencilSystem({len(self.terms)} terms, {self.nin} -> {self.nout}, {self.dtype})"


class SystemPlan(StencilPlan):
    """sb_stencil_sys_plan_create: the system over a list of boxes [lo, hi) (global coordinates) of one subdomain's output
    and input allocations (an input no term reads may be Pitched(None, 0, 0))."""

    def __init__(self, device: int, system: StencilSystem, outputs: Sequence[Pitched], inputs: Sequence[Pitched], acc_origin, zsize: int,
                 boxes: Sequence[Tuple[Sequence[int], Sequence[int]]]):
        nb = len(boxes)
        lo = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[0]])
        hi = (C.c_int64 * (3 * max(1, nb)))(*[int(v) for b in boxes for v in b[1]])
        outs = (Pitched * max(1, len(outputs)))(*outputs)
        ins = (Pitched * max(1, len(inputs)))(*inputs)
        h = C.c_void_p()
        check(lib().sb_stencil_sys_plan_create(C.byref(h), device, system.dtype_code, system.c_terms(), len(system.terms), outs, len(outputs), ins,
                                               len(inputs), i3(acc_origin), int(zsize), nb, lo, hi))
        self._h = h
        self.device = device
        self.bytes = int(lib().sb_stencil_plan_bytes(h))
