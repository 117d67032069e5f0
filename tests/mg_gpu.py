"""A V(nu1, nu2) cycle on DistributedDomains from public calls only: the GPU twin of transfer_oracle.vcycle, used by the
GPU tests, tests/mp_mg_check.py and scripts/time_transfer.py.

Each level is its own DistributedDomain of u, f and r (radius 1 in all 26 directions, so prolongation can read the
coarse ghost corners), with ODD(0) on u at every wall face.  Per level: red-black Gauss-Seidel (sb_stencil_relax with
omega = 1, one in-place apply per colour), the residual r = f - A u as one apply, restriction of r into the coarser f,
u = 0 * f there, the recursion, and the in-place correction u <- u + P e."""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

import colour_oracle as co
import stencil_b200 as sb
import transfer_oracle as to

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED


class GpuLevel:
    def __init__(self, size, h: float, sigma: float, dtype, boundary: Sequence[sb.Boundary], gpus: Sequence[int]):
        self.size = tuple(size)
        dd = sb.DistributedDomain(*size)
        dd.set_gpus(list(gpus))
        dd.set_radius(sb.Radius.constant(1))
        self.u, self.f, self.r = (dd.add_data(dtype, n) for n in ("u", "f", "r"))
        dd.set_boundary(*boundary)
        for fc in range(6):
            if boundary[fc // 2] == F:
                dd.set_boundary_condition(self.u, sb.FACES[fc], sb.BC.ODD(0.0))
        dd.realize()
        self.dd = dd
        A = co.helmholtz(h, sigma)
        self.gs = sb.StencilOp(co.relax(A, 1.0), dtype)
        self.res = sb.StencilOp(to.residual_terms(A), dtype)
        self.zero = sb.StencilOp(to.ZERO_TERMS, dtype)

    def smooth(self, sweeps: int) -> None:
        for _ in range(sweeps):
            for c in range(2):
                self.dd.apply(self.gs, (self.u, "curr"), self.u, (self.f, "curr"), colour=(2, c))

    def residual(self) -> None:
        self.dd.apply(self.res, (self.r, "curr"), self.u, (self.f, "curr"))

    def residual_norm(self) -> float:
        self.residual()
        return self.dd.reduce(self.r, "curr", exact=True).l2()


def hierarchy(size, levels: int, sigma: float, dtype, boundary: Sequence[sb.Boundary], gpus: Sequence[int]) -> List[GpuLevel]:
    """levels domains from size down by 2 per axis, spacing 1 / n_x on the finest, doubled per level (as
    transfer_oracle.hierarchy)."""
    out, h = [], 1.0 / size[0]
    for _ in range(levels):
        out.append(GpuLevel(size, h, sigma, dtype, boundary, gpus))
        size, h = tuple(n // 2 for n in size), 2 * h
    return out


def vcycle(lv: List[GpuLevel], l: int = 0, nu1: int = 2, nu2: int = 2, coarse_sweeps: int = 30) -> None:
    L = lv[l]
    if l == len(lv) - 1:
        L.smooth(coarse_sweeps)
        return
    L.smooth(nu1)
    L.residual()
    C = lv[l + 1]
    L.dd.restrict_to(C.dd, (C.f, "curr"), (L.r, "curr"))
    C.dd.apply(C.zero, (C.u, "curr"), C.f, exchange=False)
    vcycle(lv, l + 1, nu1, nu2, coarse_sweeps)
    L.dd.prolong_from(C.dd, (L.u, "curr"), (C.u, "curr"), aux=(L.u, "curr"))
    L.smooth(nu2)


def close(lv: List[GpuLevel]) -> None:
    for L in lv:
        L.dd.close()
