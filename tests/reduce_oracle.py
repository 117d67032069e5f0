"""Oracle of the reductions (sb_reduce_*): the per-cell value v and squared term q of include/stencil_b200.h in FP64,
one numpy operation per rounding (numpy never contracts a multiply and an add into an FMA), exact sums with math.fsum,
the merge tree of sb_reduce_combine, and the error bound DESIGN section 2.6 states."""
import math
from typing import List, Sequence, Tuple

import numpy as np

SCALAR, DIFF, NORM3 = 0, 1, 2
U = 2.0**-53  # unit round-off of FP64
CHAIN = 256  # kRedChain: a tile holds as many block passes as keep every lane's chain at or below this


def cell_terms(kind: int, a: np.ndarray, b: np.ndarray = None, c: np.ndarray = None) -> Tuple[np.ndarray, np.ndarray]:
    """(v, q) per cell, in FP64."""
    x = np.asarray(a, dtype=np.float64)
    if kind == SCALAR:
        return x, x * x
    y = np.asarray(b, dtype=np.float64)
    if kind == DIFF:
        v = x - y
        return v, v * v
    z = np.asarray(c, dtype=np.float64)
    s = (x * x + y * y) + z * z
    return np.sqrt(s), s


def reduce_cells(kind: int, *srcs: np.ndarray) -> dict:
    """What a reduction over these cells must give: exact min / max (NaN if any v is NaN), the exact sums (fsum of the
    FP64 terms), the sums of |term| that bound the error, and the count."""
    v, q = cell_terms(kind, *srcs)
    v, q = v.ravel(), q.ravel()
    n = int(v.size)
    if n == 0:
        return dict(min=math.inf, max=-math.inf, sum=0.0, sumsq=0.0, count=0, abs_sum=0.0, abs_sumsq=0.0)
    nan = bool(np.isnan(v).any())
    return dict(
        min=math.nan if nan else float(v.min()),
        max=math.nan if nan else float(v.max()),
        sum=math.fsum(v.tolist()),
        sumsq=math.fsum(q.tolist()),
        count=n,
        abs_sum=math.fsum(np.abs(v).tolist()),
        abs_sumsq=math.fsum(np.abs(q).tolist()),
    )


def merge(a: Sequence[float], b: Sequence[float]) -> Tuple[float, float, float, float, int]:
    """red_merge: (min, max, sum, sumsq, count); a NaN min / max operand wins, equal operands give a."""
    def mn(x, y):
        return x if x != x else y if (y != y or y < x) else x

    def mx(x, y):
        return x if x != x else y if (y != y or y > x) else x

    return (mn(a[0], b[0]), mx(a[1], b[1]), a[2] + b[2], a[3] + b[3], a[4] + b[4])


def combine(parts: Sequence[Sequence[float]]) -> Tuple[float, float, float, float, int]:
    """sb_reduce_combine: parts[i] = merge(parts[i], parts[i + s]) for i % 2s == 0, s = 1, 2, 4, ...; result parts[0]."""
    a: List = [tuple(p) for p in parts]
    n = len(a)
    s = 1
    while s < n:
        for i in range(0, n - s, 2 * s):
            a[i] = merge(a[i], a[i + s])
        s *= 2
    return a[0]


def tree_depth(n_tiles: int, n_subdomains: int) -> int:
    """Additions above the per-thread chains: 8 inside a tile (256 threads), ceil(log2 T) over the tiles of a
    subdomain, ceil(log2 P) over the subdomains.  A tile holds at least one row, so T <= the rows of the box (y * z)
    is always a safe argument."""
    return 8 + math.ceil(math.log2(max(1, n_tiles))) + math.ceil(math.log2(max(1, n_subdomains)))


def chain_len(nx: int, es: int) -> int:
    """The longest per-thread chain k of a box nx cells wide (sb_reduce_plan_create's per-row formula, taken over both
    access widths): CHAIN, or one row's cells of one lane when that is longer (one pass per tile)."""
    g = 1 << min(5, math.ceil(math.log2(max(1, (nx * es + 15) // 16))))
    k = CHAIN
    for n in (16 // es, 1):
        per_row = n * (-(-(nx // n) // g)) + 2 * (-(-min(nx, n - 1) // g))
        k = max(k, per_row)
    return k


def bound(abs_total: float, n_tiles: int, n_subdomains: int, k: int = CHAIN) -> float:
    """|computed - exact| <= (k + h + 1) * 2^-53 * sum |term|, h the depth of the tree above the chains."""
    return (k + tree_depth(n_tiles, n_subdomains) + 1) * U * abs_total
