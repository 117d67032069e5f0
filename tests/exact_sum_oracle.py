"""Oracle of the exact reductions (sb_reduce_exact_*): the exact sum of the per-cell terms of reduce_oracle.cell_terms
in Python integers (every term scaled by 2^1074), rounded once to nearest with ties to even, the special-value rule of
include/stencil_b200.h, and conversion to and from the sb_exact_sum words.  math.fsum is not used for the result: it
raises on an intermediate overflow such as [1e308, 1e308, -1e308] and on inf + -inf, where this rule gives a value."""
import math
from typing import Iterable, List, Sequence, Tuple

import numpy as np

import reduce_oracle as ro

WORDS = 34  # SB_EXACT_WORDS
NAN, POS_INF, NEG_INF = 1, 2, 4  # SB_EXACT_NAN, SB_EXACT_POS_INF, SB_EXACT_NEG_INF
SHIFT = 1074  # the unit of the accumulator is 2^-1074
MOD = 1 << (64 * WORDS)


def flags_of(x: np.ndarray) -> int:
    x = np.asarray(x, dtype=np.float64)
    f = NAN if bool(np.isnan(x).any()) else 0
    f |= POS_INF if bool((x == math.inf).any()) else 0
    f |= NEG_INF if bool((x == -math.inf).any()) else 0
    return f


def exact_int(x: np.ndarray) -> int:
    """sum of the finite elements of x times 2^1074, exactly.  Vectorised: every finite x = +-m * 2^(p - 1074) with
    m < 2^53; m is cut into three 18-bit pieces whose signed sums per p stay below 2^53 in magnitude for up to 2^34
    terms, so numpy's float64 bincount adds them exactly."""
    x = np.asarray(x, dtype=np.float64).ravel()
    x = x[np.isfinite(x)]
    if x.size == 0:
        return 0
    assert x.size < 2**34
    b = x.view(np.uint64)
    ex = ((b >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64)
    m = (b & np.uint64((1 << 52) - 1)).astype(np.int64) | np.where(ex > 0, np.int64(1) << np.int64(52), np.int64(0))
    p = np.where(ex > 0, ex - 1, 0)
    sign = np.where((b >> np.uint64(63)) != 0, -1.0, 1.0)
    total = 0
    for k in range(3):
        piece = ((m >> np.int64(18 * k)) & np.int64((1 << 18) - 1)).astype(np.float64) * sign
        sums = np.bincount(p, weights=piece, minlength=2047)
        for pos in np.nonzero(sums)[0]:
            total += int(sums[pos]) << int(pos + 18 * k)
    return total


def round_int(total: int) -> float:
    """total * 2^-1074 rounded to nearest, ties to even; +0.0 for zero; +-inf beyond the double range."""
    if total == 0:
        return 0.0
    neg, mag = total < 0, abs(total)
    top = mag.bit_length() - 1
    if top < 53:
        r = math.ldexp(float(mag), -SHIFT)
    else:
        lsb = top - 52
        mant, rem, half = mag >> lsb, mag & ((1 << lsb) - 1), 1 << (lsb - 1)
        if rem > half or (rem == half and mant & 1):
            mant += 1
        e = lsb - SHIFT
        r = math.inf if mant.bit_length() - 1 + e > 1023 else math.ldexp(float(mant), e)
    return -r if neg else r


def round_sum(total: int, flags: int) -> float:
    """The special-value rule, then round_int."""
    if flags & NAN or (flags & POS_INF and flags & NEG_INF):
        return math.nan
    if flags & POS_INF:
        return math.inf
    if flags & NEG_INF:
        return -math.inf
    return round_int(total)


def exact_sum(x: Iterable[float]) -> float:
    a = np.asarray(list(x) if not isinstance(x, np.ndarray) else x, dtype=np.float64)
    return round_sum(exact_int(a), flags_of(a))


def to_words(total: int) -> List[int]:
    t = total % MOD
    return [(t >> (64 * k)) & ((1 << 64) - 1) for k in range(WORDS)]


def from_words(words: Sequence[int]) -> int:
    t = sum(int(w) << (64 * k) for k, w in enumerate(words))
    return t - MOD if t >> (64 * WORDS - 1) else t


def reduce_cells(kind: int, *srcs: np.ndarray) -> dict:
    """What an exact reduction over these cells must give: min / max / count as reduce_oracle.reduce_cells, sum and
    sumsq correctly rounded, and the accumulators (integer, flags)."""
    with np.errstate(over="ignore", invalid="ignore"):
        v, q = ro.cell_terms(kind, *srcs)
    v, q = v.ravel(), q.ravel()
    n = int(v.size)
    sv, sq = (exact_int(v), flags_of(v)), (exact_int(q), flags_of(q))
    nan = bool(np.isnan(v).any())
    return dict(
        min=math.inf if n == 0 else math.nan if nan else float(v.min()),
        max=-math.inf if n == 0 else math.nan if nan else float(v.max()),
        sum=round_sum(*sv),
        sumsq=round_sum(*sq),
        count=n,
        acc=(sv, sq),
    )


def part_acc(part) -> Tuple[Tuple[int, int], Tuple[int, int]]:
    """((sum integer, flags), (sumsq integer, flags)) of a ctypes ReduceExactPart."""
    return tuple((from_words(list(s.word)), int(s.flags)) for s in (part.sum, part.sumsq))
