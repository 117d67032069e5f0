"""CPU checks of the exact reductions: the oracle against fractions.Fraction and math.fsum, sb_reduce_exact_round and
sb_reduce_exact_combine through ctypes on accumulators built in Python, every error of sb_reduce_exact_plan_create with
the ordered plan's messages, and the C structs against the header.  No GPU is used."""
import ctypes as C
import math
import os
import struct
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import exact_sum_oracle as xo
import stencil_b200 as sb
from stencil_b200 import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_oracle_reduce import FAKE, item  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DMAX = sys.float_info.max


def b(x: float) -> bytes:
    return struct.pack("<d", x)


def fraction_sum(xs) -> float:
    """Fraction's exact sum of finite terms, rounded by Python's correctly rounded int / int division."""
    f = sum((Fraction(float(x)) for x in xs), Fraction(0))
    if f == 0:
        return 0.0
    try:
        return f.numerator / f.denominator
    except OverflowError:
        return math.copysign(math.inf, f)


def adversarial(rng, n):
    """exponents over the whole double range, subnormals, pairs x, -x and tiny terms"""
    x = rng.standard_normal(n) * np.ldexp(1.0, rng.integers(-1074, 1000, n))
    x[: n // 4] = np.ldexp(rng.integers(-(2**52), 2**52, n // 4).astype(np.float64), -1074)  # subnormals
    x[n // 4 : n // 2] = -x[n // 2 : n // 2 + n // 4]
    return x


@pytest.mark.parametrize("seed", range(6))
def test_oracle_against_fraction_and_fsum(seed):
    rng = np.random.default_rng(seed)
    for n in (1, 2, 7, 100, 1000):
        for x in (rng.standard_normal(n) * 3.0, adversarial(rng, max(n, 4)), rng.standard_normal(n) * 1e300):
            want = fraction_sum(x)
            got = xo.exact_sum(x)
            assert b(got) == b(want), (seed, n)
            try:
                assert b(math.fsum(x.tolist()) + 0.0) == b(got)  # fsum, where it returns
            except OverflowError:
                pass


def test_oracle_where_fsum_raises():
    assert xo.exact_sum([1e308, 1e308, -1e308]) == 1e308
    assert math.isnan(xo.exact_sum([math.inf, -math.inf, 1.0]))
    assert xo.exact_sum([DMAX, DMAX]) == math.inf and xo.exact_sum([-DMAX, -DMAX]) == -math.inf
    assert xo.exact_sum([math.inf, 1.0, math.inf]) == math.inf and xo.exact_sum([-math.inf, 2.0]) == -math.inf
    assert math.isnan(xo.exact_sum([1.0, math.nan]))
    z = xo.exact_sum([-0.0, -0.0])
    assert b(z) == b(0.0)
    assert b(xo.exact_sum([1.5, -1.5])) == b(0.0)


def test_words_round_trip():
    rng = np.random.default_rng(1)
    for _ in range(100):
        t = int(rng.integers(-(2**62), 2**62)) << int(rng.integers(0, 2000))
        assert xo.from_words(xo.to_words(t)) == t


# ------------------------------------------------------------------------------------------ round / combine via ctypes
def part_of(total: int, flags: int = 0, total_q: int = 0, flags_q: int = 0, mn=math.inf, mx=-math.inf, count=0) -> _lib.ReduceExactPart:
    p = _lib.ReduceExactPart()
    p.min, p.max, p.count = mn, mx, count
    for s, t, f in ((p.sum, total, flags), (p.sumsq, total_q, flags_q)):
        for k, w in enumerate(xo.to_words(t)):
            s.word[k] = w
        s.flags = f
    return p


def rounded(total: int, flags: int = 0) -> float:
    return sb.reduce_exact_round(part_of(total, flags)).sum


ONE = 1 << 1074  # 1.0 in accumulator units


@pytest.mark.parametrize(
    "total, want",
    [
        (0, 0.0),
        (ONE, 1.0),
        (-3 * ONE, -3.0),
        (ONE + (ONE >> 53), 1.0),  # tie between 1 and 1 + 2^-52: to even (1)
        (ONE + 3 * (ONE >> 53), 1.0 + 2.0**-51),  # tie between 1 + 2^-52 and 1 + 2^-51: to even
        (ONE + (ONE >> 53) + 1, 1.0 + 2.0**-52),  # just above the tie
        (-(ONE + (ONE >> 53)), -1.0),
        (1, 5e-324),  # the smallest subnormal
        (-7, -7 * 5e-324),
        ((1 << 52) - 1, math.ldexp((1 << 52) - 1, -1074)),  # the largest subnormal
        ((1 << 53) + 1, math.ldexp((1 << 53) + 1 - 1, -1074)),  # 54 bits, tie to even
        ((1 << 2098) - (1 << 2044), math.inf),  # 2^1024 - 2^970: the overflow threshold rounds to inf
        ((1 << 2098) - (1 << 2044) - 1, DMAX),  # one unit below it: DBL_MAX
        (-((1 << 2098) - (1 << 2044)), -math.inf),
        (1 << 2150, math.inf),  # far beyond the double range
    ],
)
def test_round(total, want):
    got = rounded(total)
    assert b(got) == b(want), (got, want)
    assert b(got) == b(xo.round_int(total))


def test_round_flags_and_passthrough():
    assert math.isnan(rounded(ONE, xo.NAN))
    assert math.isnan(rounded(ONE, xo.POS_INF | xo.NEG_INF))
    assert rounded(-ONE, xo.POS_INF) == math.inf and rounded(ONE, xo.NEG_INF) == -math.inf
    r = sb.reduce_exact_round(part_of(ONE, 0, 2 * ONE, xo.POS_INF, mn=-2.0, mx=5.0, count=9))
    assert (r.min, r.max, r.sum, r.sumsq, r.count) == (-2.0, 5.0, 1.0, math.inf, 9)


def test_combine_cancels_to_positive_zero_and_ors_flags():
    a, c = part_of(12345 * ONE + 17, 0, count=3), part_of(-(12345 * ONE + 17), xo.NEG_INF, count=4)
    got = sb.reduce_exact_combine([a, c])
    assert xo.part_acc(got)[0] == (0, xo.NEG_INF) and got.count == 7
    assert bytes(got.sum) == bytes(part_of(0, xo.NEG_INF).sum)
    got = sb.reduce_exact_combine([part_of(ONE, 0), part_of(-ONE, 0)])
    assert b(sb.reduce_exact_round(got).sum) == b(0.0)


@pytest.mark.parametrize("seed", range(4))
def test_combine_in_shuffled_orders(seed):
    rng = np.random.default_rng(seed)
    parts, total, totq, flags, count = [], 0, 0, 0, 0
    mins, maxs = [], []
    for _ in range(int(rng.integers(1, 40))):
        t = int(rng.integers(-(2**62), 2**62)) << int(rng.integers(0, 2030))
        q = int(rng.integers(0, 2**62)) << int(rng.integers(0, 2030))
        f = int(rng.choice([0, 0, 0, xo.NAN, xo.POS_INF, xo.NEG_INF]))
        mn, mx = sorted([float(x) for x in rng.choice([-0.0, 0.0, 1.5, -2.5, math.nan], 2)])
        n = int(rng.integers(0, 100))
        parts.append(part_of(t, f, q, 0, mn, mx, n))
        total, totq, flags, count = total + t, totq + q, flags | f, count + n
        mins.append(mn)
        maxs.append(mx)
    ref = None
    for _ in range(6):
        order = rng.permutation(len(parts))
        got = sb.reduce_exact_combine([parts[i] for i in order])
        assert xo.part_acc(got) == ((total, flags), (totq, 0)) and got.count == count
        if ref is None:
            ref = bytes(got)
        assert bytes(got) == ref  # min / max (NaN payloads and signed zeros included) do not depend on the order


# ------------------------------------------------------------------------------------------ errors (no GPU)
def create_exact(items, n=None):
    arr = (_lib.ReduceItem * max(1, len(items)))(*items)
    h = C.c_void_p()
    rc = sb.lib().sb_reduce_exact_plan_create(C.byref(h), 0, arr, len(items) if n is None else n)
    return rc, sb.lib().sb_last_error().decode()


def create_plain(items):
    arr = (_lib.ReduceItem * max(1, len(items)))(*items)
    h = C.c_void_p()
    rc = sb.lib().sb_reduce_plan_create(C.byref(h), 0, arr, len(items))
    return rc, sb.lib().sb_last_error().decode()


BAD = [
    item(dtype=0),
    item(dtype=3),
    item(kind=3),
    item(kind=1, pitches=[80, 88, 80]),
    item(kind=2, ysizes=[10, 10, 11]),
    item(ptrs=(FAKE + 4, FAKE, FAKE)),
    item(dtype=1, pitch=42),
    item(kind=1, ptrs=(FAKE, FAKE + 2, FAKE), dtype=1, pitch=40),
    item(lo=(1, 5, 1), hi=(9, 4, 9)),
    item(lo=(-1, 1, 1)),
    item(hi=(11, 9, 9)),
    item(ptrs=(0, FAKE, FAKE)),
    item(kind=1, ptrs=(FAKE, 0, FAKE)),
]


@pytest.mark.parametrize("i", range(len(BAD)))
def test_plan_create_rejects_with_the_ordered_plans_messages(i):
    rc, err = create_exact([item(), BAD[i]])
    rc0, err0 = create_plain([item(), BAD[i]])
    assert rc == rc0 == -1 and err == err0, (err, err0)


def test_plan_create_needs_items_and_rejects_very_long_rows():
    rc, err = create_exact([item()], n=0)
    assert rc == -1 and "sb_reduce_exact_plan_create needs an output handle and n >= 1 items" in err
    h = C.c_void_p()
    assert sb.lib().sb_reduce_exact_plan_create(C.byref(h), 0, None, 1) == -1
    assert sb.lib().sb_reduce_exact_plan_create(None, 0, (_lib.ReduceItem * 1)(item()), 1) == -1
    wide = item(dtype=1, pitch=4 * ((1 << 27) + 8), hi=((1 << 27) + 2, 2, 2), lo=(0, 0, 0))
    rc, err = create_exact([wide])
    assert rc == -1 and "rows of more than 2^27 cells" in err, err


def test_launch_combine_and_round_reject_bad_arguments():
    L = sb.lib()
    assert L.sb_reduce_exact_plan_launch(None, C.c_void_p(FAKE), None) == -1 and "null plan" in L.sb_last_error().decode()
    out = _lib.ReduceExactPart()
    assert L.sb_reduce_exact_combine(None, 1, C.byref(out)) == -1
    assert L.sb_reduce_exact_combine((_lib.ReduceExactPart * 1)(), 0, C.byref(out)) == -1
    assert L.sb_reduce_exact_round(None, C.byref(_lib.ReduceResult())) == -1
    assert L.sb_reduce_exact_round(C.byref(out), None) == -1
    assert L.sb_reduce_exact_plan_bytes(None) == 0 and L.sb_reduce_exact_plan_destroy(None) == 0


def test_exact_structs_match_the_header(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "stencil_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu %zu %d\\n", sizeof(sb_exact_sum), sizeof(sb_reduce_exact_part), '
                   'offsetof(sb_exact_sum, flags), offsetof(sb_reduce_exact_part, count), offsetof(sb_reduce_exact_part, sum), '
                   'offsetof(sb_reduce_exact_part, sumsq), SB_EXACT_WORDS); return 0; }\n')
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    P = _lib.ReduceExactPart
    assert got == [C.sizeof(_lib.ExactSum), C.sizeof(P), _lib.ExactSum.flags.offset, P.count.offset, P.sum.offset, P.sumsq.offset, _lib.EXACT_WORDS]
    for name in ("sb_reduce_exact_plan_create", "sb_reduce_exact_plan_launch", "sb_reduce_exact_plan_bytes", "sb_reduce_exact_plan_destroy",
                 "sb_reduce_exact_combine", "sb_reduce_exact_round"):
        assert hasattr(sb.lib(), name)
