"""CPU checks of the reductions: sb_reduce_combine against the oracle's tree bit for bit, the C structs against the
header, the oracle's per-cell rule, and every error sb_reduce_plan_create / _launch / sb_reduce_combine report.  No GPU
is used: every error is found before anything is allocated."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import reduce_oracle as ro
import stencil_b200 as sb
from stencil_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bits(r) -> tuple:
    return tuple(struct.pack("<d", float(x)) for x in r[:4]) + (int(r[4]),)


def random_part(rng) -> tuple:
    kind = rng.integers(0, 10)
    if kind == 0:  # an empty subdomain box
        return (math.inf, -math.inf, 0.0, 0.0, 0)
    vals = rng.standard_normal(int(rng.integers(1, 6))) * 10.0 ** rng.integers(-3, 4)
    if kind == 1:
        vals[0] = math.nan
    elif kind == 2:
        vals[0] = math.inf
    elif kind == 3:
        vals[0] = -math.inf
    elif kind == 4:
        vals[0] = -0.0
    mn = math.nan if np.isnan(vals).any() else float(vals.min())
    mx = math.nan if np.isnan(vals).any() else float(vals.max())
    return (mn, mx, float(vals.sum()), float((vals * vals).sum()), int(vals.size))


@pytest.mark.parametrize("seed", range(4))
def test_combine_matches_the_oracle_tree_bit_for_bit(seed):
    rng = np.random.default_rng(seed)
    for n in range(1, 65):
        parts = [random_part(rng) for _ in range(n)]
        got = sb.reduce_combine([sb.Reduction(*p) for p in parts])
        want = ro.combine(parts)
        assert bits((got.min, got.max, got.sum, got.sumsq, got.count)) == bits(want), (seed, n)


def test_combine_propagates_nan_and_keeps_empty_parts_neutral():
    empty = sb.Reduction(math.inf, -math.inf, 0.0, 0.0, 0)
    one = sb.Reduction(-1.5, 2.0, 0.5, 6.25, 2)
    got = sb.reduce_combine([empty, one, empty])
    assert (got.min, got.max, got.sum, got.sumsq, got.count) == (-1.5, 2.0, 0.5, 6.25, 2)
    got = sb.reduce_combine([one, sb.Reduction(math.nan, math.nan, math.nan, 1.0, 1)])
    assert math.isnan(got.min) and math.isnan(got.max) and math.isnan(got.sum) and got.count == 3
    e = sb.reduce_combine([empty])
    assert (e.min, e.max, e.sum, e.sumsq, e.count) == (math.inf, -math.inf, 0.0, 0.0, 0)


def test_reduction_helpers():
    r = sb.Reduction(-1.0, 3.0, 4.0, 16.0, 4)
    assert r.mean() == 1.0 and r.rms() == 2.0 and r.l2() == 4.0


def test_reduce_structs_match_the_header(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "stencil_b200.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu\\n", sizeof(sb_reduce_item), sizeof(sb_reduce_result), '
                   'offsetof(sb_reduce_item, acc_origin), offsetof(sb_reduce_result, count)); return 0; }\n')
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_lib.ReduceItem), C.sizeof(_lib.ReduceResult), _lib.ReduceItem.acc_origin.offset, _lib.ReduceResult.count.offset]


def test_oracle_terms_are_separately_rounded():
    a = np.array([1.0 + 2.0**-30, 3.0], dtype=np.float64)
    b = np.array([1.0, -4.0], dtype=np.float64)
    c = np.array([2.0**-27, 0.0], dtype=np.float64)
    v, q = ro.cell_terms(ro.NORM3, a, b, c)
    s0 = (a[0] * a[0] + b[0] * b[0]) + c[0] * c[0]
    assert q[0] == s0 and v[1] == 5.0 and q[1] == 25.0
    v, q = ro.cell_terms(ro.DIFF, np.float32([0.1]), np.float32([0.3]))
    assert v[0] == float(np.float32(0.1)) - float(np.float32(0.3))
    r = ro.reduce_cells(ro.SCALAR, np.array([1.0, math.nan, -2.0]))
    assert math.isnan(r["min"]) and math.isnan(r["max"]) and math.isnan(r["sum"])
    r = ro.reduce_cells(ro.SCALAR, np.zeros((0, 3, 3)))
    assert (r["min"], r["max"], r["count"]) == (math.inf, -math.inf, 0)


# ------------------------------------------------------------------------------------------ errors (no GPU)
FAKE = 0x10000  # never dereferenced: every check below fails before any device access


def item(kind=0, dtype=2, ptrs=(FAKE, FAKE, FAKE), pitch=10 * 8, ysize=10, lo=(1, 1, 1), hi=(9, 9, 9), pitches=None, ysizes=None):
    src = (_lib.Pitched * 3)()
    for s in range(3):
        src[s] = _lib.Pitched(ptrs[s], (pitches or [pitch] * 3)[s], (ysizes or [ysize] * 3)[s])
    return _lib.ReduceItem(kind, dtype, src, _lib.I3(0, 0, 0), _lib.I3(*lo), _lib.I3(*hi))


def create(items, n=None):
    arr = (_lib.ReduceItem * max(1, len(items)))(*items)
    h = C.c_void_p()
    rc = sb.lib().sb_reduce_plan_create(C.byref(h), 0, arr, len(items) if n is None else n)
    return rc, sb.lib().sb_last_error().decode()


@pytest.mark.parametrize(
    "it, msg",
    [
        (item(dtype=0), "dtype"),
        (item(dtype=3), "dtype"),
        (item(kind=3), "unknown kind"),
        (item(kind=1, pitches=[80, 88, 80]), "different pitches or row counts"),
        (item(kind=2, ysizes=[10, 10, 11]), "different pitches or row counts"),
        (item(ptrs=(FAKE + 4, FAKE, FAKE)), "multiples of the 8-byte element"),
        (item(dtype=1, pitch=42), "multiples of the 4-byte element"),
        (item(kind=1, ptrs=(FAKE, FAKE + 2, FAKE), dtype=1, pitch=40), "multiples of the 4-byte element"),
        (item(lo=(1, 5, 1), hi=(9, 4, 9)), "lo > hi on axis 1"),
        (item(lo=(-1, 1, 1)), "outside the allocation"),
        (item(hi=(11, 9, 9)), "outside the allocation"),
        (item(ptrs=(0, FAKE, FAKE)), "bad pitched pointer"),
        (item(kind=1, ptrs=(FAKE, 0, FAKE)), "bad pitched pointer"),
    ],
)
def test_plan_create_rejects(it, msg):
    rc, err = create([it])
    assert rc == -1 and msg in err, err


def test_plan_create_needs_items():
    rc, err = create([item()], n=0)
    assert rc == -1 and "n >= 1" in err
    h = C.c_void_p()
    assert sb.lib().sb_reduce_plan_create(C.byref(h), 0, None, 1) == -1


def test_launch_and_combine_reject_bad_arguments():
    L = sb.lib()
    assert L.sb_reduce_plan_launch(None, C.c_void_p(FAKE), None) == -1 and "null plan" in L.sb_last_error().decode()
    out = _lib.ReduceResult()
    assert L.sb_reduce_combine(None, 1, C.byref(out)) == -1
    assert L.sb_reduce_combine((_lib.ReduceResult * 1)(), 0, C.byref(out)) == -1
    assert L.sb_reduce_plan_bytes(None) == 0 and L.sb_reduce_plan_destroy(None) == 0


def test_domain_rejects_bad_items_before_any_allocation():
    dd = sb.DistributedDomain(8, 8, 8)
    h = dd.add_data(np.float64)
    i8 = dd.add_data(np.int8)
    f4 = dd.add_data(np.float32)
    for bad in [("sum", h), ("scalar",), ("scalar", h, "prev"), ("diff", h, h), ("norm", h, h), ("scalar", i8), ("norm", h, f4, h)]:
        with pytest.raises(sb.StencilError):
            dd._reduce_key(bad)
    assert dd._reduce_key(("scalar", h, "next")) == (0, (0,), "next")


def test_chain_length_follows_the_planner():
    """k is kRedChain up to rows of about 8000 cells; wider rows give one pass per tile and a chain of one lane's body
    cells plus one head and one tail cell."""
    assert ro.chain_len(512, 8) == ro.CHAIN and ro.chain_len(8000, 8) == ro.CHAIN
    assert ro.chain_len(8192, 8) == 8192 // 32 + 2
    assert ro.chain_len(65536, 8) == 65536 // 32 + 2
    assert ro.chain_len(1, 4) == ro.CHAIN
