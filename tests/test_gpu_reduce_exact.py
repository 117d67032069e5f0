"""Exact reductions on the GPU (sb_reduce_exact_*, DistributedDomain.reduce*(exact=True)): sum and sumsq equal the
oracle (tests/exact_sum_oracle.py) bit for bit, min / max / count equal the ordered plan's bits, and every result and
combined accumulator is the same for every partition.  Ghost cells hold NaN and 1e300, so a reduction that read one
would fail."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

import exact_sum_oracle as xo
import reduce_oracle as ro
import stencil_b200 as sb
from gpu_util import DevArray
from stencil_b200 import _lib
from test_gpu_reduce import RADII, cabi_item, fields, load, make_domain

pytestmark = pytest.mark.gpu


def bits(r) -> tuple:
    return tuple(struct.pack("<d", float(getattr(r, f))) for f in ("min", "max", "sum", "sumsq")) + (r.count,)


def assert_exact(got: sb.Reduction, want: dict, plain: sb.Reduction = None):
    for f in ("sum", "sumsq"):
        g, w = getattr(got, f), want[f]
        assert (math.isnan(g) and math.isnan(w)) or struct.pack("<d", g) == struct.pack("<d", w), (f, g, w)
    assert got.count == want["count"]
    if plain is not None:  # min / max / count: the ordered plan's bits
        for f in ("min", "max"):
            g, w = getattr(got, f), getattr(plain, f)
            assert (math.isnan(g) and math.isnan(w)) or struct.pack("<d", g) == struct.pack("<d", w), (f, g, w)
        assert got.count == plain.count


ITEMS = lambda hs: [("scalar", hs[0]), ("scalar", hs[0], "next"), ("diff", hs[0]), ("norm", hs[0], hs[1], hs[2])]  # noqa: E731


def check_all_kinds(dd, hs, size, seed):
    dt = dd.dtypes_[hs[0].id]
    a, b, c, nx = fields(size, dt, 4, seed=seed)
    load(dd, hs[0], a)
    load(dd, hs[0], nx, "next", poison=1e300)
    load(dd, hs[1], b, poison=1e300)
    load(dd, hs[2], c)
    got = dd.reduce_many(ITEMS(hs), exact=True)
    plain = dd.reduce_many(ITEMS(hs))
    want = [xo.reduce_cells(ro.SCALAR, a), xo.reduce_cells(ro.SCALAR, nx), xo.reduce_cells(ro.DIFF, a, nx), xo.reduce_cells(ro.NORM3, a, b, c)]
    for g, w, p in zip(got, want, plain):
        assert_exact(g, w, p)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("rname", list(RADII))
def test_layouts(dtype, rname):
    size = (37, 11, 9)
    dd, hs = make_domain(size, RADII[rname](), dtype, 1, 3)
    try:
        check_all_kinds(dd, hs, size, 7)
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_narrow_and_mid_vector_boxes_through_the_c_abi(dtype):
    rng = np.random.default_rng(3)
    shape = (6, 7, 43)
    hosts = [rng.standard_normal(shape).astype(dtype) for _ in range(3)]
    arrs = [DevArray(h) for h in hosts]
    try:
        cases, items = [], []
        for x0 in range(5):
            for w in (0, 1, 2, 3, 5, 17, 38 - x0):
                lo, hi = (x0, 1, 2), (x0 + w, 6, 5)
                for kind, n in ((ro.SCALAR, 1), (ro.DIFF, 2), (ro.NORM3, 3)):
                    cases.append((kind, lo, hi, n))
                    items.append(cabi_item(kind, dtype, arrs[:n], lo, hi))
        plan, pplan = sb.ExactReducePlan(0, items), sb.ReducePlan(0, items)
        plan.launch()
        pplan.launch()
        parts, plain = plan.parts(), pplan.results()
        for (kind, lo, hi, n), part, p in zip(cases, parts, plain):
            box = [h[lo[2] : hi[2], lo[1] : hi[1], lo[0] : hi[0]] for h in hosts[:n]]
            want = xo.reduce_cells(kind, *box)
            assert xo.part_acc(part) == want["acc"]
            assert_exact(sb.reduce_exact_round(part), want, p)
        plan.destroy()
        pplan.destroy()
    finally:
        for a in arrs:
            a.free()


def adversarial(rng, shape, case):
    n = int(np.prod(shape))
    if case == "spread":  # exponents over the whole range, subnormals included
        x = rng.standard_normal(n) * np.ldexp(1.0, rng.integers(-1074, 1015, n))
        x[::7] = np.ldexp(rng.integers(-(2**52), 2**52, x[::7].size).astype(np.float64), -1074)
    elif case == "pairs":  # x, -x and tiny terms
        x = rng.standard_normal(n) * 1e200
        x[1::2] = -x[0::2][: x[1::2].size]
        x[::97] = rng.standard_normal(x[::97].size) * 1e-300
    elif case == "specials":  # NaN, +-inf, q overflow (|v| > 1.4e154)
        x = rng.standard_normal(n) * 1e160
        x[5] = math.inf
        x[n // 2] = -math.inf
    elif case == "nan":
        x = rng.standard_normal(n)
        x[n // 3] = math.nan
    else:  # near the overflow threshold: the exact sum leaves the double range, then comes back
        x = np.finfo(np.float64).max * rng.choice([-1.0, 1.0], n)
    return x.reshape(shape)


@pytest.mark.parametrize("case", ["spread", "pairs", "specials", "nan", "huge"])
def test_adversarial_fp64(case):
    size = (45, 13, 11)
    dd, hs = make_domain(size, 1, np.float64, 2, 3)
    try:
        rng = np.random.default_rng(["spread", "pairs", "specials", "nan", "huge"].index(case))
        a, b, c = (adversarial(rng, tuple(reversed(size)), case) for _ in range(3))
        for h, f in zip(hs, (a, b, c)):
            load(dd, h, f)
        load(dd, hs[0], b, "next")
        got = dd.reduce_many(ITEMS(hs), exact=True)
        plain = dd.reduce_many(ITEMS(hs))
        want = [xo.reduce_cells(ro.SCALAR, a), xo.reduce_cells(ro.SCALAR, b), xo.reduce_cells(ro.DIFF, a, b), xo.reduce_cells(ro.NORM3, a, b, c)]
        for g, w, p in zip(got, want, plain):
            assert_exact(g, w, p)
    finally:
        dd.close()


def test_fp32_extremes():
    size = (33, 9, 7)
    dd, hs = make_domain(size, 1, np.float32, 3, 3)
    try:
        rng = np.random.default_rng(5)
        fi = np.finfo(np.float32)
        vals = np.array([fi.max, -fi.max, fi.tiny, -fi.tiny, np.float32(1.4e-45), 1.0, -3.0], dtype=np.float32)
        a, b, c = (rng.choice(vals, tuple(reversed(size))).astype(np.float32) for _ in range(3))
        for h, f in zip(hs, (a, b, c)):
            load(dd, h, f)
        load(dd, hs[0], b, "next")
        got = dd.reduce_many(ITEMS(hs), exact=True)
        plain = dd.reduce_many(ITEMS(hs))
        want = [xo.reduce_cells(ro.SCALAR, a), xo.reduce_cells(ro.SCALAR, b), xo.reduce_cells(ro.DIFF, a, b), xo.reduce_cells(ro.NORM3, a, b, c)]
        for g, w, p in zip(got, want, plain):
            assert_exact(g, w, p)
    finally:
        dd.close()


def combined_parts(dd, hs):
    """every item's combined accumulator bytes (sum and sumsq; min / max / count excluded)"""
    plans = dd.reduce_plans(ITEMS(hs), exact=True)
    per = []
    for plan, s in zip(plans, dd._streams):
        plan.launch(s)
        per.append(plan.parts(s))
    order = sorted(range(len(per)), key=lambda i: tuple(reversed(dd.domain_idx_[i])))
    out = []
    for i in range(len(ITEMS(hs))):
        tot = sb.reduce_exact_combine([per[k][i] for k in order])
        out.append(bytes(tot.sum) + bytes(tot.sumsq))
    return out


@pytest.mark.parametrize("align", ["1", "0"])
def test_partition_independence(align, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    size = (53, 29, 23)  # uneven cuts on every axis
    rng = np.random.default_rng(11)
    glob = [rng.standard_normal(tuple(reversed(size))) * np.ldexp(1.0, rng.integers(-40, 40, tuple(reversed(size)))) for _ in range(4)]
    ref = None
    for nsub in (1, 2, 3, 4, 8):
        dd, hs = make_domain(size, 2, np.float64, nsub, 3)
        try:
            load(dd, hs[0], glob[0])
            load(dd, hs[0], glob[3], "next")
            load(dd, hs[1], glob[1])
            load(dd, hs[2], glob[2])
            res = [bits(r) for r in dd.reduce_many(ITEMS(hs), exact=True)]
            acc = combined_parts(dd, hs)
            if ref is None:
                ref = (res, acc)
            assert (res, acc) == ref, nsub
        finally:
            dd.close()
    want = [xo.reduce_cells(ro.SCALAR, glob[0]), xo.reduce_cells(ro.SCALAR, glob[3]), xo.reduce_cells(ro.DIFF, glob[0], glob[3]),
            xo.reduce_cells(ro.NORM3, *glob[:3])]  # fmt: skip
    for r, w in zip(ref[0], want):
        assert r[2] == struct.pack("<d", w["sum"]) and r[3] == struct.pack("<d", w["sumsq"])


def test_repeats_and_graph_replay_are_bit_identical():
    import torch

    size = (64, 48, 40)
    dd, hs = make_domain(size, 1, np.float64, 1, 3)
    try:
        for h, f in zip(hs, fields(size, np.float64, 3, 11)):
            load(dd, h, f)
        d = dd.domains()[0]
        lo, hi = d.get_compute_region()
        src = (_lib.Pitched * 3)(*[d.curr_data(h.id) for h in hs])
        items = [_lib.ReduceItem(k, 2, src, _lib.I3(*d.accessor_origin()), _lib.I3(*lo), _lib.I3(*hi)) for k in (0, 1, 2)]
        plan = sb.ExactReducePlan(0, items)
        s = torch.cuda.Stream()
        runs = []
        for _ in range(3):
            plan.launch(s)
            runs.append([bytes(p) for p in plan.parts(s)])
        assert runs[0] == runs[1] == runs[2]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            plan.launch(s)
        _lib.check(sb.lib().sb_memset(C.c_void_p(plan.out_dev), 0, 3 * C.sizeof(_lib.ReduceExactPart), 0, None))
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            g.replay()
        assert [bytes(p) for p in plan.parts(s)] == runs[0]
        plan.destroy()
    finally:
        dd.close()


def test_512_cubed_fp64_against_the_oracle():
    size = (512, 512, 512)
    dd, hs = make_domain(size, 1, np.float64, 1, 1)
    try:
        a = np.random.default_rng(0).standard_normal((512, 512, 512)) * 3.0
        load(dd, hs[0], a)
        got = dd.reduce(hs[0], exact=True)
        assert_exact(got, xo.reduce_cells(ro.SCALAR, a), dd.reduce(hs[0]))
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_heat_steps_give_the_same_total_on_every_partition(dtype):
    """10 periodic heterogeneous heat steps u <- u + dt div(kappa grad u): the exact reduce(u) is the same bits on 1, 2,
    4 and 8 subdomains after every step."""
    from test_gpu_stencil_domain import SIZE, domain
    from test_gpu_stencil_domain import load as load_q
    from test_gpu_vstencil_domain import heat_terms, kappas

    dtype = np.dtype(dtype)
    op = sb.StencilOp(heat_terms(0.05), dtype)
    rng = np.random.default_rng(8)
    u = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    ks = kappas(rng, dtype)
    runs = []
    for ndom in (1, 2, 4, 8):
        dd, (h, kx, ky, kz) = domain(ndom, sb.Radius.face_edge_corner(1, 0, 0), [dtype] * 4)
        try:
            load_q(dd, h.id, "curr", u)
            for q, k in zip((kx, ky, kz), ks):
                load_q(dd, q.id, "curr", k)
                load_q(dd, q.id, "next", k)
            seq = []
            for _ in range(10):
                dd.apply(op, h, h, coefs=[kx, ky, kz])
                dd.swap()
                seq.append(bits(dd.reduce(h, exact=True)))
            runs.append(seq)
        finally:
            dd.close()
    assert runs[0] == runs[1] == runs[2] == runs[3]


@pytest.mark.parametrize("align", ["1", "0"])
def test_partition_independence_walled(align, monkeypatch):
    """The same on a grid walled on x and z (sb.Boundary.FIXED): 1, 2, 3, 4 and 8 subdomains give the same bits,
    which are the oracle's.  Ghost cells hold NaN."""
    from test_gpu_stencil_domain import SIZE, domain
    from test_gpu_stencil_domain import load as load_q

    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
    rng = np.random.default_rng(13)
    glob = [rng.standard_normal(SIZE[::-1]) * np.ldexp(1.0, rng.integers(-40, 40, SIZE[::-1])) for _ in range(4)]
    ref = None
    for nsub in (1, 2, 3, 4, 8):
        dd, hs = domain(nsub, sb.Radius.constant(2), [np.float64] * 3, boundary=(F, P, F))
        try:
            load_q(dd, hs[0].id, "curr", glob[0])
            load_q(dd, hs[0].id, "next", glob[3])
            load_q(dd, hs[1].id, "curr", glob[1])
            load_q(dd, hs[2].id, "curr", glob[2])
            res = [bits(r) for r in dd.reduce_many(ITEMS(hs), exact=True)]
            acc = combined_parts(dd, hs)
            if ref is None:
                ref = (res, acc)
            assert (res, acc) == ref, nsub
        finally:
            dd.close()
    want = [xo.reduce_cells(ro.SCALAR, glob[0]), xo.reduce_cells(ro.SCALAR, glob[3]), xo.reduce_cells(ro.DIFF, glob[0], glob[3]),
            xo.reduce_cells(ro.NORM3, *glob[:3])]  # fmt: skip
    for r, w in zip(ref[0], want):
        assert r[2] == struct.pack("<d", w["sum"]) and r[3] == struct.pack("<d", w["sumsq"])
