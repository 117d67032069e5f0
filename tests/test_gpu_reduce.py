"""Reductions on the GPU against the oracle (tests/reduce_oracle.py): min and max bit for bit, sums within the bound of
DESIGN section 2.6.  Ghost cells hold NaN and 1e300, so a reduction that read one would fail."""
import ctypes as C
import math
import struct

import numpy as np
import pytest

import reduce_oracle as ro
import stencil_b200 as sb
from gpu_util import DevArray
from stencil_b200 import _lib
from stencil_b200.astaroth import FIELDS, Astaroth, conf_params
from stencil_b200.jacobi import Jacobi3D, jacobi_radius

pytestmark = pytest.mark.gpu


def assert_matches(got: sb.Reduction, want: dict, rows: int, nsub: int = 1, nx: int = 0, es: int = 8):
    """min / max bit for bit, sums within the bound; nx, es: the widest box row and the element size (they fix k)."""
    k = ro.chain_len(nx, es)
    for f in ("min", "max"):
        g, w = getattr(got, f), want[f]
        assert (math.isnan(g) and math.isnan(w)) or struct.pack("<d", g) == struct.pack("<d", w) or (g == w == 0.0), (f, g, w)
    assert got.count == want["count"]
    for f, a in (("sum", "abs_sum"), ("sumsq", "abs_sumsq")):
        g, w = getattr(got, f), want[f]
        if math.isnan(w):
            assert math.isnan(g), (f, g)
        else:
            assert abs(g - w) <= ro.bound(want[a], rows, nsub, k), (f, g, w, ro.bound(want[a], rows, nsub, k))


def load(dd, h, glob, which="curr", poison=math.nan):
    """Scatter the global [z, y, x] field into every local subdomain's `which` buffer; ghost cells = poison."""
    for d in dd.domains():
        dt = dd.dtypes_[h.id]
        host = np.full(tuple(reversed(d.raw_size())), min(poison, float(np.finfo(dt).max)) if poison == poison else poison, dtype=dt)
        p, o, sz = d.halo_pos((0, 0, 0), True), d.origin(), d.size()
        host[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]] = glob[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]]
        d.quantity_from_host(h.id, host, which)


def make_domain(size, radius, dtype, nsub, nq):
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([0] * nsub)
    dd.set_radius(radius)
    hs = [dd.add_data(dtype) for _ in range(nq)]
    dd.realize()
    return dd, hs


def fields(size, dtype, n, seed):
    rng = np.random.default_rng(seed)
    return [(rng.standard_normal(tuple(reversed(size))) * 3.0).astype(dtype) for _ in range(n)]


def check_all_kinds(dd, hs, size, nsub):
    """scalar (curr and next), diff and norm of four loaded fields, in one plan."""
    dt = dd.dtypes_[hs[0].id]
    a, b, c, nx = fields(size, dt, 4, seed=7 + nsub)
    load(dd, hs[0], a)
    load(dd, hs[0], nx, "next", poison=1e300)
    load(dd, hs[1], b, poison=1e300)
    load(dd, hs[2], c)
    got = dd.reduce_many([("scalar", hs[0]), ("scalar", hs[0], "next"), ("diff", hs[0]), ("norm", hs[0], hs[1], hs[2])])
    rows, w, es = size[1] * size[2], size[0], np.dtype(dt).itemsize
    assert_matches(got[0], ro.reduce_cells(ro.SCALAR, a), rows, nsub, w, es)
    assert_matches(got[1], ro.reduce_cells(ro.SCALAR, nx), rows, nsub, w, es)
    assert_matches(got[2], ro.reduce_cells(ro.DIFF, a, nx), rows, nsub, w, es)
    assert_matches(got[3], ro.reduce_cells(ro.NORM3, a, b, c), rows, nsub, w, es)
    if dt == np.float32:  # every q of an FP32 scalar is exact, and so are these sums' terms
        assert got[0].sumsq == pytest.approx(math.fsum((a.astype(np.float64) ** 2).ravel().tolist()), rel=300 * ro.U)


def asymmetric_radius() -> sb.Radius:
    """1 cell on -x, 3 on +x, 2 on -y, none elsewhere."""
    r = sb.Radius.constant(0)
    r.set_dir((-1, 0, 0), 1)
    r.set_dir((1, 0, 0), 3)
    r.set_dir((0, -1, 0), 2)
    return r


RADII = {"r0": lambda: sb.Radius.constant(0), "r1": lambda: sb.Radius.constant(1), "r2": lambda: sb.Radius.constant(2),
         "r3": lambda: sb.Radius.constant(3), "asym": asymmetric_radius}  # fmt: skip


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("rname", list(RADII))
def test_layouts(dtype, rname):
    r = RADII[rname]()
    size = (37, 11, 9)
    dd, hs = make_domain(size, r, dtype, 1, 3)
    try:
        check_all_kinds(dd, hs, size, 1)
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_unaligned_allocations(dtype, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    size = (29, 13, 7)
    dd, hs = make_domain(size, 1, dtype, 2, 3)
    try:
        check_all_kinds(dd, hs, size, 2)
    finally:
        dd.close()


@pytest.mark.parametrize("nsub", [1, 4, 8])
def test_subdomains(nsub):
    size = (41, 23, 19)
    dd, hs = make_domain(size, 2, np.float64, nsub, 3)
    try:
        check_all_kinds(dd, hs, size, nsub)
    finally:
        dd.close()


def plan_of(items):
    return sb.ReducePlan(0, items)


def cabi_item(kind, dtype, arrs, lo, hi):
    src = (_lib.Pitched * 3)(*[a.pitched() for a in arrs] + [arrs[0].pitched()] * (3 - len(arrs)))
    return _lib.ReduceItem(kind, 1 if dtype == np.float32 else 2, src, _lib.I3(0, 0, 0), _lib.I3(*lo), _lib.I3(*hi))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_narrow_and_mid_vector_boxes_through_the_c_abi(dtype):
    """Boxes 1-3 cells wide and boxes that start mid-vector, on rows whose 16-byte phase alternates (odd x extents)."""
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
        plan = plan_of(items)
        plan.launch()
        got = plan.results()
        for (kind, lo, hi, n), g in zip(cases, got):
            box = [h[lo[2] : hi[2], lo[1] : hi[1], lo[0] : hi[0]] for h in hosts[:n]]
            assert_matches(g, ro.reduce_cells(kind, *box), 4 * 5, 1, hi[0] - lo[0], np.dtype(dtype).itemsize)
        plan.destroy()
        # sources whose 16-byte phases differ (one element apart) take the element-wise path
        base = DevArray(hosts[0], extra=64)
        shifted = _lib.Pitched(base.ptr + np.dtype(dtype).itemsize, base.pitched().pitch, base.pitched().ysize)
        src = (_lib.Pitched * 3)(base.pitched(), shifted, base.pitched())
        it = _lib.ReduceItem(ro.DIFF, 1 if dtype == np.float32 else 2, src, _lib.I3(0, 0, 0), _lib.I3(0, 0, 0), _lib.I3(40, 7, 6))
        plan = plan_of([it])
        plan.launch()
        g = plan.results()[0]
        flat = hosts[0].ravel()
        sh = np.concatenate([flat[1:], flat[:1]]).reshape(shape)  # element p + 1 (the last one lies in the padding)
        want = ro.reduce_cells(ro.DIFF, hosts[0][:, :, :40], sh[:, :, :40])
        assert_matches(g, want, 42, 1, 40, np.dtype(dtype).itemsize)
        plan.destroy()
        base.free()
    finally:
        for a in arrs:
            a.free()


def test_rows_wider_than_one_tile_pass():
    """Rows of 20000 FP64 cells: one block pass per tile and a chain longer than kRedChain (the bound uses the planner's k)."""
    rng = np.random.default_rng(9)
    hosts = [rng.standard_normal((2, 3, 20000)) for _ in range(2)]
    arrs = [DevArray(h) for h in hosts]
    try:
        plan = plan_of([cabi_item(ro.SCALAR, np.float64, arrs[:1], (1, 0, 0), (20000, 3, 2)), cabi_item(ro.DIFF, np.float64, arrs, (0, 0, 0), (19999, 3, 2))])
        plan.launch()
        g = plan.results()
        assert ro.chain_len(19999, 8) > ro.CHAIN
        assert_matches(g[0], ro.reduce_cells(ro.SCALAR, hosts[0][:, :, 1:]), 6, 1, 19999, 8)
        assert_matches(g[1], ro.reduce_cells(ro.DIFF, hosts[0][:, :, :19999], hosts[1][:, :, :19999]), 6, 1, 19999, 8)
        plan.destroy()
    finally:
        for a in arrs:
            a.free()


def test_null_output_buffer_at_launch():
    a = DevArray(np.zeros((2, 2, 4)))
    try:
        plan = plan_of([cabi_item(ro.SCALAR, np.float64, [a], (0, 0, 0), (4, 2, 2))])
        with pytest.raises(sb.StencilError, match="null output buffer"):
            sb._lib.check(sb.lib().sb_reduce_plan_launch(plan._h, None, None))
        plan.destroy()
    finally:
        a.free()


def test_empty_box_and_single_nan():
    size = (16, 8, 8)
    dd, hs = make_domain(size, 1, np.float64, 2, 1)
    try:
        glob = fields(size, np.float64, 1, 1)[0]
        glob[3, 5, 7] = math.nan
        load(dd, hs[0], glob)
        r = dd.reduce(hs[0])
        assert math.isnan(r.min) and math.isnan(r.max) and math.isnan(r.sum) and r.count == 16 * 8 * 8
        d = dd.domains()[0]
        lo, _ = d.get_compute_region()
        plan = plan_of([_lib.ReduceItem(ro.SCALAR, 2, (_lib.Pitched * 3)(*[d.curr_data(0)] * 3), _lib.I3(*d.accessor_origin()), _lib.I3(*lo), _lib.I3(*lo))])
        plan.launch()
        e = plan.results()[0]
        assert (e.min, e.max, e.sum, e.sumsq, e.count) == (math.inf, -math.inf, 0.0, 0.0, 0)
        plan.destroy()
    finally:
        dd.close()


def test_reduce_after_swap_reads_the_new_curr():
    size = (24, 16, 12)
    dd, hs = make_domain(size, 1, np.float32, 2, 1)
    try:
        a, b = fields(size, np.float32, 2, 5)
        load(dd, hs[0], a)
        load(dd, hs[0], b, "next")
        r0 = dd.reduce(hs[0])
        dd.swap()
        r1 = dd.reduce(hs[0])
        rn = dd.reduce(hs[0], "next")
        assert_matches(r0, ro.reduce_cells(ro.SCALAR, a), 16 * 12, 2)
        assert_matches(r1, ro.reduce_cells(ro.SCALAR, b), 16 * 12, 2)
        assert rn == r0
        dd.swap()
        assert dd.reduce(hs[0]) == r0
    finally:
        dd.close()


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
        plan = plan_of(items)
        s = torch.cuda.Stream()
        runs = []
        for _ in range(3):
            plan.launch(s)
            runs.append(plan.results(s))
        assert runs[0] == runs[1] == runs[2]
        check = [struct.pack("<4dq", r.min, r.max, r.sum, r.sumsq, r.count) for r in runs[0]]
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            plan.launch(s)
        _lib.check(sb.lib().sb_memset(C.c_void_p(plan.out_dev), 0, 3 * C.sizeof(_lib.ReduceResult), 0, None))
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            g.replay()
        after = plan.results(s)
        assert [struct.pack("<4dq", r.min, r.max, r.sum, r.sumsq, r.count) for r in after] == check
        # the domain-level call gives the same bits for the same items
        assert dd.reduce_many([("scalar", hs[0]), ("diff", hs[0])])[0] == runs[0][0]
        plan.destroy()
    finally:
        dd.close()


def test_512_cubed_fp64_exact_sums():
    """512^3 FP64 at radius 1: integer multiples of 2^-10 below 2^2 in magnitude, so every sum is exact in any order
    and must equal the integer sum bit for bit."""
    size = (512, 512, 512)
    dd, hs = make_domain(size, 1, np.float64, 1, 1)
    try:
        rng = np.random.default_rng(0)
        ints = rng.integers(-(2**11), 2**11, size=(512, 512, 512), dtype=np.int64)
        load(dd, hs[0], ints.astype(np.float64) * 2.0**-10)
        r = dd.reduce(hs[0])
        assert r.count == 512**3
        assert r.min == ints.min() * 2.0**-10 and r.max == ints.max() * 2.0**-10
        assert r.sum == float(ints.sum()) * 2.0**-10
        assert r.sumsq == float((ints * ints).sum()) * 2.0**-20
    finally:
        dd.close()


@pytest.mark.parametrize("schedule", ["step", "step_async", "step_fused"])
def test_jacobi_residual(schedule):
    n = 48
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0, 0])
    dd.set_radius(jacobi_radius())
    h = dd.add_data(np.float64)
    dd.realize()
    try:
        jac = Jacobi3D(dd, h)
        jac.init(0.5)
        for _ in range(10):
            getattr(jac, schedule)()
        res = jac.residual()  # no synchronize first: the reduction orders after the queued iterations
        jac.synchronize()
        diffs = []
        for d in dd.domains():
            c = d.interior_to_host(0)
            full = d.quantity_to_host(0, "next")
            p, sz = d.halo_pos((0, 0, 0), True), d.size()
            nx = full[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]]
            diffs.append(((c - nx) ** 2).ravel())
        sq = np.concatenate(diffs)
        want = math.sqrt(math.fsum(sq.tolist()))
        assert res > 0 and abs(res * res - want * want) <= ro.bound(want * want, n * n, 2, ro.chain_len(n, 8))
        # the difference is symmetric; the scalar reductions pin which buffer is curr after this schedule
        glob = {w: np.empty((n, n, n)) for w in ("curr", "next")}
        for d in dd.domains():
            o, sz, p = d.origin(), d.size(), d.halo_pos((0, 0, 0), True)
            for w in glob:
                full = d.quantity_to_host(0, w)
                glob[w][o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]] = full[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]]
        assert not np.array_equal(glob["curr"], glob["next"])
        for w in glob:
            assert_matches(dd.reduce(h, w), ro.reduce_cells(ro.SCALAR, glob[w]), n * n, 2, n, 8)
        jac.close()
    finally:
        dd.close()


def test_astaroth_diagnostics():
    size = (24, 20, 16)
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([0, 0])
    dd.set_radius(3)
    hs = [dd.add_data(np.float64, nm) for nm in FIELDS]
    dd.realize()
    try:
        rng = np.random.default_rng(2)
        for q, h in enumerate(hs):
            load(dd, h, rng.uniform(-0.5, 0.5, tuple(reversed(size))) + (1.0 if q == 0 else 0.0))
            load(dd, h, np.zeros(tuple(reversed(size))), "next")
        sim = Astaroth(dd, hs, conf_params(1e-3))
        sim.step()
        diag = sim.diagnostics()
        assert list(diag) == list(FIELDS) + ["uu", "aa"]
        glob = [np.empty(tuple(reversed(size))) for _ in range(8)]
        for d in dd.domains():
            o, sz = d.origin(), d.size()
            for q in range(8):
                glob[q][o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]] = d.interior_to_host(q)
        rows = size[1] * size[2]
        for q, name in enumerate(FIELDS):
            assert_matches(diag[name], ro.reduce_cells(ro.SCALAR, glob[q]), rows, 2)
            want_rms = math.sqrt(math.fsum((glob[q] ** 2).ravel().tolist()) / glob[q].size)
            assert diag[name].rms() == pytest.approx(want_rms, rel=1e-12)
        for name, (i, j, k) in (("uu", (1, 2, 3)), ("aa", (4, 5, 6))):
            assert_matches(diag[name], ro.reduce_cells(ro.NORM3, glob[i], glob[j], glob[k]), rows, 2)
            mag2 = glob[i] ** 2 + glob[j] ** 2 + glob[k] ** 2
            assert diag[name].max == float(np.sqrt(mag2).max())
            assert diag[name].rms() == pytest.approx(math.sqrt(mag2.mean()), rel=1e-12)
        sim.synchronize()
    finally:
        dd.close()
