"""GPU parity of linear stencil systems through the C ABI (sb_stencil_sys_plan_create): raw bits of every output allocation
against the numpy rule of tests/system_oracle.py, float and double -- grad, div and curl at each stagger, the in-place Yee
E and H updates, and a 6-input / 4-output mix with coefficient terms -- on the shapes of test_gpu_stencil_op.py, with
different allocation leads across the buffers.  Every input cell outside that input's own reach is NaN, and every output
cell outside the box must stay NaN.  Single-output systems give the bits of sb_stencil_vplan_create."""
import numpy as np
import pytest

import stencil_b200 as sb
import stencil_op_oracle as so
import system_oracle as yo
import vstencil_oracle as vo
from gpu_util import DevArray
from stencil_b200._lib import Pitched, check, lib
from test_gpu_stencil_op import SHAPES
from test_gpu_vstencil_op import OPS as VOPS

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
ACC = (-3, 5, 7)
H = (0.5, 0.25, 0.5)


def yee_e(c=0.3):
    """E = E + c curl- H in place: inputs Hx, Hy, Hz, Ex, Ey, Ez; outputs Ex, Ey, Ez (inputs 3..5)."""
    return [(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)] + yo.scaled(yo.curl(-1, H), c)


def yee_h(c=0.3):
    """H = H - c curl+ E in place: inputs Ex, Ey, Ez, Hx, Hy, Hz; outputs Hx, Hy, Hz (inputs 3..5)."""
    return [(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)] + yo.scaled(yo.curl(1, H), -c)


def mix(seed=0):
    """6 inputs, 4 outputs, terms of different outputs interleaved, reach up to 2, coefficient terms on inputs 4 and 5."""
    rng = np.random.default_rng(seed)
    dirs = [(x, y, z) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]
    terms = []
    for t in range(40):
        j, i = t % 4, int(rng.integers(0, 6))
        o = tuple(int(v) for v in rng.integers(-2, 3, 3)) if t % 3 else (0, 0, 0)
        w = float(rng.uniform(-1, 1))
        terms.append((j, i, o, w, 4 + t % 2, dirs[t % 27]) if t % 5 == 1 else (j, i, o, w))
    return terms


SYSTEMS = {
    "grad+": (yo.grad(1, H), 1, {}),
    "grad0": (yo.grad(0, H), 1, {}),
    "div-": (yo.div(-1, H), 3, {}),
    "curl+": (yo.curl(1, H), 3, {}),
    "curl0": (yo.curl(0, H), 3, {}),
    "yee_e": (yee_e(), 6, {0: 3, 1: 4, 2: 5}),
    "yee_h": (yee_h(), 6, {0: 3, 1: 4, 2: 5}),
    "mix": (mix(), 6, {}),
}


def run_sys(terms, nin, alias, dtype, ext, leads=(0,), extra=0, seed=0):
    """alias: output j -> the input it is (read only at offset 0).  leads: bytes before element 0, by buffer in turn."""
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(seed)
    nout = yo.nout_of(terms)
    R = [max(max(yo.reach(terms, i)[s][a] for i in range(nin)) for s in (0, 1)) for a in range(3)]
    lo = tuple(R[a] + extra for a in range(3))
    raw = tuple(ext[a] + 2 * R[a] + 2 * extra for a in range(3))
    shape = raw[::-1]
    ins = []
    for i in range(nin):
        m = np.zeros(shape, bool)
        for t in terms:
            j, ii, o, w, k, c = yo.split(t)
            if ii == i:
                so._view(m, lo, ext, o)[...] = True
            if k == i:
                so._view(m, lo, ext, c)[...] = True
        a = rng.uniform(0.5, 2.0, shape).astype(dtype) if i >= 4 else rng.uniform(-1, 1, shape).astype(dtype)
        a[~m] = np.nan
        ins.append(a if m.any() else None)
    outs = [ins[alias[j]] if j in alias else np.full(shape, np.nan, dtype) for j in range(nout)]
    want_ins = [a.copy() if a is not None else None for a in ins]
    want = [want_ins[alias[j]] if j in alias else np.full(shape, np.nan, dtype) for j in range(nout)]
    yo.apply_box(terms, want_ins, want, lo, ext)
    k = 0
    d_in = []
    for a in ins:
        d_in.append(DevArray(a, lead=leads[k % len(leads)]) if a is not None else None)
        k += 1
    d_out = []
    for j in range(nout):
        d_out.append(d_in[alias[j]] if j in alias else DevArray(outs[j], lead=leads[k % len(leads)]))
        k += 1
    glo = tuple(lo[a] + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    system = sb.StencilSystem(terms, dtype, nin=nin)
    plan = sb.SystemPlan(0, system, [d.pitched() for d in d_out], [d.pitched() if d is not None else Pitched(None, 0, 0) for d in d_in], ACC,
                         raw[2], [(glo, ghi)])
    try:
        nread = sum(a is not None for a in ins)
        assert plan.bytes == int(np.prod(ext)) * dtype.itemsize * (nread + nout)
        plan.launch()
        check(lib().sb_device_sync(0))
        got = [d.get() for d in d_out]
        got_in = [d.get() if d is not None else None for d in d_in]
    finally:
        plan.destroy()
    u = UINT[dtype]
    for j in range(nout):
        bad = got[j].view(u) != want[j].view(u)
        assert not bad.any(), (j, int(bad.sum()), np.argwhere(bad)[:4].tolist())
    for i, (g, w) in enumerate(zip(got_in, want_ins)):
        if g is not None:
            assert np.array_equal(g.view(u), w.view(u)), i


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", list(SYSTEMS))
@pytest.mark.parametrize("si", range(len(SHAPES)))
def test_system_bits(name, dtype, si):
    terms, nin, alias = SYSTEMS[name]
    es = np.dtype(dtype).itemsize
    leads = tuple((es * (si + k)) % 16 for k in range(4))
    run_sys(terms, nin, alias, dtype, SHAPES[si], leads=leads, extra=si % 2, seed=si)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("lead", [0, 4, 8, 12])
@pytest.mark.parametrize("name", ["curl+", "yee_e", "mix"])
def test_system_leads(name, dtype, lead):
    if np.dtype(dtype).itemsize == 8 and lead % 8:
        pytest.skip("an FP64 allocation starts on an 8-byte boundary")
    terms, nin, alias = SYSTEMS[name]
    for extra in (0, 2):
        run_sys(terms, nin, alias, dtype, (45, 19, 17), leads=(lead, (lead + 8) % 16, lead), extra=extra, seed=lead + extra)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("xsize", [62, 63, 65])
def test_alternating_row_phase(dtype, xsize):
    """Rows whose pitch is not a multiple of 16 bytes: the element path for every input."""
    terms, nin, alias = SYSTEMS["yee_h"]
    run_sys(terms, nin, alias, dtype, (xsize, 21, 19), leads=(np.dtype(dtype).itemsize, 0), seed=xsize)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_output_aliases_input_read_by_another_output(dtype):
    """Output 0 is input 2, which output 1 also reads at offset 0 (every read happens before the write)."""
    terms = [(0, 0, (1, 0, 0), 0.5), (0, 2, (0, 0, 0), 1.0), (1, 2, (0, 0, 0), -2.0), (1, 1, (0, -1, 1), 0.25), (0, 1, (0, 0, 0), 3.0)]
    for shape in ((37, 29, 23), (1, 17, 9)):
        run_sys(terms, 3, {0: 2}, dtype, shape, leads=(8, 0), seed=7)


def as_system(terms):
    """A single-output op of test_gpu_vstencil_op.py as a system: src = input 0, aux = input 1, field k = input 2 + k."""
    out = []
    for t in terms:
        s, o, w, k, c = vo.split(t)
        out.append((0, s, o, w, 2 + k, c) if k >= 0 else (0, s, o, w))
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("op", list(VOPS))
def test_single_output_matches_vplan(op, dtype):
    dtype = np.dtype(dtype)
    terms = VOPS[op]
    vop = sb.StencilOp(terms, dtype)
    rng = np.random.default_rng(11)
    ext = (70, 20, 18)
    shape = tuple(e + 4 for e in ext)[::-1]
    src, aux = rng.uniform(-1, 1, shape).astype(dtype), rng.uniform(-1, 1, shape).astype(dtype)
    coefs = [rng.uniform(0.5, 2, shape).astype(dtype) for _ in range(4)]
    d_src, d_aux = DevArray(src, lead=8), DevArray(aux)
    d_c = [DevArray(c, lead=(8 * k) % 16) for k, c in enumerate(coefs)]
    r = sb.Radius.constant(2)
    glo = tuple(2 + ACC[a] for a in range(3))
    ghi = tuple(glo[a] + ext[a] for a in range(3))
    import ctypes as C

    ilo, ihi = (C.c_int64 * 3)(), (C.c_int64 * 3)()
    check(lib().sb_interior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), ilo, ihi))
    elo, ehi = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    ne = check(lib().sb_exterior((C.c_int64 * 3)(*glo), (C.c_int64 * 3)(*ghi), r.c27(), elo, ehi))
    cut = [(tuple(ilo), tuple(ihi))] + [(tuple(elo[3 * k : 3 * k + 3]), tuple(ehi[3 * k : 3 * k + 3])) for k in range(ne)]
    outs = []
    d_dst = DevArray(np.full(shape, np.nan, dtype))
    plan = sb.StencilPlan(0, vop, d_dst.pitched(), d_src.pitched(), d_aux.pitched(), ACC, shape[0], cut, [c.pitched() for c in d_c[: vop.ncoef]])
    plan.launch()
    check(lib().sb_device_sync(0))
    outs.append(d_dst.get())
    plan.destroy()
    d_dst = DevArray(np.full(shape, np.nan, dtype))
    system = sb.StencilSystem(as_system(terms), dtype, nin=6)
    plan = sb.SystemPlan(0, system, [d_dst.pitched()], [d_src.pitched(), d_aux.pitched()] + [c.pitched() for c in d_c], ACC, shape[0], cut)
    plan.launch()
    check(lib().sb_device_sync(0))
    outs.append(d_dst.get())
    plan.destroy()
    u = UINT[dtype]
    assert np.array_equal(outs[0].view(u), outs[1].view(u))


def test_512_fp64_curl():
    """One 512^3 FP64 forward curl, bit-identical to the oracle."""
    n = 512
    shape = (n + 2,) * 3
    rng = np.random.default_rng(512)
    ins = [rng.uniform(-1, 1, shape) for _ in range(3)]
    d_in = [DevArray(a) for a in ins]
    d_out = [DevArray(np.zeros(shape)) for _ in range(3)]
    plan = sb.SystemPlan(0, sb.StencilSystem.curl(1, H, np.float64), [d.pitched() for d in d_out], [d.pitched() for d in d_in], (0, 0, 0),
                         shape[0], [((1, 1, 1), (1 + n, 1 + n, 1 + n))])
    plan.launch()
    got = [d.get() for d in d_out]
    plan.destroy()
    for d in d_in + d_out:
        d.free()
    want = [np.zeros(shape) for _ in range(3)]
    yo.apply_box(yo.curl(1, H), ins, want, (1, 1, 1), (n, n, n))
    for g, w in zip(got, want):
        assert np.array_equal(g.view(np.uint64), w.view(np.uint64))


def test_shared_memory_limit():
    """8 inputs read at reach 4 on every axis need more shared memory than a block may have: an error that gives the bytes."""
    terms = [(0, i, (4 * (-1) ** i, 4, -4), 1.0) for i in range(8)] + [(0, i, (-4 * (-1) ** i, -4, 4), 1.0) for i in range(8)]
    shape = (20, 20, 80)
    d_in = [DevArray(np.zeros(shape)) for _ in range(8)]
    d_out = DevArray(np.zeros(shape))
    with pytest.raises(sb.StencilError, match=r"needs \d+ bytes of shared memory per block, the device allows \d+"):
        sb.SystemPlan(0, sb.StencilSystem(terms, np.float64), [d_out.pitched()], [d.pitched() for d in d_in], (0, 0, 0), shape[0],
                      [((4, 4, 4), (76, 16, 16))])
