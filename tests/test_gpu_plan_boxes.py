"""GPU parity of the shared box planner of the operator, system and fused-restriction plans over many boxes: raw bits of
every output allocation against the oracles applied box by box to the arrays as they were before the launch, and
against the single-box plan on the boxes' union, float and double.  The plans: sb_stencil_plan_create (order-8
Laplacian, an asymmetric upwind op, an op with an aux term), sb_stencil_vplan_create (div(kappa grad u), a coefficient
mix), sb_stencil_cplan_create in place (SOR under 2 colours, a 27-point SOR under 8, every colour),
sb_stencil_dplan_create (m = 1 out of place, m = 2 in place), sb_stencil_sys_plan_create (the in-place Yee E update, a
6-input / 4-output mix), sb_transfer_oplan_create and sb_transfer_voplan_create.  The box lists: 16, 17, 32 and 33 thin
boxes with empty boxes among them (second cell-kernel groups), thick and thin boxes from a guillotine partition in two
orders, boxes at the thick threshold, tile-grid remainders, and a thin group of three full grid-stride passes with
pass boundaries inside a box and on a box's first cell.  Every input cell no box reads is NaN, every output cell outside
the boxes is NaN and must stay so; inputs keep their bits; sb_launch_count grows by one per thick box plus one per 16
thin boxes; the plan's bytes are the header's formula summed over the boxes."""
import numpy as np
import pytest
import torch

import colour_oracle as co
import mg_oracle as mo
import stencil_b200 as sb
import stencil_op_oracle as so
import system_oracle as yo
import vmg_oracle as vm
import vstencil_oracle as vo
from gpu_util import DevArray
from stencil_b200._lib import Pitched, check, lib
from test_gpu_colour_op import OPS as COPS
from test_gpu_mg_restrict_op import seven
from test_gpu_stencil_op import OPS as POPS
from test_gpu_system_op import SYSTEMS
from test_gpu_vmg_op import NCOEF, OPS as VMG_OPS
from test_gpu_vstencil_op import OPS as VOPS

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
NONE = Pitched(None, 0, 0)
GROUP = 16  # thin boxes per cell-kernel launch
R0 = (3, -2, 5)  # global lo of every region: boxes start at odd and even global coordinates


def same(a, b):
    return np.array_equal(a.view(UINT[a.dtype]), b.view(UINT[b.dtype]))


def ext_of(b):
    return tuple(b[1][a] - b[0][a] for a in range(3))


def nonempty(boxes):
    return [b for b in boxes if min(ext_of(b)) > 0]


def region_mask(shape, origin, lo, hi):
    """[z, y, x] cells of an array whose element 0 sits at global origin that lie in [lo, hi)."""
    m = np.ones(shape, bool)
    for a in range(3):
        c = np.arange(shape[2 - a]) + origin[a]
        sh = [1, 1, 1]
        sh[2 - a] = shape[2 - a]
        m &= ((c >= lo[a]) & (c < hi[a])).reshape(sh)
    return m


# ------------------------------------------------------------------------------------------- box lists
def shifted(boxes, lo):
    return [(tuple(b[0][a] + lo[a] for a in range(3)), tuple(b[1][a] + lo[a] for a in range(3))) for b in boxes]


def thin_group(n, seed, thick):
    """n thin boxes tiling a region: z layers 1 .. thick - 1 planes thick, each one box 40 cells wide in x (x fastest in
    the cell kernel), or cut in x into two boxes narrower than 32 (y fastest), or cut in y.  3 to 5 empty boxes (lo ==
    hi on one axis) go in between.  Returns (boxes, region extent)."""
    rng = np.random.default_rng(seed)
    X, Y = 40, 12
    out, z = [], 0
    while len(out) < n:
        t = int(rng.integers(1, min(3, thick - 1) + 1))
        kind = "whole" if n - len(out) == 1 else ("whole", "x", "y")[int(rng.integers(0, 3))]
        if kind == "whole":
            out.append(((0, 0, z), (X, Y, z + t)))
        elif kind == "x":
            c = int(rng.integers(9, 32))
            out += [((0, 0, z), (c, Y, z + t)), ((c, 0, z), (X, Y, z + t))]
        else:
            c = int(rng.integers(1, Y))
            out += [((0, 0, z), (X, c, z + t)), ((0, c, z), (X, Y, z + t))]
        z += t
    for _ in range(int(rng.integers(3, 6))):
        p = [int(rng.integers(0, v)) for v in (X, Y, z)]
        a = int(rng.integers(0, 3))
        h = [p[b] if b == a else p[b] + 2 for b in range(3)]
        out.insert(int(rng.integers(0, len(out) + 1)), (tuple(p), tuple(h)))
    return out, (X, Y, z)


def guillotine(seed, thick):
    """3 to 5 thick columns side by side in x, each with thin slabs peeled off random sides until about 20 thin boxes
    exist; the cores stay thick.  Returns (boxes, region extent)."""
    rng = np.random.default_rng(seed)
    ncol = int(rng.integers(3, 6))
    side = 4 * thick
    widths = [int(rng.integers(thick + 4, 5 * thick + 1)) for _ in range(ncol)]
    cores, x = [], 0
    for w in widths:
        cores.append([[x, 0, 0], [x + w, side, side]])
        x += w
    thin = []
    while len(thin) < 20:
        k = int(rng.integers(0, ncol))
        a = int(rng.integers(0, 3))
        lo, hi = cores[k]
        room = hi[a] - lo[a] - thick
        if room < 1:
            continue
        t = int(rng.integers(1, min(3, room, thick - 1) + 1))
        s_lo, s_hi = list(lo), list(hi)
        if rng.integers(0, 2):
            s_hi[a] = lo[a] + t
            lo[a] += t
        else:
            s_lo[a] = hi[a] - t
            hi[a] -= t
        thin.append((tuple(s_lo), tuple(s_hi)))
    return [(tuple(c[0]), tuple(c[1])) for c in cores] + thin, (x, side, side)


def threshold(thick):
    """The cube of side 2 thick - 1 cut at thick on every axis: one box of thick on every axis, three one short of it on
    one axis, and the rest of the cube in three more boxes."""
    t, n = thick, 2 * thick - 1
    return [((0, 0, 0), (t, t, t)), ((t, 0, 0), (n, t, t)), ((0, t, 0), (t, n, t)), ((0, 0, t), (t, t, n)), ((t, t, 0), (n, n, t)),
            ((t, 0, t), (n, n, n)), ((0, t, t), (t, n, n))], (n, n, n)


def grid_stride():
    """x slabs of widths 2, 3, 1 of a region 6 x 4096 x SMs: one cell-kernel group of exactly three grid-stride passes of
    32 x SMs CTAs of 256 threads; box 0 is one pass, so the second pass starts on box 1's first cell and the third inside
    box 1."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert 2 * 4096 * sms == 32 * sms * 256
    out, x = [], 0
    for w in (2, 3, 1):
        out.append(((x, 0, 0), (x + w, 4096, sms)))
        x += w
    return out, (6, 4096, sms)


def box_set(name, thick):
    if name.startswith("group"):
        return thin_group(int(name[5:]), int(name[5:]), thick)
    if name.startswith("mixed"):
        boxes, ext = guillotine(7, thick)
        order = np.random.default_rng(int(name[5:])).permutation(len(boxes))
        return [boxes[i] for i in order], ext
    if name == "threshold":
        return threshold(thick)
    if name == "column":
        return [((0, 0, 0), (thick, thick, 1009))], (thick, thick, 1009)
    if name == "remainders":
        return [((0, 0, 0), (65, 9, 17))], (65, 9, 17)
    assert name == "stride"
    return grid_stride()


SETS = ["group16", "group17", "group32", "group33", "mixed1", "mixed2", "threshold", "column", "remainders"]


def expected_launches(boxes, thick):
    ne = nonempty(boxes)
    nthick = sum(min(ext_of(b)) >= thick for b in ne)
    return nthick + -(-(len(ne) - nthick) // GROUP)


# ------------------------------------------------------------------------------------------- one plan, three ways
def launch(make, boxes):
    """Create, launch once and destroy; returns (launches, bytes)."""
    h, run, nbytes, destroy = make(boxes)
    try:
        n0 = lib().sb_launch_count()
        run(h)
        check(lib().sb_device_sync(0))
        return lib().sb_launch_count() - n0, nbytes(h)
    finally:
        destroy(h)


def stencil_make(op, dst, src, aux, coefs, origin, zsize, colour, omega):
    def make(boxes):
        p = sb.StencilPlan(0, op, dst.pitched(), src.pitched(), aux.pitched() if aux is not None else NONE, origin, zsize, boxes,
                           [k.pitched() for k in coefs] if coefs is not None else None, colour, omega)
        return p, lambda q: q.launch(), lambda q: q.bytes, lambda q: q.destroy()

    return make


def check_plan(make, new_arrays, outputs, inputs, boxes, region, thick, want, want_bytes):
    """make(boxes) on arrays new_arrays() returns; outputs / inputs pick the output and read-only device arrays from them.
    The multi-box plan must give want in every output, leave every input alone, launch as the planner says and count
    want_bytes; the single-box plan on the region must give the same bits."""
    arrs = new_arrays()
    n, nbytes = launch(make(arrs), boxes)
    assert n == expected_launches(boxes, thick)
    assert nbytes == want_bytes
    got = [d.get() for d in outputs(arrs)]
    for j, (g, w) in enumerate(zip(got, want)):
        bad = g.view(UINT[g.dtype]) != w.view(UINT[w.dtype])
        assert not bad.any(), (j, int(bad.sum()), np.argwhere(bad)[:4].tolist())
    for d, a in inputs(arrs):
        assert same(d.get(), a)
    del arrs
    arrs = new_arrays()
    launch(make(arrs), [region])
    for g, d in zip(got, outputs(arrs)):
        assert same(d.get(), g)


# ------------------------------------------------------------------------------------------- operators
def read_masks(terms, shape, origin, region):
    """Cells of src and of each coefficient field the terms read over the region, and the region itself."""
    inreg = region_mask(shape, origin, *region)
    lo = tuple(region[0][a] - origin[a] for a in range(3))
    ext = ext_of(region)
    src, cf = np.zeros(shape, bool), [np.zeros(shape, bool) for _ in range(NCOEF)]
    for t in terms:
        s, o, w, k, c = vo.split(t)
        if s == 0:
            so._view(src, lo, ext, o)[...] = True
        if k >= 0:
            so._view(cf[k], lo, ext, c)[...] = True
    return src, cf, inreg


def colour_cells(b, m, c):
    """The cells of box b of colour c under m, from their global coordinates."""
    e = ext_of(b)
    return int((co.colours(e[::-1], b[0], m) == c).sum())


def run_stencil(kind, dtype, name, colour=None, seed=0):
    """kind: op / vop / sor7 / sor27 / diag1 / diag2."""
    dtype = np.dtype(dtype)
    es = dtype.itemsize
    boxes, rext = box_set(name, 8)
    boxes = shifted(boxes, R0)
    region = (R0, tuple(R0[a] + rext[a] for a in range(3)))
    plain, in_place, omega, m = False, False, None, 1
    if kind.startswith("op:"):
        terms, plain = POPS[kind[3:]], True
    elif kind.startswith("vop:"):
        terms = VOPS[kind[4:]]
    elif kind in ("sor7", "sor27"):
        terms, m = COPS[kind]
        in_place = True
    else:
        terms, omega = VMG_OPS["kappa+sigma"](), 0.8
        m, in_place = (1, False) if kind == "diag1" else (2, True)
    op = sb.StencilOp(terms, dtype)
    rm, rp = vo.reach(terms)
    pad = 5
    origin = tuple(R0[a] - pad for a in range(3))
    shape = tuple(rext[a] + 2 * pad for a in (2, 1, 0))
    rng = np.random.default_rng(seed)
    ms, mc, inreg = read_masks(terms, shape, origin, region)
    u = rng.uniform(-1, 1, shape).astype(dtype)
    u[~ms] = np.nan
    has_aux = op.has_aux or omega is not None
    aux = rng.uniform(-1, 1, shape).astype(dtype) if has_aux else None
    if aux is not None:
        aux[~inreg] = np.nan
    nk = op.ncoef if not plain else 0
    ks = []
    for k in range(nk):
        a = rng.uniform(0.5, 2.0, shape).astype(dtype)
        a[~mc[k]] = np.nan
        ks.append(a)
    dst0 = u if in_place else np.full(shape, np.nan, dtype)
    want = dst0.copy()
    nf = len({vo.split(t)[3] for t in terms} - {-1})
    c = colour if colour is not None else 0
    want_bytes = 0
    for b in nonempty(boxes):
        l, e = tuple(b[0][a] - origin[a] for a in range(3)), ext_of(b)
        if omega is not None:
            vm.diag_box(terms, omega, u, aux, ks, want, l, e, origin, m, c)
        elif m > 1:
            co.apply_box(terms, u, aux, ks, want, l, e, origin, m, c)
        elif plain:
            so.apply_box(terms, u, aux, want, l, e)
        else:
            vo.apply_box(terms, u, aux, ks, want, l, e)
        cells = int(np.prod(e))
        want_bytes += (cells * ((2 if has_aux else 1) + nf) + colour_cells(b, m, c)) * es

    def new_arrays():
        d = {"u": DevArray(u), "aux": DevArray(aux) if aux is not None else None, "ks": [DevArray(k) for k in ks]}
        d["dst"] = d["u"] if in_place else DevArray(dst0)
        return d

    def make(d):
        col = (m, c) if (m > 1 or kind.startswith("sor")) else None
        return stencil_make(op, d["dst"], d["u"], d["aux"], None if plain else d["ks"], origin, shape[0], col, omega)

    def inputs(d):
        out = [(k, a) for k, a in zip(d["ks"], ks)] + ([(d["aux"], aux)] if aux is not None else [])
        return out + ([] if in_place else [(d["u"], u)])

    check_plan(make, new_arrays, lambda d: [d["dst"]], inputs, boxes, region, 8, [want], want_bytes)


STENCIL_KINDS = ["op:lap8", "op:upwind", "op:aux", "vop:div_grad", "vop:mix", "diag1"]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("kind", STENCIL_KINDS)
def test_stencil_boxes(kind, name, dtype):
    run_stencil(kind, dtype, name, seed=len(name))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("kind", ["sor7", "sor27", "diag2"])
def test_coloured_boxes_every_colour(kind, name, dtype):
    m = 8 if kind == "sor27" else 2
    for c in range(m):
        run_stencil(kind, dtype, name, colour=c, seed=c)


# ------------------------------------------------------------------------------------------- systems
def run_system(sysname, dtype, name, seed=0):
    dtype = np.dtype(dtype)
    es = dtype.itemsize
    terms, nin, alias = SYSTEMS[sysname]
    nout = yo.nout_of(terms)
    boxes, rext = box_set(name, 8)
    boxes = shifted(boxes, R0)
    region = (R0, tuple(R0[a] + rext[a] for a in range(3)))
    pad = 3
    origin = tuple(R0[a] - pad for a in range(3))
    shape = tuple(rext[a] + 2 * pad for a in (2, 1, 0))
    lo, ext = tuple(R0[a] - origin[a] for a in range(3)), rext
    rng = np.random.default_rng(seed)
    ins = []
    for i in range(nin):
        mk = np.zeros(shape, bool)
        for t in terms:
            j, ii, o, w, k, c = yo.split(t)
            if ii == i:
                so._view(mk, lo, ext, o)[...] = True
            if k == i:
                so._view(mk, lo, ext, c)[...] = True
        a = rng.uniform(0.5, 2.0, shape).astype(dtype) if i >= 4 else rng.uniform(-1, 1, shape).astype(dtype)
        a[~mk] = np.nan
        ins.append(a)
    outs0 = [ins[alias[j]] if j in alias else np.full(shape, np.nan, dtype) for j in range(nout)]
    want = [o.copy() for o in outs0]
    for b in nonempty(boxes):
        yo.apply_box(terms, ins, want, tuple(b[0][a] - origin[a] for a in range(3)), ext_of(b))
    want_bytes = sum(int(np.prod(ext_of(b))) for b in nonempty(boxes)) * es * (len(yo.reads(terms)) + nout)

    def new_arrays():
        d_in = [DevArray(a) for a in ins]
        return {"in": d_in, "out": [d_in[alias[j]] if j in alias else DevArray(outs0[j]) for j in range(nout)]}

    def make(d):
        def mk(boxes):
            p = sb.SystemPlan(0, sb.StencilSystem(terms, dtype, nin=nin), [o.pitched() for o in d["out"]], [i.pitched() for i in d["in"]], origin,
                              shape[0], boxes)
            return p, lambda q: q.launch(), lambda q: q.bytes, lambda q: q.destroy()

        return mk

    aliased = set(alias.values())
    check_plan(make, new_arrays, lambda d: d["out"], lambda d: [(d["in"][i], ins[i]) for i in range(nin) if i not in aliased], boxes, region, 8,
               want, want_bytes)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("sysname", ["yee_e", "mix"])
def test_system_boxes(sysname, name, dtype):
    run_system(sysname, dtype, name, seed=len(name))


# ------------------------------------------------------------------------------------------- fused restriction
FUSED = {"7pt": seven, "7pt-noaux": lambda: [t for t in seven() if t[0] == 0], "kappa": lambda: vm.vresidual_terms(VMG_OPS["kappa+sigma"]())}


def run_fused(opname, dtype, name, seed=0):
    dtype = np.dtype(dtype)
    es = dtype.itemsize
    terms = FUSED[opname]()
    op = sb.StencilOp(terms, dtype)
    boxes, rext = box_set(name, 4)
    boxes = shifted(boxes, R0)
    lo, hi = R0, tuple(R0[a] + rext[a] for a in range(3))
    rng = np.random.default_rng(seed)
    pad = (2, 1, 3)
    so_ = tuple(2 * lo[a] - 1 - pad[a] for a in range(3))
    sshape = tuple(2 * rext[a] + 2 + 2 * pad[a] for a in (2, 1, 0))
    offs = [t[1] for t in terms if t[0] == 0]
    src = rng.uniform(-1, 1, sshape).astype(dtype)
    src[~region_mask(sshape, so_, [2 * lo[a] + min(o[a] for o in offs) for a in range(3)],
                     [2 * hi[a] + max(o[a] for o in offs) for a in range(3)])] = np.nan
    has_aux = op.has_aux
    aux = rng.uniform(-1, 1, sshape).astype(dtype) if has_aux else None
    if has_aux:
        aux[~region_mask(sshape, so_, [2 * v for v in lo], [2 * v for v in hi])] = np.nan
    nf = op.ncoef
    ks = []
    for k in range(nf):
        c_ = [vo.split(t)[4] for t in terms if vo.split(t)[3] == k] or [(0, 0, 0)]
        arr = rng.uniform(0.5, 1.5, sshape).astype(dtype)
        arr[~region_mask(sshape, so_, [2 * lo[a] + min(o[a] for o in c_) for a in range(3)], [2 * hi[a] + max(o[a] for o in c_) for a in range(3)])] = np.nan
        ks.append(arr)
    do = tuple(lo[a] - 1 for a in range(3))
    dshape = tuple(rext[a] + 3 for a in (2, 1, 0))
    dst0 = np.full(dshape, np.nan, dtype)
    want = dst0.copy()
    for b in nonempty(boxes):
        if nf:
            vm.restrict_vop_box(want, do, terms, src, aux, ks, so_, b[0], b[1])
        else:
            mo.restrict_op_box(want, do, terms, src, aux, so_, b[0], b[1])
    nfields = len({vo.split(t)[3] for t in terms} - {-1})
    want_bytes = sum(int(np.prod(ext_of(b))) for b in nonempty(boxes)) * es * (8 * ((2 if has_aux else 1) + nfields) + 1)

    def new_arrays():
        return {"dst": DevArray(dst0), "src": DevArray(src), "aux": DevArray(aux) if has_aux else None, "ks": [DevArray(k) for k in ks]}

    def make(d):
        def mk(boxes):
            p = sb.TransferPlan.fused(0, op, d["dst"].pitched(), do, dshape[0], d["src"].pitched(), so_, sshape[0],
                                      d["aux"].pitched() if has_aux else None, boxes, [k.pitched() for k in d["ks"]] if nf else None)
            return p, lambda q: q.launch(), lambda q: q.bytes, lambda q: q.destroy()

        return mk

    def inputs(d):
        return [(d["src"], src)] + ([(d["aux"], aux)] if has_aux else []) + list(zip(d["ks"], ks))

    check_plan(make, new_arrays, lambda d: [d["dst"]], inputs, boxes, (lo, hi), 4, [want], want_bytes)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("opname", ["7pt", "kappa"])
def test_fused_restriction_boxes(opname, name, dtype):
    run_fused(opname, dtype, name, seed=len(name))


# ------------------------------------------------------------------------------------------- grid-stride passes
@pytest.mark.parametrize("kind", ["op:lap8", "vop:div_grad", "sor7", "diag2", "sys:yee_e", "fused:7pt-noaux"])
def test_grid_stride_passes(kind):
    """Three full passes of the cell kernels' grid-stride loop, in FP32 (FP64 too for the plain op)."""
    if kind.startswith("sys:"):
        run_system(kind[4:], np.float32, "stride")
    elif kind.startswith("fused:"):
        run_fused(kind[6:], np.float32, "stride")
    else:
        for dtype in ([np.float32, np.float64] if kind == "op:lap8" else [np.float32]):
            run_stencil(kind, dtype, "stride", colour=1 if kind in ("sor7", "diag2") else None)


# ------------------------------------------------------------------------------------------- only empty boxes
def test_only_empty_boxes():
    """A list of empty boxes gives plans with no launch and 0 bytes, and writes nothing."""
    empty = [((1, 1, 1), (1, 3, 3)), ((2, 2, 2), (4, 2, 4)), ((0, 0, 0), (5, 5, 0))]
    shape = (8, 8, 8)
    a, b = DevArray(np.zeros(shape)), DevArray(np.full(shape, np.nan))
    op = sb.StencilOp(POPS["7pt"], np.float64)
    plans = [
        lambda: sb.StencilPlan(0, op, b.pitched(), a.pitched(), NONE, (0, 0, 0), 8, empty),
        lambda: sb.SystemPlan(0, sb.StencilSystem([(0, 0, (1, 0, 0), 1.0)], np.float64), [b.pitched()], [a.pitched()], (0, 0, 0), 8, empty),
        lambda: sb.TransferPlan.fused(0, sb.StencilOp(FUSED["7pt-noaux"](), np.float64), b.pitched(), (0, 0, 0), 8, a.pitched(), (-1, -1, -1), 8, None,
                                      empty),
    ]
    for mk in plans:
        p = mk()
        try:
            assert p.bytes == 0
            n0 = lib().sb_launch_count()
            p.launch()
            check(lib().sb_device_sync(0))
            assert lib().sb_launch_count() == n0
        finally:
            p.destroy()
    assert np.isnan(b.get()).all()
