"""The jacobi kernels against the C oracle at every allocation phase, row remainder and neighbour layout, bit for bit over
whole allocations: sb_jacobi3d / sb_jacobi3d_regions on raw buffers, sb_jacobi3d_fused through its C ABI (pushes, in-place
wraps and dense x arrays checked cell by cell), and the three Jacobi3D schedules through DistributedDomain.

Every cell a kernel must not read is NaN, and so is every cell it must not write: a stray read shows up as a NaN in a
result, a stray write as a number where NaN belongs.  The case lists and the launch decisions they are meant to reach are in
tests/jacobi_layout.py (checked without a GPU by tests/test_jacobi_layout_host.py)."""
import ctypes as C
import zlib

import numpy as np
import pytest

import jacobi_layout as jl
import stencil_b200 as sb
from gpu_util import DevArray
from oracle import c_oracle as co
from oracle import geometry as g
from oracle import np_oracle as no
from stencil_b200._lib import HaloPush, Pitched, StencilError, check, i3, lib

pytestmark = pytest.mark.gpu

DTYPES = {4: np.float32, 8: np.float64}
UINT = {4: np.uint32, 8: np.uint64}
FAR = (5000, 5000, 5000)  # a global region this far away puts no sphere near the cells (and no int overflow in its test)


def same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    return a.shape == b.shape and np.array_equal(a.view(UINT[a.dtype.itemsize]), b.view(UINT[b.dtype.itemsize]))


def mismatch(a: np.ndarray, b: np.ndarray) -> str:
    bad = np.argwhere(a.view(UINT[a.dtype.itemsize]) != b.view(UINT[b.dtype.itemsize]))
    return f"{len(bad)} cells differ, first (z,y,x) {[tuple(int(v) for v in p) for p in bad[:4]]}: got {a[tuple(bad[0])]} want {b[tuple(bad[0])]}" if len(bad) else "same"


def upload(dev: DevArray, host: np.ndarray) -> None:
    assert host.shape == dev.shape and host.dtype == dev.dtype
    host = np.ascontiguousarray(host)
    check(lib().sb_memcpy(C.c_void_p(dev.ptr), host.ctypes.data, host.nbytes, dev.device, None))
    check(lib().sb_stream_sync(dev.device, None))


# ------------------------------------------------------------------------------------------- sb_jacobi3d / _regions
def read_mask(shape, boxes):
    """Cells the 7-point stencil reads for the cells of `boxes` (allocation [lo, hi) boxes, x y z): the six neighbours only."""
    m = np.zeros(shape, dtype=bool)
    for lo, hi in boxes:
        for a in range(3):
            for s in (-1, 1):
                sl = [slice(lo[k], hi[k]) for k in range(3)]
                sl[a] = slice(lo[a] + s, hi[a] + s)
                m[sl[2], sl[1], sl[0]] = True
    return m


def run_sweep_case(c: jl.SweepCase, spheres: bool = False):
    dt = DTYPES[c.es]
    raw = c.raw
    shape = raw[::-1]
    gh = c.ghost
    origin = (1000, 2000, 3000)  # global coordinate of the first compute cell
    acc = tuple(o - gh for o in origin)
    n = (c.nx, c.ny, c.nz)
    clo, chi = (origin, tuple(origin[a] + n[a] for a in range(3))) if spheres else (FAR, tuple(f + 10 for f in FAR))
    rng = np.random.default_rng(c.nx * 131 + c.ghost * 7 + c.s_lead)
    vals = rng.random(shape).astype(dt)
    src = DevArray(np.zeros(shape, dt), lead=c.s_lead)
    dst = DevArray(np.zeros(shape, dt), lead=c.d_lead)

    def glob(lo):
        return tuple(acc[a] + lo[a] for a in range(3))

    # 1. sb_jacobi3d over the compute region and over boxes whose first cell is 1..3 cells later along x
    launches = []
    for xlo, xhi in c.x_ranges():
        box = ((xlo, gh, gh), (xhi, gh + c.ny, gh + c.nz))
        launches.append(("one", [box]))
    # 2. sb_jacobi3d_regions: the interior and the exterior slabs of a ghost-width-`gh` subdomain, in one launch
    ro = g.Radius.face_edge_corner(gh, 0, 0)
    lo_g, hi_g = origin, tuple(origin[a] + n[a] for a in range(3))
    regs = [g.get_interior(lo_g, hi_g, ro)] + g.get_exterior(lo_g, hi_g, ro)
    regs = [(tuple(l[a] - acc[a] for a in range(3)), tuple(h[a] - acc[a] for a in range(3))) for l, h in regs]
    regs = [r for r in regs if all(r[1][a] > r[0][a] for a in range(3))]
    launches.append(("regions", regs))
    results = []
    for kind, boxes in launches:
        poisoned = np.where(read_mask(shape, boxes), vals, np.nan).astype(dt)
        upload(src, poisoned)
        upload(dst, np.full(shape, np.nan, dt))
        if kind == "one":
            (lo, hi), = boxes
            check(lib().sb_jacobi3d(dst.pitched(), src.pitched(), c.es, i3(acc), i3(glob(lo)), i3(glob(hi)), i3(clo), i3(chi), None))
        else:
            elo = (C.c_int64 * (3 * len(boxes)))(*[v for lo, _ in boxes for v in glob(lo)])
            ehi = (C.c_int64 * (3 * len(boxes)))(*[v for _, hi in boxes for v in glob(hi)])
            check(lib().sb_jacobi3d_regions(dst.pitched(), src.pitched(), c.es, i3(acc), len(boxes), elo, ehi, i3(clo), i3(chi), None))
        want = np.full(shape, np.nan, dt)
        for lo, hi in boxes:
            co.jacobi_region(want, poisoned, acc, glob(lo), glob(hi), clo, chi)
        got = dst.get()
        assert same_bits(got, want), f"{c} {kind} {boxes[0]}: {mismatch(got, want)}"
        written = np.zeros(shape, dtype=bool)
        for lo, hi in boxes:
            written[lo[2]:hi[2], lo[1]:hi[1], lo[0]:hi[0]] = True
        assert not np.isnan(want[written]).any() and np.isnan(want[~written]).all()  # every result a number, nothing else written
        results.append(got)
    src.free()
    dst.free()
    return results


def _sweep_params():
    out = []
    for es in (4, 8):
        for s_lead, d_lead in [(lead, lead) for lead in jl.LEADS[es]] + list(jl.MIXED_LEADS[es]):
            out.append(pytest.param(es, s_lead, d_lead, id=f"f{8 * es}-lead{s_lead}.{d_lead}"))
    return out


@pytest.mark.parametrize("es,s_lead,d_lead", _sweep_params())
def test_jacobi_sweep_bit_exact_over_the_whole_allocation(es, s_lead, d_lead):
    """Every x width of jacobi_layout.SWEEP_NX at ghost widths 1..3, odd and even row counts: the compute region, boxes
    starting 1..3 cells later along x, and interior + exterior slabs in one sb_jacobi3d_regions launch."""
    cases = [c for c in jl.sweep_cases() if (c.es, c.s_lead, c.d_lead) == (es, s_lead, d_lead)]
    assert cases
    for c in cases:
        run_sweep_case(c)


@pytest.mark.parametrize("es", [4, 8], ids=["float32", "float64"])
def test_jacobi_sweep_with_spheres_inside_the_region(es):
    """The global region is the compute region itself: the hot (1) and cold (0) spheres are cut into the result."""
    lead = 12 if es == 4 else 8
    c = jl.SweepCase(es, lead, lead, 130, 17, 16, 1)
    for got in run_sweep_case(c, spheres=True)[:1]:
        core = got[1:-1, 1:-1, 1:-1]
        assert (core == 1).sum() > 0 and (core == 0).sum() > 0


# ------------------------------------------------------------------------------------------- sb_jacobi3d_fused
OPP = (1, 0, 3, 2, 5, 4)


def face_slice(f: int):
    """The ghost cells of face f of an allocation with ghost width 1 (no edges or corners), as a [z, y, x] index."""
    a, s = f // 2, f % 2
    sl = [slice(1, -1)] * 3  # x, y, z
    sl[a] = -1 if s else 0
    return (sl[2], sl[1], sl[0])


def face_cells(f: int):
    """The compute cells of face f (what a push of face f stores), [z, y, x] index."""
    a, s = f // 2, f % 2
    sl = [slice(1, -1)] * 3
    sl[a] = -2 if s else 1
    return (sl[2], sl[1], sl[0])


def window(G: np.ndarray, origin, size):
    """The periodic global field as subdomain `origin`/`size` sees it through an allocation with ghost width 1."""
    idx = [(origin[a] - 1 + np.arange(size[a] + 2)) % G.shape[2 - a] for a in range(3)]
    return G[np.ix_(idx[2], idx[1], idx[0])]


def jacobi_periodic(G: np.ndarray, clo, chi) -> np.ndarray:
    Gp = np.ascontiguousarray(np.pad(G, 1, mode="wrap"))
    out = np.zeros_like(Gp)
    nz, ny, nx = G.shape
    co.jacobi_region(out, Gp, (-1, -1, -1), (0, 0, 0), (nx, ny, nz), clo, chi)
    return np.ascontiguousarray(out[1:-1, 1:-1, 1:-1])


def run_fused_case(c: jl.FusedCase, iters: int = 3):
    dt = DTYPES[c.es]
    es = c.es
    gsize = c.global_size
    rng = np.random.default_rng(zlib.crc32(c.id().encode()))
    G = rng.random(gsize[::-1]).astype(dt)
    clo, chi = (0, 0, 0), gsize  # spheres of the global grid (radius nx / 10) cut through the subdomains
    origins = c.origins()
    nd = len(c.sizes)
    nbr_index = lambda i, f: i if c.nbrs(i)[f] == "self" else (1 - i if c.nbrs(i)[f] == "other" else None)
    raws = [(s[0] + 2, s[1] + 2, s[2] + 2) for s in c.sizes]
    # buffers: [subdomain][0 = curr, 1 = next]; host mirrors of what each must hold
    mirror = [[np.full(r[::-1], np.nan, dt) for _ in range(2)] for r in raws]
    bufs = [[DevArray(mirror[i][b], lead=c.leads[i][b]) for b in range(2)] for i in range(nd)]
    dense = c.config == "dense_x"
    # dense x arrays [subdomain][side][parity], (rows, planes) of the receiving subdomain
    recv, recv_mirror = {}, {}
    plans0 = c.plans(0)
    for i in range(nd):
        W = window(G, origins[i], c.sizes[i])
        mirror[i][0][1:-1, 1:-1, 1:-1] = W[1:-1, 1:-1, 1:-1]
        for f in range(6):  # what the first iteration reads: ghosts of every face not wrapped in place nor received densely
            if not plans0[i].wrap[f // 2] and not (f < 2 and plans0[i].dense[f]):
                mirror[i][0][face_slice(f)] = W[face_slice(f)]
        upload(bufs[i][0], mirror[i][0])
        if dense:
            for s in (0, 1):
                for par in (0, 1):
                    m = np.full((raws[i][1], raws[i][2]), np.nan, dt)
                    if par == 0:  # the neighbour's face cells of the initial field, [y][z]
                        m[1:-1, 1:-1] = W[face_slice(s)].T
                    recv_mirror[(i, s, par)] = m
                    recv[(i, s, par)] = DevArray(m)
    try:
        for it in range(iters):
            sb_, db_ = it % 2, 1 - it % 2
            plans = c.plans(sb_)
            Gn = jacobi_periodic(G, clo, chi)
            if c.config == "null":  # the host supplies every ghost face of src
                for i in range(nd):
                    W = window(G, origins[i], c.sizes[i])
                    for f in range(6):
                        mirror[i][sb_][face_slice(f)] = W[face_slice(f)]
                    upload(bufs[i][sb_], mirror[i][sb_])
            for i in range(nd):
                pl = plans[i]
                push = HaloPush()
                for f in range(6):
                    j = nbr_index(i, f)
                    if j is None:
                        push.nbr[f] = Pitched(None, 0, 0)
                    elif f < 2 and dense:
                        t = recv[(j, 1 - f, (it + 1) % 2)]
                        push.nbr[f] = Pitched(t.ptr, es, raws[i][1])
                        push.nbr_zsize[f] = raws[i][2]
                        push.x_dense[f] = 1
                        push.x_recv[f] = recv[(i, f, it % 2)].ptr
                    else:
                        push.nbr[f] = bufs[j][db_].pitched()
                        push.nbr_zsize[f] = raws[j][2]
                lo = origins[i]
                hi = tuple(lo[a] + c.sizes[i][a] for a in range(3))
                acc = tuple(v - 1 for v in lo)
                check(lib().sb_jacobi3d_fused(bufs[i][db_].pitched(), bufs[i][sb_].pitched(), es, i3(acc), i3(lo), i3(hi), i3(clo), i3(chi), C.byref(push), None))
            # expected contents of every dst buffer: compute cells; ghost faces a neighbour pushed into; nothing else changes
            for i in range(nd):
                Wn = window(Gn, origins[i], c.sizes[i])
                exp = mirror[i][db_]
                exp[1:-1, 1:-1, 1:-1] = Wn[1:-1, 1:-1, 1:-1]
                for f in range(6):
                    j = nbr_index(i, f)  # the subdomain whose ghost face OPP[f] ... is written by i's push f
                    if j is not None and plans[i].push[f]:
                        mirror[j][db_][face_slice(OPP[f])] = window(Gn, origins[j], c.sizes[j])[face_slice(OPP[f])]
                    if j is not None and f < 2 and plans[i].dense[f]:
                        m = recv_mirror[(j, 1 - f, (it + 1) % 2)]
                        m[1:-1, 1:-1] = Wn[face_cells(f)].T
            for i in range(nd):
                got = bufs[i][db_].get()
                assert same_bits(got, mirror[i][db_]), f"{c.id()} iteration {it} subdomain {i} {plans[i]}: {mismatch(got, mirror[i][db_])}"
                if dense:
                    for s in (0, 1):
                        key = (i, s, (it + 1) % 2)
                        gr = recv[key].get()
                        assert same_bits(gr, recv_mirror[key]), f"{c.id()} iteration {it} dense array {key}: {mismatch(gr, recv_mirror[key])}"
            # wrapped faces keep NaN ghosts in both buffers: the kernel never read them
            for i in range(nd):
                for f in range(6):
                    if plans[i].wrap[f // 2]:
                        assert np.isnan(mirror[i][db_][face_slice(f)]).all() and np.isnan(mirror[i][sb_][face_slice(f)]).all()
            G = Gn
    finally:
        for row in bufs:
            for b in row:
                b.free()
        for d in recv.values():
            d.free()


FUSED = jl.fused_cases()


@pytest.mark.parametrize("case", FUSED, ids=[c.id() for c in FUSED])
def test_fused_through_the_c_abi_bit_exact_with_exact_pushes(case):
    """Three iterations with src / dst swapped between them: after each, every compute cell against the oracle on the
    periodic global field, every ghost face pushed or untouched as the launch decision says, every other cell NaN."""
    run_fused_case(case)


@pytest.mark.parametrize("name", sorted(jl.FUSED_ERRORS))
def test_fused_rejects_what_it_cannot_run(name):
    es, lead, size, dense = jl.FUSED_ERROR_CASES[name]
    dt = DTYPES[es]
    raw = (size[0] + 2, size[1] + 2, size[2] + 2)
    a = DevArray(np.zeros(raw[::-1], dt), lead=lead)
    b = DevArray(np.zeros(raw[::-1], dt), lead=lead)
    recv = DevArray(np.zeros((raw[1], raw[2]), dt)) if any(dense) else None
    push = HaloPush()
    for f in range(6):
        push.nbr[f] = Pitched(None, 0, 0)
    for s in (0, 1):
        if dense[s]:
            push.x_recv[s] = recv.ptr
    lo, hi = (1, 1, 1), tuple(1 + v for v in size)
    rc = lib().sb_jacobi3d_fused(b.pitched(), a.pitched(), es, i3((0, 0, 0)), i3(lo), i3(hi), i3((0, 0, 0)), i3(size), C.byref(push), None)
    msg = lib().sb_last_error().decode()
    assert rc == -1 and jl.FUSED_ERRORS[name] in msg, (rc, msg)  # SB_ERR_INVALID
    with pytest.raises(StencilError):
        check(rc)


# ------------------------------------------------------------------------------------------- through DistributedDomain
@pytest.mark.parametrize("align", ["1", "0"])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2])
@pytest.mark.parametrize("size", [(30, 9, 10), (130, 17, 33), (66, 12, 9), (64, 10, 9)], ids=str)
def test_jacobi3d_schedules_match_the_oracle(monkeypatch, align, dtype, ndom, size):
    """Jacobi3D.step, step_async and step_fused, 6 iterations from a random field, against the oracle's interior -> exchange
    -> exterior loop, with allocations placed for a 16-byte aligned first compute cell (SB_ALLOC_ALIGN=1) and at the start
    of their blocks (0)."""
    from stencil_b200.jacobi import Jacobi3D, jacobi_radius

    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    ro = g.Radius.face_edge_corner(1, 0, 0)
    creg = ((0, 0, 0), size)
    od = no.Domains(size, ro, [dtype], n_subdomains=ndom)
    rng = np.random.default_rng(sum(size) * 10 + ndom)
    G = rng.random(size[::-1]).astype(dtype)
    start = {}
    for i in od.indices:
        lo, sz = od.origins[i], od.sizes[i]
        od.arrays[i][0][...] = 0
        no.box(od.arrays[i][0], (1, 1, 1), sz)[...] = G[lo[2]:lo[2] + sz[2], lo[1]:lo[1] + sz[1], lo[0]:lo[0] + sz[0]]
        start[i] = od.arrays[i][0].copy()
    nxt = {i: np.zeros_like(od.arrays[i][0]) for i in od.indices}
    for _ in range(6):
        boxes = {}
        for i in od.indices:
            lo = od.origins[i]
            hi = tuple(lo[a] + od.sizes[i][a] for a in range(3))
            boxes[i] = (g.accessor_origin(lo, ro), lo, hi)
            co.jacobi_region(nxt[i], od.arrays[i][0], boxes[i][0], *g.get_interior(lo, hi, ro), *creg)
        od.exchange()
        for i in od.indices:
            acc, lo, hi = boxes[i]
            for elo, ehi in g.get_exterior(lo, hi, ro):
                co.jacobi_region(nxt[i], od.arrays[i][0], acc, elo, ehi, *creg)
            od.arrays[i][0], nxt[i] = nxt[i], od.arrays[i][0]
    for mode in ("step", "step_async", "step_fused"):
        dd = sb.DistributedDomain(*size)
        dd.set_gpus([0] * ndom)
        dd.set_radius(jacobi_radius())
        h = dd.add_data(dtype, "d")
        dd.realize()
        try:
            for di, d in enumerate(dd.domains()):
                i = dd.domain_idx_[di]
                assert tuple(d.size()) == tuple(od.sizes[i])
                upload_domain(d, h, start[i])
            jac = Jacobi3D(dd, h)
            for _ in range(6):
                getattr(jac, mode)()
            jac.synchronize()
            for di, d in enumerate(dd.domains()):
                i = dd.domain_idx_[di]
                sz = od.sizes[i]
                got, want = no.box(d.quantity_to_host(0), (1, 1, 1), sz), no.box(od.arrays[i][0], (1, 1, 1), sz)
                assert np.array_equal(got, want), f"{mode} subdomain {i}: {mismatch(np.ascontiguousarray(got), np.ascontiguousarray(want))}"
        finally:
            dd.close()


def upload_domain(d, h, host: np.ndarray) -> None:
    """Both buffers of a subdomain's quantity = host (the whole allocation, ghost cells included)."""
    for which in ("curr", "next"):
        p = d.pitched(h.id, which)
        assert p.pitch * p.ysize * host.shape[0] == host.nbytes
        check(lib().sb_memcpy(C.c_void_p(p.ptr), host.ctypes.data, host.nbytes, d.gpu(), None))
    check(lib().sb_stream_sync(d.gpu(), None))
