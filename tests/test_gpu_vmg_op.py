"""GPU parity of the three variable-coefficient multigrid plans through the C ABI, bit for bit against tests/vmg_oracle.py:
the diagonal relaxation (sb_stencil_dplan_create), the face-coefficient restriction (sb_transfer_fplan_create) and the
fused residual-restriction with coefficient fields (sb_transfer_voplan_create).  float and double, boxes of many shapes
(odd origins and extents, negative origins, thin boxes for the cell kernels), allocation leads of 0 .. 12 bytes on each
buffer, NaN in every cell a rule does not read and in dst outside the boxes, every colour in place and out of place,
interior + exterior slabs against one box, the fused plan against sb_stencil_vplan_create followed by the restriction on
the GPU, and one 512^3 FP64 launch of each."""
import ctypes as C

import numpy as np
import pytest

import colour_oracle as co
import transfer_oracle as to
import vmg_oracle as vm
import vstencil_oracle as vo
from gpu_util import DevArray
from stencil_b200._lib import I3, Pitched, StencilVTerm, check, lib

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
DT = {np.dtype(np.float32): 1, np.dtype(np.float64): 2}
NONE = Pitched(None, 0, 0)


def same(a, b):
    return np.array_equal(a.view(UINT[a.dtype]), b.view(UINT[b.dtype]))


def c_vterms(terms):
    arr = (StencilVTerm * len(terms))()
    for i, t in enumerate(terms):
        s, o, w, k, c = vo.split(t)
        arr[i] = StencilVTerm(s, (C.c_int32 * 3)(*o), k, (C.c_int32 * 3)(*c), w)
    return arr


def boxes_arg(boxes):
    lo = (C.c_int64 * (3 * max(1, len(boxes))))(*[v for b in boxes for v in b[0]])
    hi = (C.c_int64 * (3 * max(1, len(boxes))))(*[v for b in boxes for v in b[1]])
    return lo, hi


def mask(shape, origin, lo, hi):
    m = np.ones(shape, bool)
    for a in range(3):
        c = np.arange(shape[2 - a]) + origin[a]
        sh = [1, 1, 1]
        sh[2 - a] = shape[2 - a]
        m &= ((c >= lo[a]) & (c < hi[a])).reshape(sh)
    return m


def kappa_op(h=1.0 / 32, sigma="field"):
    """-div(kappa grad u) + sigma u: sigma a fourth (cell) field, a constant, or none."""
    return vm.helmholtz_div_grad(h, sigma_field=sigma == "field", sigma=0.75 if sigma == "const" else 0.0)


def aniso_op():
    """A 19-term coefficient op with two offset-0 terms of different fields and a plain 27-point corner."""
    A = kappa_op(1.0 / 16, "field")
    return A + [(0, (1, 1, 1), -0.01), (0, (-1, -1, -1), -0.02, 0, (0, 0, 0)), (0, (0, 0, 0), 0.5, 1, (0, 1, 0))]


OPS = {"kappa+sigma": kappa_op, "kappa": lambda: kappa_op(sigma=None), "kappa+const": lambda: kappa_op(sigma="const"), "aniso": aniso_op}
NCOEF = 4


# ------------------------------------------------------------------------------------------- diagonal relaxation
def run_diag(dtype, terms, boxes, m, c, omega=1.0, inplace=False, leads=(0, 0, 0, 0), seed=0):
    """One dplan over boxes (global coordinates; their union one box) of an allocation of ghost width 2 + pad."""
    dtype = np.dtype(dtype)
    lo = [min(b[0][a] for b in boxes) for a in range(3)]
    hi = [max(b[1][a] for b in boxes) for a in range(3)]
    rng = np.random.default_rng(seed + sum(lo) + 3 * sum(hi) + m + 7 * c)
    pad = (2, 3, 2)
    origin = tuple(lo[a] - pad[a] for a in range(3))
    shape = tuple(hi[a] - lo[a] + 2 * pad[a] for a in (2, 1, 0))
    offs = [t[1] for t in terms]
    rlo = [lo[a] + min(o[a] for o in offs) for a in range(3)]
    rhi = [hi[a] + max(o[a] for o in offs) for a in range(3)]
    u = rng.uniform(-1, 1, shape).astype(dtype)
    u[~mask(shape, origin, rlo, rhi)] = np.nan
    f = rng.uniform(-1, 1, shape).astype(dtype)
    f[~mask(shape, origin, lo, hi)] = np.nan
    ks = []
    for k in range(NCOEF):
        co_ = [vo.split(t)[4] for t in terms if vo.split(t)[3] == k] or [(0, 0, 0)]
        kl = [lo[a] + min(o[a] for o in co_) for a in range(3)]
        kh = [hi[a] + max(o[a] for o in co_) for a in range(3)]
        arr = rng.uniform(0.5, 1.5, shape).astype(dtype)
        arr[~mask(shape, origin, kl, kh)] = np.nan
        ks.append(arr)
    dst0 = u.copy() if inplace else np.full(shape, np.nan, dtype)
    U, Fd = DevArray(u, lead=leads[0]), DevArray(f, lead=leads[1])
    K = [DevArray(a, lead=leads[2]) for a in ks]
    D = U if inplace else DevArray(dst0, lead=leads[3])
    karr = (Pitched * NCOEF)(*[k.pitched() for k in K])
    blo, bhi = boxes_arg(boxes)
    h = C.c_void_p()
    check(lib().sb_stencil_dplan_create(C.byref(h), 0, DT[dtype], c_vterms(terms), len(terms), D.pitched(), U.pitched(), Fd.pitched(), karr,
                                        NCOEF, float(omega), m, c, I3(*origin), shape[0], len(boxes), blo, bhi))
    try:
        check(lib().sb_stencil_plan_launch(h, None))
        check(lib().sb_device_sync(0))
        got = D.get()
    finally:
        lib().sb_stencil_plan_destroy(h)
    want = dst0.copy()
    for b in boxes:
        l = [b[0][a] - origin[a] for a in range(3)]
        e = [b[1][a] - b[0][a] for a in range(3)]
        if min(e) > 0:
            vm.diag_box(terms, omega, u, f, ks, want, l, e, origin, m, c)
    assert same(got, want)
    if not inplace:
        assert same(U.get(), u)
    assert same(Fd.get(), f)


BOXES = [((0, 0, 0), (1, 1, 1)), ((0, 0, 0), (8, 8, 8)), ((0, 0, 0), (7, 5, 3)), ((3, -2, 1), (21, 12, 17)), ((-5, 2, 0), (70, 11, 19)),
         ((1, 1, 1), (130, 20, 9)), ((2, 3, -1), (3, 40, 9))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", BOXES)
@pytest.mark.parametrize("op", sorted(OPS))
def test_diag_boxes_jacobi(dtype, box, op):
    run_diag(dtype, OPS[op](), [box], 1, 0, omega=0.8)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("m", [2, 8])
@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("box", [((0, 0, 0), (9, 9, 9)), ((-3, 1, 2), (70, 13, 12)), ((1, 0, 0), (4, 30, 11))])
def test_diag_colours(dtype, m, inplace, box):
    terms = kappa_op(sigma="field") if m == 2 else aniso_op()
    for c in range(m):
        run_diag(dtype, terms, [box], m, c, omega=1.0, inplace=inplace)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", range(4))
def test_diag_leads(dtype, which):
    es = np.dtype(dtype).itemsize
    for lead in range(0, 16, es):
        leads = [0, 0, 0, 0]
        leads[which] = lead
        run_diag(dtype, kappa_op(), [((1, 0, 2), (70, 9, 11))], 2, 1, inplace=False, leads=tuple(leads))


def slabs(lo, hi, w=1):
    """[lo, hi) as its interior cut by w and the six exterior slabs."""
    il, ih = [v + w for v in lo], [v - w for v in hi]
    out = [(tuple(il), tuple(ih))]
    for a in range(3):
        for side in (0, 1):
            l, h = list(lo), list(hi)
            for b in range(a):
                l[b], h[b] = il[b], ih[b]
            if side == 0:
                h[a] = lo[a] + w
            else:
                l[a] = hi[a] - w
            out.append((tuple(l), tuple(h)))
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_diag_interior_and_exterior_equal_one_box(dtype):
    lo, hi = (-3, 2, 1), (69, 25, 22)
    for m, c in ((1, 0), (2, 1), (8, 5)):
        run_diag(dtype, aniso_op() if m == 8 else kappa_op(), slabs(lo, hi), m, c, seed=1)
        run_diag(dtype, aniso_op() if m == 8 else kappa_op(), [(lo, hi)], m, c, seed=1)


def test_diag_512_fp64():
    """One in-place red pass of -div(kappa grad u) on 512^3 (ghost width 1), the oracle in slabs of 32 planes."""
    n = 512
    rng = np.random.default_rng(5)
    u = rng.uniform(-1, 1, (n + 2,) * 3)
    f = rng.uniform(-1, 1, (n + 2,) * 3)
    ks = [rng.uniform(0.5, 1.5, (n + 2,) * 3) for _ in range(3)]
    terms = kappa_op(1.0 / n, None)
    U, Fd = DevArray(u), DevArray(f)
    K = [DevArray(a) for a in ks]
    karr = (Pitched * 3)(*[k.pitched() for k in K])
    blo, bhi = boxes_arg([((0, 0, 0), (n, n, n))])
    h = C.c_void_p()
    check(lib().sb_stencil_dplan_create(C.byref(h), 0, 2, c_vterms(terms), len(terms), U.pitched(), U.pitched(), Fd.pitched(), karr, 3, 1.0, 2,
                                        0, I3(-1, -1, -1), n + 2, 1, blo, bhi))
    try:
        check(lib().sb_stencil_plan_launch(h, None))
        got = U.get()
    finally:
        lib().sb_stencil_plan_destroy(h)
    del U, K
    for z0 in range(0, n, 32):
        sl = slice(z0, z0 + 34)  # padded planes z0 .. z0 + 33: the slab's planes and their neighbours
        want = u[sl].copy()
        vm.diag_box(terms, 1.0, u[sl], f[sl], [k[sl] for k in ks], want, (1, 1, 1), (n, n, 32), (-1, -1, z0 - 1), 2, 0)
        assert same(got[z0 + 1 : z0 + 33], want[1:33]), z0


# ------------------------------------------------------------------------------------------- face restriction
def run_face(dtype, axis, lo, hi, lead_d=0, lead_s=0):
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(sum(lo) + 5 * sum(hi) + axis)
    pad = (3, 1, 2)
    so = tuple(2 * lo[a] - pad[a] for a in range(3))
    sshape = tuple(2 * (hi[a] - lo[a]) + 2 * pad[a] for a in (2, 1, 0))
    src = rng.uniform(0.1, 2, sshape).astype(dtype)
    # only the fine plane 2 I_axis of each coarse cell is read
    keep = mask(sshape, so, [2 * v for v in lo], [2 * v for v in hi])
    c = np.arange(sshape[2 - axis]) + so[axis]
    sh = [1, 1, 1]
    sh[2 - axis] = sshape[2 - axis]
    keep &= (c % 2 == 0).reshape(sh)
    src[~keep] = np.nan
    do = tuple(lo[a] - 1 for a in range(3))
    dshape = tuple(hi[a] - lo[a] + 3 for a in (2, 1, 0))
    dst0 = np.full(dshape, np.nan, dtype)
    S, D = DevArray(src, lead=lead_s), DevArray(dst0, lead=lead_d)
    h = C.c_void_p()
    check(lib().sb_transfer_fplan_create(C.byref(h), 0, DT[dtype], axis, D.pitched(), I3(*do), dshape[0], S.pitched(), I3(*so), sshape[0],
                                         I3(*lo), I3(*hi)))
    try:
        cells = int(np.prod([hi[a] - lo[a] for a in range(3)]))
        assert lib().sb_transfer_plan_bytes(h) == 5 * cells * dtype.itemsize
        check(lib().sb_transfer_plan_launch(h, None))
        got = D.get()
    finally:
        lib().sb_transfer_plan_destroy(h)
    want = dst0.copy()
    vm.face_restrict_box(want, do, src, so, axis, lo, hi)
    assert same(got, want)


FBOXES = [((0, 0, 0), (1, 1, 1)), ((0, 0, 0), (7, 5, 3)), ((3, -2, 1), (11, 6, 9)), ((-5, 2, 0), (60, 11, 17)), ((1, 1, 1), (66, 35, 21))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("box", FBOXES)
def test_face_boxes(dtype, axis, box):
    run_face(dtype, axis, *box)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", ["d", "s"])
def test_face_leads(dtype, which):
    es = np.dtype(dtype).itemsize
    for lead in range(0, 16, es):
        for axis in range(3):
            run_face(dtype, axis, (1, 0, 2), (40, 9, 7), **{f"lead_{which}": lead})


def test_face_512_fp64():
    n, m = 512, 256
    rng = np.random.default_rng(6)
    src = rng.uniform(0.1, 2, (n,) * 3)
    S = DevArray(src)
    for axis in range(3):
        D = DevArray(np.full((m,) * 3, np.nan))
        h = C.c_void_p()
        check(lib().sb_transfer_fplan_create(C.byref(h), 0, 2, axis, D.pitched(), I3(0, 0, 0), m, S.pitched(), I3(0, 0, 0), n, I3(0, 0, 0),
                                             I3(m, m, m)))
        try:
            check(lib().sb_transfer_plan_launch(h, None))
            got = D.get()
        finally:
            lib().sb_transfer_plan_destroy(h)
        want = np.empty((m,) * 3)
        vm.face_restrict_box(want, (0, 0, 0), src, (0, 0, 0), axis, (0, 0, 0), (m, m, m))
        assert same(got, want), axis


# ------------------------------------------------------------------------------------------- fused, with coefficients
def vo_plan(dtype, terms, D, do, S, so, A, K, boxes):
    blo, bhi = boxes_arg(boxes)
    karr = (Pitched * max(1, len(K)))(*[k.pitched() for k in K])
    h = C.c_void_p()
    check(lib().sb_transfer_voplan_create(C.byref(h), 0, DT[np.dtype(dtype)], c_vterms(terms), len(terms), D.pitched(), I3(*do), D.shape[0],
                                          S.pitched(), I3(*so), S.shape[0], A.pitched() if A is not None else NONE, karr, len(K), len(boxes),
                                          blo, bhi))
    return h


def run_vop(dtype, terms, boxes, lead_d=0, lead_s=0, lead_a=0, lead_k=0):
    dtype = np.dtype(dtype)
    lo = [min(b[0][a] for b in boxes) for a in range(3)]
    hi = [max(b[1][a] for b in boxes) for a in range(3)]
    rng = np.random.default_rng(sum(lo) + 7 * sum(hi) + len(terms))
    pad = (2, 1, 3)
    so = tuple(2 * lo[a] - 1 - pad[a] for a in range(3))
    sshape = tuple(2 * (hi[a] - lo[a]) + 2 + 2 * pad[a] for a in (2, 1, 0))
    rlo, rhi = [2 * v - 1 for v in lo], [2 * v + 1 for v in hi]
    src = rng.uniform(-1, 1, sshape).astype(dtype)
    offs = [t[1] for t in terms if t[0] == 0]
    src[~mask(sshape, so, [2 * lo[a] + min(o[a] for o in offs) for a in range(3)], [2 * hi[a] + max(o[a] for o in offs) for a in range(3)])] = np.nan
    aux = rng.uniform(-1, 1, sshape).astype(dtype)
    aux[~mask(sshape, so, [2 * v for v in lo], [2 * v for v in hi])] = np.nan
    ks = []
    for k in range(NCOEF):
        co_ = [vo.split(t)[4] for t in terms if vo.split(t)[3] == k] or [(0, 0, 0)]
        arr = rng.uniform(0.5, 1.5, sshape).astype(dtype)
        arr[~mask(sshape, so, [2 * lo[a] + min(o[a] for o in co_) for a in range(3)], [2 * hi[a] + max(o[a] for o in co_) for a in range(3)])] = np.nan
        ks.append(arr)
    assert all(rlo[a] >= so[a] for a in range(3))
    do = tuple(lo[a] - 1 for a in range(3))
    dshape = tuple(hi[a] - lo[a] + 3 for a in (2, 1, 0))
    dst0 = np.full(dshape, np.nan, dtype)
    S, D, A = DevArray(src, lead=lead_s), DevArray(dst0, lead=lead_d), DevArray(aux, lead=lead_a)
    K = [DevArray(a, lead=lead_k) for a in ks]
    h = vo_plan(dtype, terms, D, do, S, so, A, K, boxes)
    try:
        cells = int(np.prod([hi[a] - lo[a] for a in range(3)]))
        nf = len({vo.split(t)[3] for t in terms} - {-1})
        assert lib().sb_transfer_plan_bytes(h) == cells * dtype.itemsize * (8 * (2 + nf) + 1)
        check(lib().sb_transfer_plan_launch(h, None))
        got = D.get()
    finally:
        lib().sb_transfer_plan_destroy(h)
    want = dst0.copy()
    vm.restrict_vop_box(want, do, terms, src, aux, ks, so, lo, hi)
    assert same(got, want)


VOPS = {k: (lambda f=f: vm.vresidual_terms(f())) for k, f in OPS.items()}
VBOXES = [((0, 0, 0), (1, 1, 1)), ((0, 0, 0), (4, 4, 4)), ((0, 0, 0), (7, 5, 3)), ((3, -2, 1), (11, 6, 9)), ((-5, 2, 0), (60, 11, 17)),
          ((2, 3, -1), (3, 40, 9))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", VBOXES)
@pytest.mark.parametrize("op", sorted(VOPS))
def test_vop_boxes(dtype, box, op):
    run_vop(dtype, VOPS[op](), [box])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", ["d", "s", "a", "k"])
def test_vop_leads(dtype, which):
    es = np.dtype(dtype).itemsize
    for lead in range(0, 16, es):
        run_vop(dtype, VOPS["kappa+sigma"](), [((1, 0, 2), (40, 9, 7))], **{f"lead_{which}": lead})


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_vop_interior_and_exterior_equal_one_box(dtype):
    lo, hi = (-3, 2, 1), (37, 15, 12)
    run_vop(dtype, VOPS["aniso"](), slabs(lo, hi))
    run_vop(dtype, VOPS["aniso"](), [(lo, hi)])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_vop_equals_vplan_then_restrict_on_gpu(dtype):
    """The fused plan's bits are sb_stencil_vplan_create into a scratch buffer followed by SB_TRANSFER_RESTRICT, both on
    the GPU."""
    dtype = np.dtype(dtype)
    n, m = 40, 20
    rng = np.random.default_rng(9)
    terms = VOPS["kappa+sigma"]()
    u, f = (rng.uniform(-1, 1, (n + 2,) * 3).astype(dtype) for _ in range(2))
    ks = [rng.uniform(0.5, 1.5, (n + 2,) * 3).astype(dtype) for _ in range(NCOEF)]
    U, Fd, K = DevArray(u), DevArray(f), [DevArray(a) for a in ks]
    Dv, R = DevArray(np.full((m,) * 3, np.nan, dtype)), DevArray(np.full((m,) * 3, np.nan, dtype))
    Scr = DevArray(np.full((n + 2,) * 3, np.nan, dtype))
    hs = []
    try:
        hs.append(vo_plan(dtype, terms, Dv, (0, 0, 0), U, (-1, -1, -1), Fd, K, [((0, 0, 0), (m, m, m))]))
        karr = (Pitched * NCOEF)(*[k.pitched() for k in K])
        blo, bhi = boxes_arg([((0, 0, 0), (n, n, n))])
        h = C.c_void_p()
        check(lib().sb_stencil_vplan_create(C.byref(h), 0, DT[dtype], c_vterms(terms), len(terms), Scr.pitched(), U.pitched(), Fd.pitched(), karr,
                                            NCOEF, I3(-1, -1, -1), n + 2, 1, blo, bhi))
        hs.append(h)
        h = C.c_void_p()
        check(lib().sb_transfer_plan_create(C.byref(h), 0, DT[dtype], 0, R.pitched(), I3(0, 0, 0), m, Scr.pitched(), I3(-1, -1, -1), n + 2, NONE,
                                            I3(0, 0, 0), I3(m, m, m)))
        hs.append(h)
        check(lib().sb_transfer_plan_launch(hs[0], None))
        check(lib().sb_stencil_plan_launch(hs[1], None))
        check(lib().sb_transfer_plan_launch(hs[2], None))
        assert same(Dv.get(), R.get())
    finally:
        lib().sb_transfer_plan_destroy(hs[0]) if hs else None
        if len(hs) > 1:
            lib().sb_stencil_plan_destroy(hs[1])
        if len(hs) > 2:
            lib().sb_transfer_plan_destroy(hs[2])


def test_vop_512_fp64():
    n, m = 512, 256
    rng = np.random.default_rng(7)
    u = rng.uniform(-1, 1, (n + 2,) * 3)
    f = rng.uniform(-1, 1, (n + 2,) * 3)
    ks = [rng.uniform(0.5, 1.5, (n + 2,) * 3) for _ in range(3)]
    terms = vm.vresidual_terms(kappa_op(1.0 / n, None))
    U, Fd, K = DevArray(u), DevArray(f), [DevArray(a) for a in ks]
    Cd = DevArray(np.full((m,) * 3, np.nan))
    h = vo_plan(np.float64, terms, Cd, (0, 0, 0), U, (-1, -1, -1), Fd, K, [((0, 0, 0), (m, m, m))])
    try:
        check(lib().sb_transfer_plan_launch(h, None))
        got = Cd.get()
    finally:
        lib().sb_transfer_plan_destroy(h)
    for z0 in range(0, m, 32):
        want = np.empty((32, m, m))
        sl = slice(2 * z0, 2 * z0 + 66)
        vm.restrict_vop_box(want, (0, 0, z0), terms, u[sl], f[sl], [k[sl] for k in ks], (-1, -1, 2 * z0 - 1), (0, 0, z0), (m, m, z0 + 32))
        assert same(got[z0 : z0 + 32], want), z0
