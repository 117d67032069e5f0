"""GPU parity of the transfer kernels through the C ABI (sb_transfer_plan_*): restriction and prolongation, float and
double, over boxes of many shapes (fine boxes with odd origin and odd extent included), at every allocation lead of
each buffer independently, with NaN in every src cell the rule does not read and in dst outside the box, prolongation
in place, into a separate dst and without aux, sb_transfer_plan_bytes, and 512^3 <-> 256^3 FP64 bit for bit."""
import ctypes as C

import numpy as np
import pytest

import transfer_oracle as to
from gpu_util import DevArray
from stencil_b200._lib import I3, Pitched, check, lib

pytestmark = pytest.mark.gpu

UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
DT = {np.dtype(np.float32): 1, np.dtype(np.float64): 2}


def same(a, b):
    return np.array_equal(a.view(UINT[a.dtype]), b.view(UINT[b.dtype]))


def plan(kind, dtype, dst, do, src, so, lo, hi, aux=None):
    h = C.c_void_p()
    check(lib().sb_transfer_plan_create(C.byref(h), 0, DT[np.dtype(dtype)], kind, dst.pitched(), I3(*do), dst.shape[0], src.pitched(), I3(*so),
                                        src.shape[0], aux.pitched() if aux is not None else Pitched(None, 0, 0), I3(*lo), I3(*hi)))
    return h


def run(h):
    check(lib().sb_transfer_plan_launch(h, None))
    check(lib().sb_device_sync(0))


def read_mask(shape, origin, lo, hi):
    """The cells of an array (element 0 at global origin) inside [lo, hi) per axis."""
    m = np.ones(shape, bool)
    for a in range(3):
        c = np.arange(shape[2 - a]) + origin[a]
        ok = (c >= lo[a]) & (c < hi[a])
        sh = [1, 1, 1]
        sh[2 - a] = shape[2 - a]
        m &= ok.reshape(sh)
    return m


def restrict_case(dtype, lo, hi, lead_d=0, lead_s=0, pad=(2, 1, 3)):
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(sum(lo) + 7 * sum(hi))
    # src: the fine cells [2 lo, 2 hi) plus a NaN margin; dst: the box plus a NaN margin
    so = tuple(2 * lo[a] - pad[a] for a in range(3))
    sshape = tuple(2 * (hi[a] - lo[a]) + 2 * pad[a] + 1 for a in (2, 1, 0))
    src = rng.uniform(-1, 1, sshape).astype(dtype)
    src[~read_mask(sshape, so, [2 * v for v in lo], [2 * v for v in hi])] = np.nan
    do = tuple(lo[a] - 1 for a in range(3))
    dshape = tuple(hi[a] - lo[a] + 3 for a in (2, 1, 0))
    dst0 = np.full(dshape, np.nan, dtype)
    S, D = DevArray(src, lead=lead_s), DevArray(dst0, lead=lead_d)
    h = plan(0, dtype, D, do, S, so, lo, hi)
    try:
        cells = int(np.prod([hi[a] - lo[a] for a in range(3)]))
        assert lib().sb_transfer_plan_bytes(h) == 9 * cells * dtype.itemsize
        run(h)
        want = dst0.copy()
        to.restrict_box(want, do, src, so, lo, hi)
        assert same(D.get(), want)
        assert same(S.get(), src)
    finally:
        lib().sb_transfer_plan_destroy(h)


def prolong_case(dtype, lo, hi, aux_mode="dst", lead_d=0, lead_s=0, lead_a=0):
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(3 * sum(lo) + sum(hi))
    rlo = [(lo[a] - 1) // 2 for a in range(3)]  # the coarse cells the rule reads
    rhi = [hi[a] // 2 + 1 for a in range(3)]
    clo = [lo[a] // 2 - 1 for a in range(3)]  # what the plan's check covers
    chi = [(hi[a] - 1) // 2 + 2 for a in range(3)]
    so = tuple(clo[a] - 1 for a in range(3))
    sshape = tuple(chi[a] - clo[a] + 2 for a in (2, 1, 0))
    src = rng.uniform(-1, 1, sshape).astype(dtype)
    src[~read_mask(sshape, so, rlo, rhi)] = np.nan
    do = tuple(lo[a] - 2 for a in range(3))
    dshape = tuple(hi[a] - lo[a] + 3 for a in (2, 1, 0))
    inbox = read_mask(dshape, do, lo, hi)
    base = rng.uniform(-1, 1, dshape).astype(dtype)
    base[~inbox] = np.nan
    other = rng.uniform(-1, 1, dshape).astype(dtype)
    other[~inbox] = np.nan
    dst0 = base if aux_mode == "dst" else np.full(dshape, np.nan, dtype)
    S, D = DevArray(src, lead=lead_s), DevArray(dst0, lead=lead_d)
    A = DevArray(other, lead=lead_a) if aux_mode == "other" else None
    aux_dev = D if aux_mode == "dst" else A
    h = plan(1, dtype, D, do, S, so, lo, hi, aux_dev)
    try:
        cells = int(np.prod([hi[a] - lo[a] for a in range(3)]))
        reads = int(np.prod([rhi[a] - rlo[a] for a in range(3)]))
        assert lib().sb_transfer_plan_bytes(h) == (reads + cells * (1 if aux_mode is None else 2)) * dtype.itemsize
        run(h)
        want = dst0.copy()
        aux_host = {"dst": want, "other": other, None: None}[aux_mode]
        to.prolong_box(want, do, src, so, lo, hi, aux=aux_host)
        assert same(D.get(), want)
        assert same(S.get(), src)
    finally:
        lib().sb_transfer_plan_destroy(h)


COARSE_BOXES = [((0, 0, 0), (1, 1, 1)), ((0, 0, 0), (7, 5, 3)), ((3, -2, 1), (11, 6, 9)), ((0, 0, 0), (32, 8, 8)),
                ((-5, 2, 0), (60, 11, 17)), ((1, 1, 1), (66, 35, 21))]
FINE_BOXES = [((0, 0, 0), (2, 2, 2)), ((1, 1, 1), (2, 2, 2)), ((0, 0, 0), (8, 8, 8)), ((1, 3, 5), (64, 12, 22)), ((-3, 0, -1), (62, 17, 20)),
              ((0, 0, 0), (64, 16, 16)), ((5, 4, 3), (136, 37, 30)), ((2, 1, 0), (3, 70, 9))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", COARSE_BOXES)
def test_restrict_boxes(dtype, box):
    restrict_case(dtype, *box)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("box", FINE_BOXES)
@pytest.mark.parametrize("aux_mode", ["dst", "other", None])
def test_prolong_boxes(dtype, box, aux_mode):
    prolong_case(dtype, *box, aux_mode=aux_mode)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("which", ["dst", "src", "aux"])
def test_leads(dtype, which):
    """Leads 0 .. 12 bytes (every multiple of the element size) on each buffer, the others at 0."""
    es = np.dtype(dtype).itemsize
    for lead in range(0, 16, es):
        kw = {f"lead_{which[0] if which != 'aux' else 'a'}": lead}
        if which != "aux":
            restrict_case(dtype, (1, 0, 2), (40, 9, 7), **{k: v for k, v in kw.items() if k != "lead_a"})
        prolong_case(dtype, (1, 2, 0), (71, 13, 11), aux_mode="other", **kw)
        prolong_case(dtype, (0, 1, 3), (70, 14, 12), aux_mode="dst", **{k: v for k, v in kw.items() if k != "lead_a"})


def test_empty_box():
    src = np.zeros((4, 4, 4))
    dst = np.full((4, 4, 4), np.nan)
    S, D = DevArray(src), DevArray(dst)
    h = plan(0, np.float64, D, (0, 0, 0), S, (0, 0, 0), (1, 1, 1), (1, 2, 2))
    try:
        assert lib().sb_transfer_plan_bytes(h) == 0
        run(h)
        assert same(D.get(), dst)
    finally:
        lib().sb_transfer_plan_destroy(h)


def test_512_restrict_and_256_prolong_fp64():
    """One 512^3 -> 256^3 restriction and one in-place 256^3 -> 512^3 prolongation (ghost width 1 on the coarse side),
    each a single launch, bit for bit against the oracle (the prolongation's oracle in slabs of 64 planes)."""
    n = 512
    rng = np.random.default_rng(512)
    fine = rng.uniform(-1, 1, (n, n, n))
    coarse = np.full((n // 2,) * 3, np.nan)
    F, Cd = DevArray(fine), DevArray(coarse)
    h = plan(0, np.float64, Cd, (0, 0, 0), F, (0, 0, 0), (0, 0, 0), (n // 2,) * 3)
    try:
        run(h)
        to.restrict_box(coarse, (0, 0, 0), fine, (0, 0, 0), (0, 0, 0), (n // 2,) * 3)
        assert same(Cd.get(), coarse)
    finally:
        lib().sb_transfer_plan_destroy(h)
        Cd.free()
    m = n // 2 + 2
    E = rng.uniform(-1, 1, (m, m, m))
    Ed = DevArray(E)
    h = plan(1, np.float64, F, (0, 0, 0), Ed, (-1, -1, -1), (0, 0, 0), (n,) * 3, aux=F)
    try:
        run(h)
        got = F.get()
        for z0 in range(0, n, 64):
            want = fine[z0 : z0 + 64].copy()
            to.prolong_box(want, (0, 0, z0), E, (-1, -1, -1), (0, 0, z0), (n, n, z0 + 64), aux=want)
            assert same(got[z0 : z0 + 64], want), z0
    finally:
        lib().sb_transfer_plan_destroy(h)
