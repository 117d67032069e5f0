"""GPU parity of the box-copy engine (pack / unpack / translate / plans) against the oracle and the
reference's golden vectors.  Bit-exact: this is pure data movement."""
import ctypes as C

import numpy as np
import pytest

import stencil_b200 as sb
from oracle import geometry as g
from oracle import np_oracle as no
from stencil_b200._lib import Pitched, check, i3, lib
from gpu_util import DevArray

pytestmark = pytest.mark.gpu


def dev_pack(src: DevArray, pos, ext):
    out = DevArray(np.zeros(ext[0] * ext[1] * ext[2], dtype=src.dtype).reshape(1, 1, -1))
    check(lib().sb_pack(C.c_void_p(out.ptr), src.pitched(), i3(pos), i3(ext), src.dtype.itemsize, None))
    return out


@pytest.mark.parametrize("dtype", [np.int32, np.float64])
def test_pack_golden_values(dtype):
    """test/test_cuda_pack.cu:82-84, 107-110, 123-126, 91-92 -- same launches through our kernels."""
    a = np.arange(60, dtype=dtype).reshape(5, 4, 3)
    src = DevArray(a)
    z4 = dev_pack(src, (0, 0, 4), (3, 4, 1)).get().reshape(-1)
    assert (z4[0], z4[1], z4[11]) == (48, 49, 59)
    x0 = dev_pack(src, (0, 0, 0), (1, 4, 5)).get().reshape(-1)
    assert (x0[0], x0[1], x0[11], x0[19]) == (0, 3, 33, 57)
    y1 = dev_pack(src, (0, 1, 0), (3, 1, 5)).get().reshape(-1)
    assert (y1[0], y1[1], y1[11], y1[14]) == (3, 4, 41, 53)
    dst2 = DevArray(np.zeros_like(a))
    buf = dev_pack(src, (0, 0, 4), (3, 4, 1))
    check(lib().sb_unpack(dst2.pitched(), C.c_void_p(buf.ptr), i3((0, 0, 4)), i3((3, 4, 1)), a.dtype.itemsize, None))
    got = dst2.get().reshape(-1)
    assert got[48] == 48 and got[59] == 59 and np.count_nonzero(got[:48]) == 0


def test_unpack_real_case_30x40x50_r4():
    """test/test_cuda_pack.cu:133-162: 30x40x50, radius 4, +x face unpack (there a smoke test; here checked)."""
    raw = (58, 48, 38)
    rng = np.random.default_rng(0)
    buf = rng.integers(0, 2**31, size=4 * 40 * 50).astype(np.int32)
    dst = DevArray(np.zeros(raw, dtype=np.int32))
    dbuf = DevArray(buf.reshape(1, 1, -1))
    check(lib().sb_unpack(dst.pitched(), C.c_void_p(dbuf.ptr), i3((34, 4, 4)), i3((4, 40, 50)), 4, None))
    want = np.zeros(raw, dtype=np.int32)
    no.unpack(want, buf, (34, 4, 4), (4, 40, 50))
    assert np.array_equal(dst.get(), want)


CASES = [
    # (raw shape z,y,x), pos, ext  -- faces, edges, corners, odd sizes, full box, single cell
    ((9, 11, 13), (1, 2, 3), (5, 4, 2)),
    ((9, 11, 13), (0, 0, 0), (13, 11, 9)),
    ((9, 11, 13), (12, 0, 8), (1, 11, 1)),
    ((9, 11, 13), (5, 5, 5), (1, 1, 1)),
    ((66, 66, 66), (1, 1, 65), (64, 64, 1)),  # z face r=1
    ((66, 66, 66), (65, 1, 1), (1, 64, 64)),  # x face r=1
    ((66, 66, 66), (1, 65, 1), (64, 1, 64)),  # y face r=1
    ((70, 70, 70), (67, 3, 3), (3, 64, 64)),  # x face r=3
    ((70, 70, 70), (3, 3, 3), (64, 3, 3)),  # yz edge
    ((70, 70, 70), (0, 67, 3), (3, 3, 64)),  # xy edge
    ((70, 70, 70), (67, 67, 67), (3, 3, 3)),  # corner
    ((5, 300, 1031), (7, 3, 1), (1000, 290, 3)),  # long odd rows
    ((130, 130, 130), (1, 1, 1), (128, 128, 128)),
]


@pytest.mark.parametrize("dtype", [np.uint8, np.int16, np.float32, np.float64])
@pytest.mark.parametrize("case", CASES, ids=[str(i) for i in range(len(CASES))])
def test_pack_unpack_translate_vs_oracle(dtype, case):
    raw, pos, ext = case
    rng = np.random.default_rng(7)
    a = rng.integers(0, 250, size=raw).astype(dtype)
    src = DevArray(a)
    packed = dev_pack(src, pos, ext).get().reshape(-1)
    assert np.array_equal(packed, no.pack(a, pos, ext))
    # unpack into a poisoned array at the same place
    dst = DevArray(np.full(raw, 3, dtype=dtype))
    dbuf = DevArray(packed.reshape(1, 1, -1))
    check(lib().sb_unpack(dst.pitched(), C.c_void_p(dbuf.ptr), i3(pos), i3(ext), a.dtype.itemsize, None))
    want = np.full(raw, 3, dtype=dtype)
    no.unpack(want, packed, pos, ext)
    assert np.array_equal(dst.get(), want)
    # translate into a differently shaped allocation at another position
    raw2 = (ext[2] + 3, ext[1] + 2, ext[0] + 5)
    dpos = (4, 1, 2)
    dst2 = DevArray(np.full(raw2, 9, dtype=dtype))
    check(lib().sb_translate(dst2.pitched(), i3(dpos), src.pitched(), i3(pos), i3(ext), a.dtype.itemsize, None))
    want2 = np.full(raw2, 9, dtype=dtype)
    no.translate(want2, dpos, a, pos, ext)
    assert np.array_equal(dst2.get(), want2)


def test_empty_and_invalid_copies():
    a = DevArray(np.zeros((4, 4, 4), dtype=np.float32))
    out = DevArray(np.zeros((1, 1, 4), dtype=np.float32))
    # empty extent: a no-op, not an error (the reference's planner never creates zero-size messages)
    check(lib().sb_pack(C.c_void_p(out.ptr), a.pitched(), i3((0, 0, 0)), i3((0, 4, 4)), 4, None))
    with pytest.raises(sb.StencilError):
        check(lib().sb_pack(C.c_void_p(out.ptr), a.pitched(), i3((0, 0, 0)), i3((1, 1, 1)), 3, None))
    with pytest.raises(sb.StencilError):
        check(lib().sb_pack(None, a.pitched(), i3((0, 0, 0)), i3((1, 1, 1)), 4, None))


@pytest.mark.parametrize("rname,radius", [("r2", 2), ("asym", None), ("r3", 3)])
def test_packer_wire_format_vs_oracle(rname, radius):
    """DevicePacker/DeviceUnpacker semantics (src/packer.cu): all 26 messages x {float, char, double}
    into ONE buffer in the reference's wire order, produced by one plan launch; byte-compare with the
    oracle; then unpack into a second domain and compare ghost regions."""
    sz = (12, 9, 7)
    if radius is None:
        ro = g.Radius.constant(1)
        ro.set_dir((1, 0, 0), 2)
        ro.set_dir((0, -1, 0), 3)
    else:
        ro = g.Radius.constant(radius)
    raw = g.raw_size(sz, ro)
    dts = [np.float32, np.int8, np.float64]
    rng = np.random.default_rng(11)
    host = [rng.integers(-100, 100, size=raw[::-1]).astype(dt) for dt in dts]
    dev = [DevArray(h) for h in host]
    msgs = [(d, g.halo_extent(g.neg(d), sz, ro)) for d in g.ALL_DIRS if ro.dir(g.neg(d)) != 0]
    total, entries = g.packer_layout(sz, ro, [np.dtype(d).itemsize for d in dts], msgs)
    buf = DevArray(np.zeros((1, 1, total), dtype=np.uint8))
    copies = []
    for e in entries:
        es = np.dtype(dts[e["q"]]).itemsize
        ext = e["ext"]
        dst = Pitched(buf.ptr + e["offset"], ext[0] * es, ext[1])
        copies.append(sb.box_copy(dst, (0, 0, 0), dev[e["q"]].pitched(), e["pos"], ext, es))
    plan = sb.CopyPlan(0, copies)
    assert plan.bytes == sum(e["nbytes"] for e in entries)
    plan.launch()
    want = no.packer_pack(host, sz, ro, msgs)
    assert np.array_equal(buf.get().reshape(-1), want)
    # unpack
    host2 = [np.zeros_like(h) for h in host]
    dev2 = [DevArray(h) for h in host2]
    _, uentries = g.unpacker_layout(sz, ro, [np.dtype(d).itemsize for d in dts], msgs)
    ucopies = []
    for e in uentries:
        es = np.dtype(dts[e["q"]]).itemsize
        ext = e["ext"]
        srcp = Pitched(buf.ptr + e["offset"], ext[0] * es, ext[1])
        ucopies.append(sb.box_copy(dev2[e["q"]].pitched(), e["pos"], srcp, (0, 0, 0), ext, es))
    sb.CopyPlan(0, ucopies).launch()
    no.packer_unpack(host2, want, sz, ro, msgs)
    for q in range(3):
        assert np.array_equal(dev2[q].get(), host2[q])


def test_plan_with_many_random_copies():
    rng = np.random.default_rng(5)
    raw = (40, 37, 53)
    src_h = rng.integers(0, 2**31, size=raw).astype(np.int32)
    dst_h = np.zeros((44, 41, 61), dtype=np.int32)
    src, dst = DevArray(src_h), DevArray(dst_h)
    want = dst_h.copy()
    copies = []
    # disjoint destination slabs in z so the copies are order independent
    z = 0
    while z < 40:
        ez = int(rng.integers(1, 4))
        ey, ex = int(rng.integers(1, 37)), int(rng.integers(1, 53))
        sp = (int(rng.integers(0, 53 - ex + 1)), int(rng.integers(0, 37 - ey + 1)), z if z + ez <= 40 else 40 - ez)
        dp = (int(rng.integers(0, 61 - ex + 1)), int(rng.integers(0, 41 - ey + 1)), z)
        if z + ez > 40:
            break
        copies.append(sb.box_copy(dst.pitched(), dp, src.pitched(), sp, (ex, ey, ez), 4))
        no.translate(want, dp, src_h, sp, (ex, ey, ez))
        z += ez
    plan = sb.CopyPlan(0, copies)
    plan.launch()
    assert np.array_equal(dst.get(), want)
    # idempotent: a second launch changes nothing
    plan.launch()
    assert np.array_equal(dst.get(), want)


def test_full_size_face_roundtrip_512():
    """BASELINE size (512^3, r=1, FP64): pack each face -> unpack into the opposite ghost layer must
    reproduce the periodic wrap; checked on device-resident data via host comparison of the faces only."""
    n, r = 512, 1
    raw = (n + 2, n + 2, n + 2)
    # a cheap analytic field so we never need the 1 GiB array on the host twice
    z, y, x = np.meshgrid(np.arange(raw[0]), np.arange(raw[1]), np.arange(raw[2]), indexing="ij", sparse=True)
    a = (x * 1.0 + y * 1000.0 + z * 1e6).astype(np.float64)
    src = DevArray(a)
    ro = g.Radius.constant(1)
    for d in [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, 0, -1), (1, 1, 0), (1, 1, 1)]:
        pos = g.halo_pos(d, (n, n, n), ro, False)
        ext = g.halo_extent(g.neg(d), (n, n, n), ro)
        got = dev_pack(src, pos, ext).get().reshape(-1)
        assert np.array_equal(got, no.pack(a, pos, ext)), d
