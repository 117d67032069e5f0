"""The exchange plan of the C ABI (sb_exchange_messages, sb_staging_layout; include/stencil/exchange_plan.hpp) against
independent statements, on the CPU.  The message list of every subdomain equals the wall-aware oracle plan
(tests/bc_oracle.py) element by element and in order; the staging layout of every (src, dst) neighbour pair equals the
rule restated below.  Both ends of an exchange derive these independently, so the order and the offsets are part of
what is checked, not only the set."""
import ctypes as C

import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
from gpu_util import oracle_radius
from stencil_b200 import _lib
from stencil_b200.domain import exchange_messages, grid_args

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
BOUNDARIES = {"PPP": (P, P, P), "FFF": (F, F, F), "PPF": (P, P, F), "FPF": (F, P, F)}


def asymmetric_radius() -> sb.Radius:
    """A different radius per direction, 0 in some (so those directions send nothing)."""
    r = sb.Radius.constant(0)
    for d in sb.ALL_DIRS:
        r.set_dir(d, ((d[0] + 1) + 2 * (d[1] + 1) + 5 * (d[2] + 1)) % 3)
    return r


RADII = {
    "c1": lambda: sb.Radius.constant(1),
    "c2": lambda: sb.Radius.constant(2),
    "f2e1": lambda: sb.Radius.face_edge_corner(2, 1, 0),
    "asym": asymmetric_radius,
}
# one subdomain (every neighbour is itself), 2 (x cut in two: the same neighbour on both sides of a periodic axis,
# y and z of 1), 3 (a periodic axis of 3), 4, 6 and 8
CASES = [(size, n) for size in ((13, 9, 8), (12, 10, 14)) for n in (1, 2, 3, 4, 6, 8)]
ELEM_SIZES = [(8,), (4, 8), (2, 4, 8, 16), (4,)]


def grid(size, n, rname, walls):
    r = RADII[rname]()
    part = sb.Partition(size, r, 1, n)
    topo = sb.Topology(part.dim, BOUNDARIES[walls])
    periodic = [b == P for b in BOUNDARIES[walls]]
    od = bo.Domains(size, oracle_radius(r), [np.float64], n, periodic=periodic)
    assert tuple(od.dim) == tuple(part.dim)
    for idx in part.indices():
        assert tuple(od.sizes[idx]) == part.subdomain_size(idx)
    return part, topo, r, bo.plan_sends(od.dim, od.sizes, od.radius, periodic)


def staging_oracle(msgs, dst, elem_sizes):
    """The staging rule: src's messages to dst in order, each one's quantities in order; a pair is staged when a row of
    it is shorter than 64 bytes; each entry starts at the next multiple of 16 bytes; total = end of the last entry."""
    entries, off = [], 0
    for i, m in enumerate(msgs):
        if m["dst_idx"] != dst:
            continue
        for q, es in enumerate(elem_sizes):
            if m["ext"][0] * es < 64:
                off = (off + 15) // 16 * 16
                entries.append((i, q, off))
                off += es * m["ext"][0] * m["ext"][1] * m["ext"][2]
    return off, entries


def staging_layout(part, topo, r, src, dst, elem_sizes, cap=None):
    cap = 26 * len(elem_sizes) if cap is None else cap
    out, total = (_lib.Staged * max(cap, 1))(), C.c_int64(-1)
    n = _lib.check(sb.lib().sb_staging_layout(*grid_args(part, topo, r), _lib.i3(src), _lib.i3(dst),
                                              (C.c_int64 * len(elem_sizes))(*elem_sizes), len(elem_sizes), out, cap, C.byref(total)))
    return total.value, [(s.msg, s.q, s.offset) for s in out[:n]]


@pytest.mark.parametrize("walls", list(BOUNDARIES))
@pytest.mark.parametrize("rname", list(RADII))
@pytest.mark.parametrize("size,n", CASES)
def test_messages_and_staging_match_the_oracle(size, n, rname, walls):
    part, topo, r, want_all = grid(size, n, rname, walls)
    for src in part.indices():
        want = [m for m in want_all if m["src_idx"] == src]
        got = exchange_messages(part, topo, r, src)
        assert got == want, src
        for dst in sorted({m["dst_idx"] for m in want}):
            for es in ELEM_SIZES:
                assert staging_layout(part, topo, r, src, dst, es) == staging_oracle(want, dst, es), (src, dst, es)


def test_staging_layout_can_be_empty():
    """FFF walls and one subdomain along x: no message to the z neighbour crosses x, and 12 FP64 cells per row are 96
    bytes, so the pair has nothing staged; FP32 rows of 48 bytes are staged."""
    part, topo, r, want_all = grid((12, 10, 14), 2, "c1", "FFF")
    assert tuple(part.dim) == (1, 1, 2)
    want = [m for m in want_all if m["src_idx"] == (0, 0, 0)]
    assert staging_layout(part, topo, r, (0, 0, 0), (0, 0, 1), (8,)) == (0, []) == staging_oracle(want, (0, 0, 1), (8,))
    total, entries = staging_layout(part, topo, r, (0, 0, 0), (0, 0, 1), (4,))
    assert total > 0 and (total, entries) == staging_oracle(want, (0, 0, 1), (4,))
    # a pair that exchanges nothing at all (a subdomain and itself across a wall) is empty too
    assert staging_layout(part, topo, r, (0, 0, 0), (0, 0, 0), (4, 8)) == (0, [])


def test_message_and_staged_counts_fit_the_documented_bounds():
    part, topo, r, _ = grid((13, 9, 8), 1, "c1", "PPP")
    msgs = exchange_messages(part, topo, r, (0, 0, 0))
    assert len(msgs) == 26 and all(m["dst_idx"] == (0, 0, 0) for m in msgs)
    assert [m["dir"] for m in msgs] == sb.ALL_DIRS  # z, then y, then x, each ascending
    total, entries = staging_layout(part, topo, r, (0, 0, 0), (0, 0, 0), (1, 2))
    assert len(entries) == 2 * 26 and all(off % 16 == 0 for _, _, off in entries)


def _raw():
    """The library without ctypes argument checking, to pass NULL where the typed binding refuses it."""
    return C.CDLL(sb.LIB_PATH)


def _expect_invalid(rc):
    assert rc == -1  # SB_ERR_INVALID
    assert sb.lib().sb_last_error().decode()


def test_invalid_input_is_rejected():
    L = sb.lib()
    part, topo, r, _ = grid((12, 10, 14), 8, "c1", "PPF")
    dim, base, rem, bnd, r27 = grid_args(part, topo, r)
    out = (_lib.Message * 26)()
    staged = (_lib.Staged * 64)()
    total = C.c_int64()
    es = (C.c_int64 * 2)(4, 8)
    i3 = _lib.i3
    ok = i3((0, 0, 0))

    def messages(dim=dim, bnd=bnd, src=ok, cap=26):
        return L.sb_exchange_messages(dim, base, rem, bnd, r27, src, out, cap)

    def layout(dim=dim, bnd=bnd, src=ok, dst=i3((1, 0, 0)), es=es, nq=2, cap=64):
        return L.sb_staging_layout(dim, base, rem, bnd, r27, src, dst, es, nq, staged, cap, C.byref(total))

    nmsg, nstaged = messages(), layout()
    assert nmsg == 17 and nstaged > 0  # (0, 0, 0) sits against the -z wall
    for a in range(3):
        bad = list(part.dim)
        bad[a] = 0
        _expect_invalid(messages(dim=i3(bad)))
        _expect_invalid(layout(dim=i3(bad)))
        for v in (0, 3, -1):
            b = list(bnd)
            b[a] = v
            _expect_invalid(messages(bnd=(C.c_int32 * 3)(*b)))
            _expect_invalid(layout(bnd=(C.c_int32 * 3)(*b)))
        for off in (-1, part.dim[a]):
            idx = [0, 0, 0]
            idx[a] = off
            _expect_invalid(messages(src=i3(idx)))
            _expect_invalid(layout(src=i3(idx)))
            _expect_invalid(layout(dst=i3(idx)))
    _expect_invalid(messages(cap=nmsg - 1))
    _expect_invalid(layout(cap=nstaged - 1))
    for bad in ((0, 8), (4, -8)):
        _expect_invalid(layout(es=(C.c_int64 * 2)(*bad)))
    _expect_invalid(layout(nq=-1))
    # NULL arguments
    raw = _raw()
    args = [dim, base, rem, bnd, r27, ok]
    for k in range(len(args)):
        a = list(args)
        a[k] = None
        _expect_invalid(raw.sb_exchange_messages(*a, out, 26))
        _expect_invalid(raw.sb_staging_layout(*a, i3((1, 0, 0)), es, 2, staged, 64, C.byref(total)))
    _expect_invalid(raw.sb_exchange_messages(*args, None, 26))
    _expect_invalid(raw.sb_staging_layout(*args, None, es, 2, staged, 64, C.byref(total)))
    _expect_invalid(raw.sb_staging_layout(*args, i3((1, 0, 0)), None, 2, staged, 64, C.byref(total)))
    _expect_invalid(raw.sb_staging_layout(*args, i3((1, 0, 0)), es, 2, None, 64, C.byref(total)))
    _expect_invalid(raw.sb_staging_layout(*args, i3((1, 0, 0)), es, 2, staged, 64, None))
    # an empty result needs no output buffer
    assert raw.sb_staging_layout(*args, i3((1, 0, 0)), None, 0, None, 0, C.byref(total)) == 0 and total.value == 0


def test_plan_messages_adds_only_the_owners():
    """DistributedDomain.plan_messages (this rank's, or any rank's by number) is the C ABI list of each owned subdomain,
    in partition order, with the owner fields added."""
    dd = sb.DistributedDomain(12, 10, 14)
    dd.set_gpus([0, 0])
    dd.set_radius(sb.Radius.face_edge_corner(2, 1, 0))
    dd.add_data(np.float32)
    dd.set_boundary(F, P, F)
    dd.do_placement()
    _, _, _, want = grid((12, 10, 14), 2, "f2e1", "FPF")
    keys = ("src_idx", "dst_idx", "dir", "src_pos", "dst_pos", "ext")
    got = dd.plan_messages()
    assert got == dd.plan_messages(0) and dd.plan_messages(1) == []
    assert [{k: m[k] for k in keys} for m in got] == want
    assert all((0, m["src_slot"]) == dd._owner[m["src_idx"]] for m in got)
    assert all((m["dst_rank"], m["dst_slot"]) == dd._owner[m["dst_idx"]] for m in got)
