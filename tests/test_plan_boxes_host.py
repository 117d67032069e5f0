"""The box checks of the operator, system and transfer plans without a GPU: coordinates the kernels take as 32-bit int
(allocation-relative lo, lo + extent, the read window with its reach, the fused restriction's fine window, the
prolongation's parent window and offset) must lie below 2^31, and a box must have fewer than 2^32 cells, counted without
int64 overflow.  Boxes just inside the limits pass validation (SB_ERR_NOGPU on a machine without a device; a plan made
on a device is destroyed unlaunched).  In long box lists the messages name the right box, empty boxes included.  Every
allocation here is a fake pitched pointer: no plan built on one is ever launched."""
import ctypes as C
import re

import numpy as np
import pytest

import stencil_b200 as sb
from stencil_b200._lib import I3, TRANSFER_PROLONG, TRANSFER_RESTRICT, Pitched, lib

OK, INVALID, NOGPU = 0, -1, -3
F32, F64 = 1, 2
BIG = 1 << 31
CENTRE = sb.StencilOp([(0, (0, 0, 0), 1.0)], np.float64)


def fake(k, pitch, ysize):
    return Pitched(0x100000 * (k + 1), pitch, ysize)


def boxes_arg(boxes):
    lo = (C.c_int64 * (3 * max(1, len(boxes))))(*[v for b in boxes for v in b[0]])
    hi = (C.c_int64 * (3 * max(1, len(boxes))))(*[v for b in boxes for v in b[1]])
    return lo, hi


def outcome(rc, h, destroy):
    """(rc, message); a plan a device made is destroyed here, never launched."""
    msg = lib().sb_last_error().decode()
    if rc == OK:
        destroy(h)
    return rc, msg


def op_plan(size, boxes, terms=CENTRE, dtype=F32, origin=(0, 0, 0)):
    """sb_stencil_plan_create over fake allocations of size (x, y, z) elements."""
    es = 4 if dtype == F32 else 8
    lo, hi = boxes_arg(boxes)
    h = C.c_void_p()
    rc = lib().sb_stencil_plan_create(C.byref(h), 0, dtype, terms.c_terms(), len(terms.terms), fake(0, size[0] * es, size[1]),
                                      fake(1, size[0] * es, size[1]), Pitched(None, 0, 0), I3(*origin), size[2], len(boxes), lo, hi)
    return outcome(rc, h, lib().sb_stencil_plan_destroy)


def sys_plan(size, boxes, terms=((0, 0, (0, 0, 0), 1.0),)):
    system = sb.StencilSystem(list(terms), np.float64)
    lo, hi = boxes_arg(boxes)
    outs = (Pitched * system.nout)(*[fake(8 + j, size[0] * 8, size[1]) for j in range(system.nout)])
    ins = (Pitched * system.nin)(*[fake(i, size[0] * 8, size[1]) for i in range(system.nin)])
    h = C.c_void_p()
    rc = lib().sb_stencil_sys_plan_create(C.byref(h), 0, F64, system.c_terms(), len(system.terms), outs, system.nout, ins, system.nin,
                                          I3(0, 0, 0), size[2], len(boxes), lo, hi)
    return outcome(rc, h, lib().sb_stencil_plan_destroy)


def fused_plan(csize, fsize, boxes, corigin=(0, 0, 0), forigin=(0, 0, 0)):
    """sb_transfer_oplan_create, a centre-only op: coarse dst of csize, fine src of fsize (x, y, z elements, FP64)."""
    lo, hi = boxes_arg(boxes)
    h = C.c_void_p()
    rc = lib().sb_transfer_oplan_create(C.byref(h), 0, F64, CENTRE.c_terms(), 1, fake(0, csize[0] * 8, csize[1]), I3(*corigin), csize[2],
                                        fake(1, fsize[0] * 8, fsize[1]), I3(*forigin), fsize[2], Pitched(None, 0, 0), len(boxes), lo, hi)
    return outcome(rc, h, lib().sb_transfer_plan_destroy)


def transfer_plan(kind, dsize, dorigin, ssize, sorigin, lo, hi):
    h = C.c_void_p()
    rc = lib().sb_transfer_plan_create(C.byref(h), 0, F64, kind, fake(0, dsize[0] * 8, dsize[1]), I3(*dorigin), dsize[2],
                                       fake(1, ssize[0] * 8, ssize[1]), I3(*sorigin), ssize[2], Pitched(None, 0, 0), I3(*lo), I3(*hi))
    return outcome(rc, h, lib().sb_transfer_plan_destroy)


def passes(r):
    """Validation passed: a plan on a device, SB_ERR_NOGPU without one."""
    assert r[0] in (OK, NOGPU), r


def refused(r, pattern):
    assert r[0] == INVALID and re.search(pattern, r[1]), r


# ------------------------------------------------------------------------------------------- 32-bit coordinates
def test_lo_past_2_31():
    """A 1 x 1 x (2^31 + 64) FP32 allocation (about 8.6 GB) holds a box at z = 2^31, whose lo an int cannot hold."""
    size = (1, 1, BIG + 64)
    refused(op_plan(size, [((0, 0, BIG), (1, 1, BIG + 1))]), r"box 0: the op reads cells 2147483648 \.\. 2147483648 on axis z, beyond")
    refused(op_plan(size, [((0, 0, BIG - 1), (1, 1, BIG))]), r"box 0: .* axis z, beyond the kernels' 32-bit")
    passes(op_plan(size, [((0, 0, BIG - 2), (1, 1, BIG - 1))]))


def test_read_window_past_2_31():
    """The window counts the reach: a box ending at 2^31 - 2 that reads one cell above it is the last that fits."""
    up = sb.StencilOp([(0, (0, 0, 0), 1.0), (0, (0, 0, 1), 0.5)], np.float64)
    size = (1, 1, BIG + 8)
    passes(op_plan(size, [((0, 0, 5), (1, 1, BIG - 2))], terms=up, dtype=F64))
    refused(op_plan(size, [((0, 0, 5), (1, 1, BIG - 1))], terms=up, dtype=F64), r"box 0: the op reads cells 5 \.\. 2147483647 on axis z")


def test_lo_past_2_31_through_acc_origin():
    """Global coordinates may be anything: what must fit is the allocation-relative window."""
    size = (1, 1, BIG + 64)
    g = -(1 << 40)
    passes(op_plan(size, [((0, 0, g + BIG - 2), (1, 1, g + BIG - 1))], origin=(0, 0, g)))
    refused(op_plan(size, [((0, 0, g + BIG), (1, 1, g + BIG + 1))], origin=(0, 0, g)), r"box 0: .* on axis z, beyond")


def test_extents_whose_cell_count_overflows():
    """(2^32 + 1) x (2^32 - 1) x 1 cells: the int64 product is -1.  The x extent alone is past 2^31."""
    e = ((1 << 32) + 1, (1 << 32) - 1, 1)
    refused(op_plan(e, [((0, 0, 0), e)]), r"box 0: the op reads cells 0 \.\. 4294967296 on axis x, beyond")


def test_cell_count_without_int64_overflow():
    """(2^31 - 1)^2 x 4 cells fit the coordinates, and their int64 product wraps negative: still more than 2^32 cells."""
    n = BIG - 1
    refused(op_plan((n, n, 4), [((0, 0, 0), (n, n, 4))]), r"box 0: more than 2\^32 cells")
    refused(sys_plan((n, n, 4), [((0, 0, 0), (n, n, 4))]), r"box 0: more than 2\^32 cells")
    refused(op_plan((1 << 16, 1 << 16, 1), [((0, 0, 0), (1 << 16, 1 << 16, 1))]), r"box 0: more than 2\^32 cells")
    passes(op_plan((1 << 16, 1 << 16, 1), [((0, 0, 0), (1 << 16, (1 << 16) - 1, 1))]))


def test_system_lo_past_2_31():
    size = (1, 1, BIG + 64)
    refused(sys_plan(size, [((0, 0, BIG), (1, 1, BIG + 1))]), r"box 0: input 0 is read at cells 2147483648 \.\. 2147483648 on axis z, beyond")
    passes(sys_plan(size, [((0, 0, BIG - 2), (1, 1, BIG - 1))]))


def test_fused_restriction_fine_origin_past_2_31():
    """A coarse box at z = 2^30 fits, its fine origin 2^31 does not; the fine window reads one cell beyond each side."""
    cz = (1 << 30) + 1
    csize, fsize = (2, 2, cz), (8, 8, 2 * cz + 4)
    refused(fused_plan(csize, fsize, [((1, 1, 1 << 30), (2, 2, cz))]),
            r"box 0: the fused restriction reads fine cells 2147483647 \.\. 2147483650 on axis z, beyond")
    refused(fused_plan(csize, fsize, [((1, 1, (1 << 30) - 1), (2, 2, 1 << 30))]), r"box 0: the fused restriction reads fine .* axis z, beyond")
    passes(fused_plan(csize, fsize, [((1, 1, (1 << 30) - 2), (2, 2, (1 << 30) - 1))]))


def test_restriction_fine_origin_past_2_31():
    cz = (1 << 30) + 1
    restrict = lambda z: transfer_plan(TRANSFER_RESTRICT, (2, 2, cz), (0, 0, 0), (4, 4, 2 * cz), (0, 0, 0), (1, 1, z), (2, 2, z + 1))  # noqa: E731
    refused(restrict(1 << 30), r"box 0: the restriction reads fine cells 2147483648 \.\. 2147483649 on axis z, beyond")
    refused(restrict((1 << 30) - 1), r"box 0: the restriction reads fine cells 2147483646 \.\. 2147483647 on axis z, beyond")
    passes(restrict((1 << 30) - 2))


def test_prolongation_window_and_offset():
    """The parent window [floor(lo / 2) - 1, floor((hi - 1) / 2) + 2) and off = 2 src_acc_origin - dst_acc_origin."""
    # the last fine plane whose end fits is 2^31 - 2
    passes(transfer_plan(TRANSFER_PROLONG, (4, 4, BIG), (0, 0, 0), (4, 4, (1 << 30) + 4), (-1, -1, -1), (1, 1, BIG - 2), (2, 2, BIG - 1)))
    refused(transfer_plan(TRANSFER_PROLONG, (4, 4, BIG + 2), (0, 0, 0), (4, 4, (1 << 30) + 4), (-1, -1, -1), (1, 1, BIG - 1), (2, 2, BIG)),
            r"box 0: dst is written at cells 2147483647 \.\. 2147483647 on axis z, beyond")
    # the parents sit 2^30 cells into a coarse allocation that starts 2^30 + 1 cells below the fine one's origin / 2
    so = -(1 << 30) - 1
    refused(transfer_plan(TRANSFER_PROLONG, (4, 4, 4), (0, 0, 0), (4, 4, (1 << 30) + 8), (-1, -1, so), (1, 1, 0), (2, 2, 2)),
            r"offset 2 \* src_acc_origin - dst_acc_origin = -2147483650 on axis z does not fit 32 bits")
    passes(transfer_plan(TRANSFER_PROLONG, (4, 4, 4), (0, 0, 0), (4, 4, (1 << 30) + 8), (-1, -1, so + 2), (1, 1, 0), (2, 2, 2)))
    # parents past 2^31 in the coarse allocation
    refused(transfer_plan(TRANSFER_PROLONG, (4, 4, 4), (0, 0, 1 << 32), (4, 4, BIG + 8), (-1, -1, 0), (1, 1, 1 << 32), (2, 2, (1 << 32) + 2)),
            r"box 0: the prolongation reads coarse cells 2147483647 \.\. 2147483649 on axis z, beyond")


# ------------------------------------------------------------------------------------------- long box lists
@pytest.mark.parametrize("kind", ["op", "sys", "fused"])
def test_messages_name_the_box(kind):
    size = (40, 40, 40)
    make = {"op": lambda b: op_plan(size, b, dtype=F64), "sys": lambda b: sys_plan(size, b),
            "fused": lambda b: fused_plan((20, 20, 30), (60, 60, 60), b, forigin=(-2, -2, -2))}[kind]
    boxes = [((2, 2, k), (6, 6, k + 1)) if k not in (4, 9) else ((2, 2, k), (2, 6, k + 1)) for k in range(25)]
    passes(make(boxes))
    inverted = list(boxes)
    inverted[20] = ((2, 2, 20), (6, 6, 19))
    refused(make(inverted), r"^box 20: lo > hi on axis z$")
    outside = list(boxes)
    outside[17] = ((2, 2, 17), (6, 60, 18))
    refused(make(outside), r"^box 17: .* on axis y, outside the allocation")
    # an empty box is numbered too, and is not checked against the allocation
    far = list(boxes)
    far[9] = ((2, 2, 100), (2, 6, 101))
    far[12] = ((2, 2, 12), (6, 6, 12 - 1))
    refused(make(far), r"^box 12: lo > hi on axis z$")


def test_fused_only_empty_boxes():
    """A fused plan of empty boxes has no launch: made without a device, with 0 bytes."""
    lo, hi = boxes_arg([((1, 1, 1), (1, 3, 3)), ((2, 2, 2), (4, 2, 4)), ((0, 0, 0), (5, 5, 0))])
    h = C.c_void_p()
    rc = lib().sb_transfer_oplan_create(C.byref(h), 0, F64, CENTRE.c_terms(), 1, fake(0, 64, 8), I3(0, 0, 0), 8, fake(1, 160, 20), I3(-2, -2, -2),
                                        20, Pitched(None, 0, 0), 3, lo, hi)
    assert rc == OK, lib().sb_last_error().decode()
    try:
        assert lib().sb_transfer_plan_bytes(h) == 0
    finally:
        lib().sb_transfer_plan_destroy(h)
