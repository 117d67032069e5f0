"""CPU checks of non-periodic grids and boundary conditions (BCs): the oracle's per-cell rule on hand-computed cases,
the product's region geometry (sb_bc_regions) and wall-aware message plan against the oracle, and every error realize()
reports.  No GPU is used."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
from gpu_util import oracle_radius
from oracle import geometry as g
from oracle import np_oracle as no
from stencil_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED


def one_domain(size, radius, dtype, periodic, fn):
    od = bo.Domains(size, radius, [dtype], 1, periodic=periodic)
    od.fill(fn)
    od.exchange()
    return od, od.arrays[(0, 0, 0)][0]


def xfield(q, x, y, z):
    return 10.0 * x + 0.5 * y + 0.25 * z


# ------------------------------------------------------------------------------------------------ hand-computed cases
@pytest.mark.parametrize("kind,c", [(bo.VALUE, 3.5), (bo.EVEN, 0.0), (bo.ODD, 0.0), (bo.ODD, 2.0)])
def test_each_kind_on_x_walls(kind, c):
    """Walls on x, radius 2 on the x faces: ghost cells 0, 1 mirror compute cells 3, 2 (low side), ghost cells 6, 7 of a
    4-cell row mirror cells 5, 4 (high side)."""
    r = g.Radius.face_edge_corner(2, 0, 0)
    od, a = one_domain((4, 3, 3), r, np.float64, (False, True, True), xfield)
    bo.apply_boundary(od, {(0, 0): (kind, c), (0, 1): (kind, c)})
    row = a[3, 3, :]  # z = 1, y = 1 in compute coordinates
    comp = [10.0 * x + 0.5 + 0.25 for x in range(4)]
    assert list(row[2:6]) == comp
    mirror = {0: comp[1], 1: comp[0], 6: comp[3], 7: comp[2]}
    for i, m in mirror.items():
        want = {bo.VALUE: c, bo.EVEN: m, bo.ODD: 2 * c - m}[kind]
        assert row[i] == want, (i, row[i], want)
    # the y and z faces are periodic: their ghost cells came from the exchange
    assert a[3, 1, 3] == 10.0 * 1 + 0.5 * 2 + 0.25  # y ghost below row 0 holds row 2 (size 3, wrap)


def test_corner_odd_x_meets_value_y():
    """Order x -> y -> z: in the (-x,-y) edge ODD(1) on -x is applied first, then VALUE(5) on -y overwrites it; with the
    kinds swapped VALUE(5) on -x comes first and ODD(1) on -y gives 2*1 - 5."""
    r = g.Radius.constant(1)
    od, a = one_domain((3, 3, 3), r, np.float64, (False, False, True), xfield)
    bo.apply_boundary(od, {(0, 0): (bo.ODD, 1.0), (0, 2): (bo.VALUE, 5.0)})
    assert a[2, 0, 0] == 5.0
    assert a[2, 0, 2] == 5.0  # y face only: VALUE
    assert a[2, 2, 0] == 2 * 1.0 - a[2, 2, 1]  # x face only: ODD about the face
    od, a = one_domain((3, 3, 3), r, np.float64, (False, False, True), xfield)
    bo.apply_boundary(od, {(0, 0): (bo.VALUE, 5.0), (0, 2): (bo.ODD, 1.0)})
    assert a[2, 0, 0] == 2 * 1.0 - 5.0
    # EVEN on both: the corner is the doubly mirrored compute cell
    od, a = one_domain((3, 3, 3), r, np.float64, (False, False, True), xfield)
    bo.apply_boundary(od, {(0, 0): (bo.EVEN, 0.0), (0, 2): (bo.EVEN, 0.0)})
    assert a[2, 0, 0] == a[2, 1, 1]
    # float32 arithmetic stays in float32
    od, a = one_domain((3, 3, 3), r, np.float32, (False, True, True), lambda q, x, y, z: 0.1 * x + 0.3)
    bo.apply_boundary(od, {(0, 0): (bo.ODD, 0.1)})
    assert a[2, 2, 0] == np.float32(2) * np.float32(0.1) - a[2, 2, 1]


def test_even_on_int8():
    r = g.Radius.constant(2)
    od, a = one_domain((4, 4, 4), r, np.int8, (True, True, False), lambda q, x, y, z: (x + 3 * y + 7 * z) % 100)
    bo.apply_boundary(od, {(0, 4): (bo.EVEN, 0.0), (0, 5): (bo.EVEN, 0.0)})
    assert a.dtype == np.int8
    assert np.array_equal(a[0], a[3]) and np.array_equal(a[1], a[2])
    assert np.array_equal(a[7], a[4]) and np.array_equal(a[6], a[5])


def test_periodic_y_between_walled_x_and_z():
    r = g.Radius.constant(1)
    fn = lambda q, x, y, z: 100.0 * x + 10.0 * y + z  # noqa: E731
    od, a = one_domain((4, 3, 5), r, np.float64, (False, True, False), fn)
    bo.apply_boundary(od, {(0, f): (bo.ODD, 0.0) for f in (0, 1, 4, 5)})
    # y ghost rows wrap: alloc y 0 holds y = 2, alloc y 4 holds y = 0, at compute x and z
    assert a[1, 0, 1] == fn(0, 0, 2, 0) and a[1, 4, 1] == fn(0, 0, 0, 0)
    # x walls: antisymmetric about the face
    assert a[1, 1, 0] == -a[1, 1, 1] and a[1, 1, 5] == -a[1, 1, 4]
    # the (-x, -y) edge: mirrored on x only, from the y ghost the exchange filled
    assert a[1, 0, 0] == -a[1, 0, 1] == -fn(0, 0, 2, 0)
    # the (-x, -z) edge: mirrored on both, two ODD(0) steps give back the compute cell
    assert a[0, 1, 0] == a[1, 1, 1]
    # an (x, y, z) corner with walls on x and z and a periodic y
    assert a[0, 0, 0] == a[1, 0, 1]


def test_fixed_without_bcs_keeps_poison():
    r = g.Radius.constant(1)
    od, a = one_domain((4, 3, 5), r, np.float32, (False, True, True), xfield)
    assert a[1, 1, 0] == no.poison(np.float32) and a[1, 1, 5] == no.poison(np.float32)
    assert np.array_equal(a, od.expected_after_exchange(xfield, (0, 0, 0), 0))


# ------------------------------------------------------------------------------------------------ product vs oracle
def named_radius(name):
    if name.startswith("c"):
        return sb.Radius.constant(int(name[1:]))
    if name == "faces1":
        return sb.Radius.face_edge_corner(1, 0, 0)
    if name == "f2e1":
        return sb.Radius.face_edge_corner(2, 1, 0)
    if name == "f3e2c1":
        return sb.Radius.face_edge_corner(3, 2, 1)
    r = sb.Radius.constant(0)
    r.set_dir((1, 0, 0), 2)
    r.set_dir((-1, 0, 0), 1)
    return r  # px2mx1


@pytest.mark.parametrize("rname", ["c1", "c2", "c3", "faces1", "f2e1", "f3e2c1", "px2mx1"])
@pytest.mark.parametrize("size,n", [((12, 10, 14), 4), ((13, 7, 9), 4), ((13, 11, 9), 2)])
def test_bc_regions_match_the_oracle(rname, size, n):
    r = named_radius(rname)
    ro = oracle_radius(r)
    part = g.NodePartition(size, ro, 1, n)
    sizes = sorted({part.subdomain_size(i) for i in part.all_indices()})
    for sz in sizes:
        for mask in range(64):
            for kind in (bo.EVEN, bo.VALUE, bo.ODD):
                kinds = [kind if mask & (1 << f) else bo.NONE for f in range(6)]
                try:
                    bo.check_widths(sz, ro, kinds)
                except ValueError:
                    with pytest.raises(sb.StencilError):
                        sb.bc_regions(sz, r, kinds)
                    continue
                got = sb.bc_regions(sz, r, kinds)
                want = bo.bc_regions(sz, ro, kinds)
                assert got == want, (sz, kinds)


@pytest.mark.parametrize("boundary", [(F, F, F), (P, P, F), (F, P, P), (F, P, F), (P, P, P)])
@pytest.mark.parametrize("size,n,rname", [((12, 10, 14), 4, "c2"), ((13, 7, 9), 6, "f2e1"), ((16, 16, 16), 8, "c1")])
def test_plan_with_walls_matches_the_oracle(boundary, size, n, rname):
    r = named_radius(rname)
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([0] * n)
    dd.set_radius(r)
    dd.add_data(np.float32)
    dd.set_boundary(*boundary)
    dd.do_placement()
    periodic = [b == P for b in boundary]
    key = lambda m: (m["src_idx"], m["dir"])  # noqa: E731
    got = sorted(({k: m[k] for k in ("src_idx", "dst_idx", "dir", "src_pos", "dst_pos", "ext")} for m in dd.plan_messages()), key=key)
    od = bo.Domains(size, oracle_radius(r), [np.float32], n, periodic=periodic)
    want = sorted(bo.plan_sends(od.dim, od.sizes, od.radius, periodic), key=key)
    assert got == want
    if all(periodic):
        assert want == sorted(g.plan_sends(od.dim, od.sizes, od.radius), key=key)


def test_set_boundary_forms():
    dd = sb.DistributedDomain(8, 8, 8)
    assert dd.boundary_ == (P, P, P)
    dd.set_boundary(F)
    assert dd.boundary_ == (F, F, F)
    dd.set_boundary(P, P, F)
    assert dd.boundary_ == (P, P, F)
    with pytest.raises(sb.StencilError):
        dd.set_boundary(P, F)
    t = sb.Topology((2, 1, 3), (F, P, F))
    assert t.get_neighbor((0, 0, 0), (-1, 0, 0)) is None
    assert t.get_neighbor((0, 0, 0), (1, -1, 0)) == (1, 0, 0)
    assert t.get_neighbor((1, 0, 2), (0, 0, 1)) is None
    assert sb.get_neighbor((0, 0, 0), (-1, 0, 0), (2, 1, 3)) == (1, 0, 0)  # the module function stays periodic


# ------------------------------------------------------------------------------------------------ errors at realize()
def realize_error(boundary, dtype, face, bc, size=(8, 8, 8), radius=1, gpus=(0,)):
    dd = sb.DistributedDomain(*size)
    dd.set_gpus(list(gpus))
    dd.set_radius(radius)
    h = dd.add_data(dtype)
    dd.set_boundary(*boundary)
    dd.set_boundary_condition(h, face, bc)
    with pytest.raises(sb.StencilError) as e:
        dd.realize()  # fails in its host-side checks, before anything is allocated
    return str(e.value)


def test_bc_on_a_periodic_axis_is_rejected():
    assert "periodic" in realize_error((P, P, F), np.float64, (1, 0, 0), sb.BC.EVEN())


def test_value_and_odd_on_integers_are_rejected():
    for bc in (sb.BC.VALUE(1.0), sb.BC.ODD(0.0)):
        assert "float" in realize_error((F, F, F), np.int8, (0, 0, -1), bc)
    assert "float" in realize_error((F, F, F), np.int32, (0, 0, 1), sb.BC.ODD(1.0))


def test_mirror_wider_than_the_subdomain_is_rejected():
    # 8 subdomains of 4 cells along x, ghost width 5
    msg = realize_error((F, P, P), np.float32, (-1, 0, 0), sb.BC.EVEN(), size=(16, 4, 4), radius=5, gpus=(0, 0, 0, 0))
    assert "ghost width" in msg
    # VALUE reads nothing: allowed
    assert sb.bc_regions((4, 4, 4), sb.Radius.constant(5), [bo.VALUE, 0, 0, 0, 0, 0])


def test_c_abi_rejects_bad_plans_without_a_gpu():
    r = sb.Radius.constant(1)
    q = _lib.BcQuantity(_lib.Pitched(0x1000, 80, 10), 1, (C.c_double * 6)(), 0, _lib.I6(1, 0, 0, 0, 0, 0))
    h = C.c_void_p()
    rc = sb.lib().sb_bc_plan_create(C.byref(h), 0, (_lib.BcQuantity * 1)(q), 1, _lib.i3((8, 8, 8)), r.c27())
    assert rc == -1 and b"floating" in sb.lib().sb_last_error()
    q.dtype, q.elem_size = 2, 4  # f64 with 4-byte elements
    rc = sb.lib().sb_bc_plan_create(C.byref(h), 0, (_lib.BcQuantity * 1)(q), 1, _lib.i3((8, 8, 8)), r.c27())
    assert rc == -1 and b"dtype" in sb.lib().sb_last_error()
    with pytest.raises(sb.StencilError):
        sb.bc_regions((8, 8, 8), r, [7, 0, 0, 0, 0, 0])


def test_jacobi_refuses_walls():
    from stencil_b200.jacobi import Jacobi3D

    dd = sb.DistributedDomain(8, 8, 8)
    dd.set_boundary(P, P, F)
    with pytest.raises(sb.StencilError):
        Jacobi3D(dd, sb.DataHandle(0, np.float64))


def test_bc_structs_match_the_header(tmp_path):
    src = tmp_path / "probe.c"
    src.write_text('#include <stdio.h>\n#include "stencil_b200.h"\n'
                   'int main(void) { printf("%zu %zu\\n", sizeof(sb_bc_region), sizeof(sb_bc_quantity)); return 0; }\n')
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_lib.BcRegion), C.sizeof(_lib.BcQuantity)]


def test_oracle_apply_is_one_pass_per_axis():
    """The one-pass rule equals the x walls, then the y walls, then the z walls applied as separate passes."""
    r = g.Radius.constant(2)
    kinds_all = list(itertools.product([bo.VALUE, bo.EVEN, bo.ODD], repeat=3))
    for ks in kinds_all[::4]:
        bcs = {(0, 2 * a + s): (ks[a], 0.5 + a) for a in range(3) for s in (0, 1)}
        od, a1 = one_domain((5, 4, 6), r, np.float64, (False, False, False), xfield)
        bo.apply_boundary(od, bcs)
        _, a2 = one_domain((5, 4, 6), r, np.float64, (False, False, False), xfield)
        for axis in range(3):
            kinds, values = [0] * 6, [0.0] * 6
            for s in (0, 1):
                kinds[2 * axis + s], values[2 * axis + s] = bcs[(0, 2 * axis + s)]
            # one pass of one axis over the whole shell, reading what the earlier passes wrote
            shell = [k if (f // 2 == axis) else 0 for f, k in enumerate(kinds)]
            full = g.Radius.constant(2)
            regs = bo.bc_regions((5, 4, 6), full, shell)
            src = a2.copy()
            for reg in regs:
                lo = list(reg["pos"])
                hi = [lo[b] + reg["ext"][b] for b in range(3)]
                # widen the box to the whole allocation on the other axes
                for b in range(3):
                    if b != axis:
                        lo[b], hi[b] = 0, a2.shape[2 - b]
                idx = [np.arange(lo[b], hi[b]) for b in range(3)]
                sidx = list(idx)
                sidx[axis] = reg["mirror"][axis] - idx[axis]
                v = src[np.ix_(sidx[2], sidx[1], sidx[0])]
                f = 2 * axis + (reg["dir"][axis] > 0)
                if kinds[f] == bo.VALUE:
                    v = np.full_like(v, values[f])
                elif kinds[f] == bo.ODD:
                    v = 2 * values[f] - v
                a2[np.ix_(idx[2], idx[1], idx[0])] = v
        assert np.array_equal(a1, a2), ks
