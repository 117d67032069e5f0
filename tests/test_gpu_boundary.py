"""GPU parity of boundary conditions on non-periodic grids: DistributedDomain.exchange() with walls on some axes and a BC
per quantity and wall face must leave the WHOLE allocation of every quantity (compute cells, exchanged ghost cells, wall
ghost cells, untouched NONE ghost cells) bit-identical to the oracle's exchange followed by its per-cell BC rule
(tests/bc_oracle.py), over three exchange/swap rounds."""
import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
from gpu_util import oracle_radius
from oracle import np_oracle as no

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
WALLS = {"all": (F, F, F), "z": (P, P, F), "x": (F, P, P)}
FLOAT_KINDS = [(bo.VALUE, 1.5), (bo.EVEN, 0.0), (bo.ODD, 0.5), (bo.ODD, 0.0), (bo.NONE, 0.0), (bo.VALUE, -2.25), (bo.ODD, -1.75)]


def mixed_bcs(dtypes, boundary):
    """A different kind per (quantity, wall face); raw (integer) quantities get EVEN or NONE."""
    bcs = {}
    for q, dt in enumerate(dtypes):
        for f in range(6):
            if boundary[f // 2] == P:
                continue
            if np.dtype(dt).kind == "f":
                bcs[(q, f)] = FLOAT_KINDS[(3 * q + f) % len(FLOAT_KINDS)]
            else:
                bcs[(q, f)] = (bo.EVEN, 0.0) if (q + f) % 3 else (bo.NONE, 0.0)
    return bcs


def run_bc_check(size, radius, gpus, dtypes, boundary, bcs, rounds=3):
    dd = sb.DistributedDomain(*size)
    dd.set_gpus(gpus)
    dd.set_radius(radius)
    hs = [dd.add_data(dt, f"d{i}") for i, dt in enumerate(dtypes)]
    dd.set_boundary(*boundary)
    for (q, f), (kind, c) in bcs.items():
        dd.set_boundary_condition(hs[q], sb.FACES[f], sb.BC(kind, c))
    dd.realize()
    od = bo.Domains(size, oracle_radius(radius), dtypes, n_subdomains=len(gpus), periodic=[b == P for b in boundary])
    try:
        assert [d.size() for d in dd.domains()] == [od.sizes[i] for i in dd.domain_idx_]
        for rep in range(rounds):
            fld = lambda q, x, y, z, rep=rep: no.hash_field(q, x, y, z) + 7 * rep  # noqa: E731
            od.fill(fld)
            for di, d in enumerate(dd.domains()):
                for q in range(len(dtypes)):
                    d.quantity_from_host(q, od.arrays[dd.domain_idx_[di]][q])
            dd.exchange()
            od.exchange()
            bo.apply_boundary(od, bcs)
            for di, d in enumerate(dd.domains()):
                idx = dd.domain_idx_[di]
                for q in range(len(dtypes)):
                    got, want = d.quantity_to_host(q), od.arrays[idx][q]
                    assert np.array_equal(got, want), (rep, idx, q, int(np.count_nonzero(got != want)))
            dd.swap()
    finally:
        dd.close()


@pytest.mark.parametrize("walls", ["all", "z", "x"])
@pytest.mark.parametrize("ndom", [1, 4, 8])
@pytest.mark.parametrize("size,rname", [((12, 10, 14), "c2"), ((13, 7, 9), "f2e1")])
def test_boundary_mixed_kinds(size, rname, ndom, walls):
    radius = sb.Radius.constant(2) if rname == "c2" else sb.Radius.face_edge_corner(2, 1, 0)
    dtypes = [np.float32, np.float64, np.int8]
    run_bc_check(size, radius, [0] * ndom, dtypes, WALLS[walls], mixed_bcs(dtypes, WALLS[walls]))


@pytest.mark.parametrize("walls", ["all", "z", "x"])
def test_boundary_radius1_faces_and_asymmetric(walls):
    """Face-only radius 1 (the jacobi shape) and an asymmetric radius (+x 2, -x 1, -y 3)."""
    dtypes = [np.float64, np.float32]
    run_bc_check((12, 10, 14), sb.Radius.face_edge_corner(1, 0, 0), [0] * 4, dtypes, WALLS[walls], mixed_bcs(dtypes, WALLS[walls]))
    r = sb.Radius.constant(1)
    r.set_dir((1, 0, 0), 2)
    r.set_dir((0, -1, 0), 3)
    run_bc_check((13, 11, 9), r, [0, 0], dtypes, WALLS[walls], mixed_bcs(dtypes, WALLS[walls]))


def test_boundary_fp64_128_radius2_8_subdomains():
    dtypes = [np.float64]
    bcs = mixed_bcs(dtypes, WALLS["all"])
    run_bc_check((128, 128, 128), sb.Radius.constant(2), [0] * 8, dtypes, WALLS["all"], bcs)
    run_bc_check((128, 128, 128), sb.Radius.constant(2), [0] * 8, dtypes, WALLS["all"], {(0, f): (bo.ODD, 0.5) for f in range(6)}, rounds=1)


@pytest.mark.parametrize("walls", ["all", "x"])
def test_boundary_raw_element_sizes(walls):
    """EVEN on 2-, 4-, 8- and 16-byte elements (int16, int32, int64, complex128 copied as raw bytes): the raw-copy paths of
    every element size, row and mirrored-row segments."""
    dtypes = [np.int16, np.int32, np.int64, np.complex128, np.float32]
    bcs = {(q, f): ((bo.EVEN, 0.0) if q < 4 else (bo.ODD, 0.5)) for q in range(5) for f in range(6) if WALLS[walls][f // 2] == F}
    run_bc_check((13, 10, 9), sb.Radius.constant(2), [0, 0], dtypes, WALLS[walls], bcs)


def test_fixed_without_bcs_keeps_wall_ghosts():
    """FIXED with no BC: no message crosses the walls and the wall ghost cells keep what was there."""
    run_bc_check((12, 10, 14), sb.Radius.constant(1), [0, 0], [np.float32], (F, P, F), {})
