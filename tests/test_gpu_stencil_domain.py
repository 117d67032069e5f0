"""GPU parity of DistributedDomain.apply: time-stepping with linear stencil operators on 1, 2, 4 and 8 subdomains of one
GPU (uneven partitions), bit-identical to the numpy rule run on the global array -- with periodic wrap, or with the ghost
cells of a walled grid filled by tests/bc_oracle.py.  exchange=True (interior || exchange -> exterior) and exchange=False
after a manual exchange() give the same bits."""
import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
import stencil_op_oracle as so
from gpu_util import oracle_radius

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
UINT = {np.dtype(np.float32): np.uint32, np.dtype(np.float64): np.uint64}
SIZE = (26, 21, 19)


def lo_of(r):
    return (r.x(-1), r.y(-1), r.z(-1))


def load(dd, q, which, glob):
    """Compute cells of every local subdomain from the global [z, y, x] array; ghost cells NaN."""
    for d in dd.domains():
        raw, sz, org, rl = d.raw_size(), d.size(), d.origin(), lo_of(d.radius())
        a = np.full(raw[::-1], np.nan, glob.dtype)
        a[rl[2] : rl[2] + sz[2], rl[1] : rl[1] + sz[1], rl[0] : rl[0] + sz[0]] = glob[org[2] : org[2] + sz[2], org[1] : org[1] + sz[1], org[0] : org[0] + sz[0]]
        d.quantity_from_host(q, a, which)


def gather(dd, q, which="curr"):
    out = np.full(dd.size()[::-1], np.nan, dd.dtypes_[q])
    for d in dd.domains():
        full, sz, org, rl = d.quantity_to_host(q, which), d.size(), d.origin(), lo_of(d.radius())
        out[org[2] : org[2] + sz[2], org[1] : org[1] + sz[1], org[0] : org[0] + sz[0]] = full[rl[2] : rl[2] + sz[2], rl[1] : rl[1] + sz[1], rl[0] : rl[0] + sz[0]]
    return out


def same(a, b):
    u = UINT[a.dtype]
    return np.array_equal(a.view(u), b.view(u))


def domain(ndom, radius, dtypes, boundary=(P, P, P), bcs=None):
    dd = sb.DistributedDomain(*SIZE)
    dd.set_gpus([0] * ndom)
    dd.set_radius(radius)
    hs = [dd.add_data(dt, f"q{i}") for i, dt in enumerate(dtypes)]
    dd.set_boundary(*boundary)
    for (q, f), (kind, c) in (bcs or {}).items():
        dd.set_boundary_condition(hs[q], sb.FACES[f], sb.BC(kind, c))
    dd.realize()
    return dd, hs


def heat_terms():
    return [(0, (0, 0, 0), 1.0)] + [(s, o, 0.02 * w) for s, o, w in so.laplacian(4, (1.0, 0.9, 1.1))]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_heat_periodic(ndom, dtype):
    """u <- u + 0.02 lap4(u), 10 steps with swap; exchange=True and exchange=False (after a manual exchange) alike."""
    dtype = np.dtype(dtype)
    terms = heat_terms()
    op = sb.StencilOp(terms, dtype)
    u0 = np.random.default_rng(ndom).uniform(-1, 1, SIZE[::-1]).astype(dtype)
    want = u0
    for _ in range(10):
        want = so.apply_periodic(terms, want, None)
    for overlap in (True, False):
        dd, (h,) = domain(ndom, sb.Radius.face_edge_corner(2, 0, 0), [dtype])
        try:
            load(dd, h.id, "curr", u0)
            for _ in range(10):
                if overlap:
                    dd.apply(op, h, h)
                else:
                    dd.exchange()
                    dd.apply(op, h, h, exchange=False)
                dd.swap()
            assert same(gather(dd, h.id), want)
        finally:
            dd.close()


def test_heat_periodic_reference_placement(monkeypatch):
    """SB_ALLOC_ALIGN=0: allocations at the start of their blocks (rows of another 16-byte phase)."""
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    test_heat_periodic(4, np.float64)
    test_heat_periodic(2, np.float32)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_wave_dst_is_aux(ndom, dtype):
    """u_new = 2u - u_prev + c^2 lap(u), written over u_prev (dst == aux == next), 10 steps with swap."""
    dtype = np.dtype(dtype)
    terms = [(0, (0, 0, 0), 2.0), (1, (0, 0, 0), -1.0)] + [(s, o, 0.15 * w) for s, o, w in so.laplacian(2, (1.0, 1.0, 1.0))]
    op = sb.StencilOp(terms, dtype)
    rng = np.random.default_rng(10 + ndom)
    u, prev = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    dd, (h,) = domain(ndom, sb.Radius.constant(1), [dtype])
    try:
        load(dd, h.id, "curr", u)
        load(dd, h.id, "next", prev)
        for _ in range(10):
            dd.apply(op, (h, "next"), h, (h, "next"))
            dd.swap()
            u, prev = so.apply_periodic(terms, u, prev), u
        assert same(gather(dd, h.id), u)
        assert same(gather(dd, h.id, "next"), prev)
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_poisson_walls(ndom, dtype):
    """Jacobi relaxation of lap(u) = f with f in aux, walls on x and z (ODD(0) / EVEN / VALUE faces), 20 sweeps."""
    dtype = np.dtype(dtype)
    h2 = 0.25
    terms = [(0, o, 1.0 / 6.0) for o in ((-1, 0, 0), (1, 0, 0), (0, -1, 0), (0, 1, 0), (0, 0, -1), (0, 0, 1))] + [(1, (0, 0, 0), -h2 / 6.0)]
    op = sb.StencilOp(terms, dtype)
    boundary = (F, P, F)
    bcs = {(0, 0): (bo.ODD, 0.0), (0, 1): (bo.EVEN, 0.0), (0, 4): (bo.VALUE, 0.5), (0, 5): (bo.VALUE, -0.25)}
    radius = sb.Radius.face_edge_corner(1, 0, 0)
    rng = np.random.default_rng(20 + ndom)
    u, f = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    # the oracle: one subdomain covering the grid, ghost cells from the oracle's exchange and BC rule
    od = bo.Domains(SIZE, oracle_radius(radius), [dtype, dtype], n_subdomains=1, periodic=[b == P for b in boundary])
    rl = lo_of(radius)
    ua, fa = od.arrays[(0, 0, 0)]
    so._view(fa, rl, SIZE, (0, 0, 0))[...] = f
    so._view(ua, rl, SIZE, (0, 0, 0))[...] = u
    for _ in range(20):
        od.exchange()
        bo.apply_boundary(od, bcs)
        new = ua.copy()
        so.apply_box(terms, ua, fa, new, rl, SIZE)
        ua[...] = new
    want = so._view(ua, rl, SIZE, (0, 0, 0)).copy()
    dd, (hu, hf) = domain(ndom, radius, [dtype, dtype], boundary, bcs)
    try:
        load(dd, hu.id, "curr", u)
        load(dd, hf.id, "curr", f)
        load(dd, hf.id, "next", f)  # swap() turns both buffers of every quantity
        for _ in range(20):
            dd.apply(op, hu, hu, hf)
            dd.swap()
        assert same(gather(dd, hu.id), want)
    finally:
        dd.close()


def test_plan_cache_and_errors():
    dd, (h, g) = domain(2, sb.Radius.face_edge_corner(1, 0, 0), [np.float64, np.float32])
    try:
        lap = sb.StencilOp.laplacian(2, (1, 1, 1), np.float64)
        load(dd, h.id, "curr", np.zeros(SIZE[::-1]))
        dd.apply(lap, h, h)
        dd.apply(lap, h, h)
        assert len(dd._stencil_plans) == 1
        dd.swap()
        dd.apply(lap, h, h)
        assert len(dd._stencil_plans) == 2
        with pytest.raises(sb.StencilError, match="dst must not be src"):
            dd.apply(lap, (h, "curr"), h)
        with pytest.raises(sb.StencilError, match="src must be a curr buffer"):
            dd.apply(lap, h, (h, "next"))
        with pytest.raises(sb.StencilError, match="float32"):
            dd.apply(lap, g, h)
        with pytest.raises(sb.StencilError, match="term"):
            dd.apply(sb.StencilOp.laplacian(4, (1, 1, 1), np.float64), h, h)
        with pytest.raises(sb.StencilError, match="term"):
            dd.apply(sb.StencilOp([(0, (1, 1, 0), 1.0)], np.float64), h, h)
        with pytest.raises(sb.StencilError, match="no aux"):
            dd.apply(sb.StencilOp([(1, (0, 0, 0), 1.0)], np.float64), h, h)
    finally:
        dd.close()
    fresh = sb.DistributedDomain(8, 8, 8)
    fresh.add_data(np.float64)
    with pytest.raises(sb.StencilError, match="realize"):
        fresh.apply(sb.StencilOp.laplacian(2, (1, 1, 1), np.float64), sb.DataHandle(0, np.float64), sb.DataHandle(0, np.float64))
