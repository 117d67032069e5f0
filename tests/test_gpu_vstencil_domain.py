"""GPU parity of DistributedDomain.apply with coefficient fields: ten steps of a heterogeneous heat equation
u <- u + dt div(kappa grad u), kappa on the faces in three quantities, on 1, 2, 4 and 8 subdomains of one GPU, each step
bit-identical to the numpy rule of tests/vstencil_oracle.py -- on a periodic grid, and on a grid walled on x and z where
exchange() fills kappa's ghost cells with its own EVEN BC and u's with VALUE BCs.  Every step swaps, so the coefficient
quantities turn with u (they hold the same compute cells in curr and next)."""
import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
import stencil_op_oracle as so
import vstencil_oracle as vo
from gpu_util import oracle_radius
from test_gpu_stencil_domain import SIZE, domain, gather, lo_of, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
SPACING = (0.9, 1.0, 1.1)


def heat_terms(dt):
    return [(s, o, dt * w, k, c) for s, o, w, k, c in vo.div_grad(SPACING)] + [(0, (0, 0, 0), 1.0)]


def kappas(rng, dtype):
    return [rng.uniform(0.2, 2.0, SIZE[::-1]).astype(dtype) for _ in range(3)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_heat_periodic(ndom, dtype):
    dtype = np.dtype(dtype)
    terms = heat_terms(0.05)
    op = sb.StencilOp(terms, dtype)
    rng = np.random.default_rng(30 + ndom)
    u = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    ks = kappas(rng, dtype)
    for overlap in (True, False):
        dd, (h, kx, ky, kz) = domain(ndom, sb.Radius.face_edge_corner(1, 0, 0), [dtype] * 4)
        try:
            load(dd, h.id, "curr", u)
            for q, k in zip((kx, ky, kz), ks):
                load(dd, q.id, "curr", k)
                load(dd, q.id, "next", k)
            want = u
            for step in range(10):
                if overlap:
                    dd.apply(op, h, h, coefs=[kx, ky, kz])
                else:
                    dd.exchange()
                    dd.apply(op, h, h, exchange=False, coefs=[kx, ky, kz])
                dd.swap()
                want = vo.apply_periodic(terms, want, None, ks)
                assert same(gather(dd, h.id), want), step
        finally:
            dd.close()


def test_heat_periodic_reference_placement(monkeypatch):
    """SB_ALLOC_ALIGN=0: allocations at the start of their blocks (rows of another 16-byte phase)."""
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    test_heat_periodic(4, np.float64)
    test_heat_periodic(2, np.float32)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_heat_walls(ndom, dtype):
    """Walls on x and z: u has VALUE faces, each kappa EVEN faces; y is periodic."""
    dtype = np.dtype(dtype)
    terms = heat_terms(0.05)
    op = sb.StencilOp(terms, dtype)
    boundary = (F, P, F)
    radius = sb.Radius.face_edge_corner(1, 0, 0)
    bcs = {(0, 0): (bo.VALUE, 1.0), (0, 1): (bo.VALUE, -0.5), (0, 4): (bo.VALUE, 0.25), (0, 5): (bo.VALUE, 0.0)}
    for q in (1, 2, 3):
        for f in (0, 1, 4, 5):
            bcs[(q, f)] = (bo.EVEN, 0.0)
    rng = np.random.default_rng(40 + ndom)
    u = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    ks = kappas(rng, dtype)
    od = bo.Domains(SIZE, oracle_radius(radius), [dtype] * 4, n_subdomains=1, periodic=[b == P for b in boundary])
    rl = lo_of(radius)
    arrs = od.arrays[(0, 0, 0)]
    for a, v in zip(arrs, [u] + ks):
        so._view(a, rl, SIZE, (0, 0, 0))[...] = v
    dd, hs = domain(ndom, radius, [dtype] * 4, boundary, bcs)
    try:
        load(dd, hs[0].id, "curr", u)
        for q, k in zip(hs[1:], ks):
            load(dd, q.id, "curr", k)
            load(dd, q.id, "next", k)
        for step in range(10):
            od.exchange()
            bo.apply_boundary(od, bcs)
            new = arrs[0].copy()
            vo.apply_box(terms, arrs[0], None, arrs[1:], new, rl, SIZE)
            arrs[0][...] = new
            dd.apply(op, hs[0], hs[0], coefs=hs[1:])
            dd.swap()
            assert same(gather(dd, hs[0].id), so._view(arrs[0], rl, SIZE, (0, 0, 0)).copy()), step
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wave_variable_speed(dtype):
    """u_new = 2u - u_prev + c^2 dt^2 lap4(u), written over u_prev, c^2 in one quantity, 10 steps on 4 subdomains."""
    dtype = np.dtype(dtype)
    terms = [(0, (0, 0, 0), 2.0), (1, (0, 0, 0), -1.0)] + [(0, o, 0.01 * w, 0, (0, 0, 0)) for _, o, w in so.laplacian(4, (1.0, 1.0, 1.0))]
    op = sb.StencilOp(terms, dtype)
    rng = np.random.default_rng(50)
    u, prev = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    c2 = rng.uniform(0.5, 1.5, SIZE[::-1]).astype(dtype)
    dd, (h, c) = domain(4, sb.Radius.face_edge_corner(2, 0, 0), [dtype, dtype])
    try:
        load(dd, h.id, "curr", u)
        load(dd, h.id, "next", prev)
        load(dd, c.id, "curr", c2)
        load(dd, c.id, "next", c2)
        for _ in range(10):
            dd.apply(op, (h, "next"), h, (h, "next"), coefs=[c])
            dd.swap()
            u, prev = vo.apply_periodic(terms, u, prev, [c2]), u
        assert same(gather(dd, h.id), u)
        assert same(gather(dd, h.id, "next"), prev)
    finally:
        dd.close()


def test_apply_coefficient_errors_and_cache():
    dd, (h, k, g) = domain(2, sb.Radius.face_edge_corner(1, 0, 0), [np.float64, np.float64, np.float32])
    try:
        op = sb.StencilOp([(0, (0, 0, 0), 1.0, 0, (1, 0, 0))], np.float64)
        load(dd, h.id, "curr", np.zeros(SIZE[::-1]))
        dd.apply(op, h, h, coefs=[k])
        dd.apply(op, h, h, coefs=[k])
        assert len(dd._stencil_plans) == 1
        dd.apply(op, h, h, coefs=[h])  # a coefficient may alias src
        assert len(dd._stencil_plans) == 2
        with pytest.raises(sb.StencilError, match="reads 1 coefficient fields, but 0"):
            dd.apply(op, h, h)
        with pytest.raises(sb.StencilError, match="reads 1 coefficient fields, but 2"):
            dd.apply(op, h, h, coefs=[k, k])
        with pytest.raises(sb.StencilError, match="reads 0 coefficient fields, but 1"):
            dd.apply(sb.StencilOp.laplacian(2, (1, 1, 1), np.float64), h, h, coefs=[k])
        with pytest.raises(sb.StencilError, match="float32"):
            dd.apply(op, h, h, coefs=[g])
        with pytest.raises(sb.StencilError, match="must not be dst"):
            dd.apply(op, (k, "curr"), h, coefs=[k])
        with pytest.raises(sb.StencilError, match="curr buffer"):
            dd.apply(op, h, h, coefs=[(k, "next")])
        with pytest.raises(sb.StencilError, match="coefficient offset"):
            dd.apply(sb.StencilOp([(0, (0, 0, 0), 1.0, 0, (1, 1, 0))], np.float64), h, h, coefs=[k])
    finally:
        dd.close()
