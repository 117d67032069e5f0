"""GPU parity of DistributedDomain.apply_system: Maxwell's equations on a Yee grid (leapfrog of in-place E and H updates)
on 1, 2, 4 and 8 subdomains of one GPU, bit-identical after every step to the numpy rule of tests/system_oracle.py --
periodic, and walled with a BC per component filled by exchange() (tests/bc_oracle.py); the Yee scheme's exact
propagation of a discrete plane wave; staggered acoustics with coefficient fields on a walled grid; curl(grad u) = 0
exactly across subdomains; and the error paths and the plan cache of apply_system."""
import numpy as np
import pytest

import bc_oracle as bo
import stencil_b200 as sb
import stencil_op_oracle as so
import system_oracle as yo
from gpu_util import oracle_radius
from test_gpu_stencil_domain import SIZE, domain, gather, lo_of, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
H = (1.0, 0.5, 0.75)
IDENT = [(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)]


def yee_terms(dt):
    """(E update, H update), eps = mu = 1.  E: inputs Hx, Hy, Hz, Ex, Ey, Ez -> Ex, Ey, Ez, E = E + dt curl- H.
    H: inputs Ex, Ey, Ez, Hx, Hy, Hz -> Hx, Hy, Hz, H = H - dt curl+ E."""
    return IDENT + yo.scaled(yo.curl(-1, H), dt), IDENT + yo.scaled(yo.curl(1, H), -dt)


def yee_step(dd, hs, e_sys, h_sys):
    """One leapfrog step: E from H, then H from E, both in place in the curr buffers."""
    E, Hf = hs[:3], hs[3:]
    dd.apply_system(e_sys, [(q, "curr") for q in E], list(Hf) + [(q, "curr") for q in E])
    dd.apply_system(h_sys, [(q, "curr") for q in Hf], list(E) + [(q, "curr") for q in Hf])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_yee_periodic(ndom, dtype):
    dtype = np.dtype(dtype)
    et, ht = yee_terms(0.2)
    e_sys, h_sys = sb.StencilSystem(et, dtype), sb.StencilSystem(ht, dtype)
    rng = np.random.default_rng(60 + ndom)
    f = [rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(6)]
    dd, hs = domain(ndom, sb.Radius.face_edge_corner(1, 0, 0), [dtype] * 6)
    try:
        for q, a in zip(hs, f):
            load(dd, q.id, "curr", a)
        for step in range(10):
            yee_step(dd, hs, e_sys, h_sys)
            f[:3] = yo.apply_periodic(et, f[3:] + f[:3])
            f[3:] = yo.apply_periodic(ht, f[:3] + f[3:])
            for q, a in zip(hs, f):
                assert same(gather(dd, q.id), a), (step, q.id)
        assert len(dd._stencil_plans) == 2  # no swap: one plan set per update
    finally:
        dd.close()


def test_yee_periodic_reference_placement(monkeypatch):
    """SB_ALLOC_ALIGN=0: allocations at the start of their blocks (rows of another 16-byte phase)."""
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    test_yee_periodic(4, np.float64)
    test_yee_periodic(2, np.float32)


def yee_bcs():
    """Walls on x and z: on a wall normal to axis a, E_a and the tangential H are EVEN, the tangential E and H_a ODD."""
    bcs = {}
    for a, faces in ((0, (0, 1)), (2, (4, 5))):
        for c in range(3):
            for f in faces:
                bcs[(c, f)] = (bo.EVEN if c == a else bo.ODD, 0.0)
                bcs[(3 + c, f)] = (bo.ODD if c == a else bo.EVEN, 0.0)
    return bcs


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_yee_walls(ndom, dtype):
    dtype = np.dtype(dtype)
    et, ht = yee_terms(0.2)
    e_sys, h_sys = sb.StencilSystem(et, dtype), sb.StencilSystem(ht, dtype)
    boundary, radius, bcs = (F, P, F), sb.Radius.face_edge_corner(1, 0, 0), yee_bcs()
    rng = np.random.default_rng(70 + ndom)
    f = [rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(6)]
    od = bo.Domains(SIZE, oracle_radius(radius), [dtype] * 6, n_subdomains=1, periodic=[b == P for b in boundary])
    rl = lo_of(radius)
    arrs = od.arrays[(0, 0, 0)]
    for a, v in zip(arrs, f):
        so._view(a, rl, SIZE, (0, 0, 0))[...] = v
    dd, hs = domain(ndom, radius, [dtype] * 6, boundary, bcs)
    try:
        for q, a in zip(hs, f):
            load(dd, q.id, "curr", a)
        for step in range(10):
            yee_step(dd, hs, e_sys, h_sys)
            for terms, ins, outs in ((et, arrs[3:] + arrs[:3], arrs[:3]), (ht, arrs[:3] + arrs[3:], arrs[3:])):
                od.exchange()
                bo.apply_boundary(od, bcs)
                yo.apply_box(terms, ins, outs, rl, SIZE)
            for q in range(6):
                assert same(gather(dd, hs[q].id), so._view(arrs[q], rl, SIZE, (0, 0, 0)).copy()), (step, q)
    finally:
        dd.close()


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_yee_plane_wave(axis):
    """A discrete plane wave along `axis` (E_b, H_c with b, c the next axes in cyclic order), h = 1, dt = 0.5, one
    wavelength over 16 cells, 32^3 cells on 2 subdomains (so the interiors run the tile kernel and the exterior slabs the
    cell kernel).  E at t = 0 and H at t = dt/2, positions staggered by h/2, with the Yee dispersion relation
    sin(w dt / 2) / dt = sin(k h / 2) / h: the scheme propagates the mode exactly up to rounding."""
    n, dt, steps = 32, 0.5, 200
    k = 2 * np.pi / 16
    w = 2 / dt * np.arcsin(dt * np.sin(k / 2))
    b, c = (axis + 1) % 3, (axis + 2) % 3
    x = np.arange(n, dtype=np.float64)
    shape = [1, 1, 1]
    shape[2 - axis] = n

    def field(v):
        return np.broadcast_to(v.reshape(shape), (n, n, n)).copy()

    unit = (1.0, 1.0, 1.0)
    e_sys = sb.StencilSystem(IDENT + yo.scaled(yo.curl(-1, unit), dt), np.float64)
    h_sys = sb.StencilSystem(IDENT + yo.scaled(yo.curl(1, unit), -dt), np.float64)
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0, 0])
    dd.set_radius(sb.Radius.face_edge_corner(1, 0, 0))
    hs = [dd.add_data(np.float64, f"q{i}") for i in range(6)]
    dd.realize()
    try:
        zero = np.zeros((n, n, n))
        init = [zero] * 6
        init[b] = field(np.cos(k * x))
        init[3 + c] = field(np.cos(k * (x + 0.5) - w * dt / 2))
        for q, a in zip(hs, init):
            load(dd, q.id, "curr", a)
        for _ in range(steps):
            yee_step(dd, hs, e_sys, h_sys)
        err_e = np.abs(gather(dd, hs[b].id) - field(np.cos(k * x - w * dt * steps))).max()
        err_h = np.abs(gather(dd, hs[3 + c].id) - field(np.cos(k * (x + 0.5) - w * dt * (steps + 0.5)))).max()
        print(f"plane wave along {'xyz'[axis]}: max error after {steps} steps E {err_e:.3e} H {err_h:.3e}")
        assert err_e <= 1e-11 and err_h <= 1e-11, (err_e, err_h)
        for q in range(6):
            if q not in (b, 3 + c):
                assert not gather(dd, hs[q].id).any()
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_acoustics_walls(dtype):
    """Staggered acoustics, v_a on the faces above a cell, p at its centre, b_a (inverse density) on the faces and K
    (bulk modulus) at the centres: v = v - dt b D+ p, then p = p - dt K div- v.  Walls on x and z with v normal ODD(0)
    and p EVEN; 10 steps on 4 subdomains against the oracle."""
    dtype = np.dtype(dtype)
    dt = 0.1
    # v update: inputs p, vx, vy, vz, bx, by, bz -> vx, vy, vz;  p update: inputs vx, vy, vz, p, K -> p
    v_terms = [(j, 1 + j, (0, 0, 0), 1.0) for j in range(3)] + [t[:3] + (-dt * t[3], 4 + t[0], (0, 0, 0)) for t in yo.grad(1, H)]
    p_terms = [(0, 3, (0, 0, 0), 1.0)] + [t[:3] + (-dt * t[3], 4, (0, 0, 0)) for t in yo.div(-1, H)]
    v_sys, p_sys = sb.StencilSystem(v_terms, dtype), sb.StencilSystem(p_terms, dtype)
    boundary, radius = (F, P, F), sb.Radius.face_edge_corner(1, 0, 0)
    bcs = {}
    for a, faces in ((0, (0, 1)), (2, (4, 5))):
        for f in faces:
            bcs[(0, f)] = (bo.EVEN, 0.0)
            for j in range(3):
                bcs[(1 + j, f)] = (bo.ODD if j == a else bo.EVEN, 0.0)
            for q in range(4, 8):
                bcs[(q, f)] = (bo.EVEN, 0.0)
    rng = np.random.default_rng(80)
    f = [rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(4)] + [rng.uniform(0.5, 2, SIZE[::-1]).astype(dtype) for _ in range(4)]
    od = bo.Domains(SIZE, oracle_radius(radius), [dtype] * 8, n_subdomains=1, periodic=[b == P for b in boundary])
    rl = lo_of(radius)
    arrs = od.arrays[(0, 0, 0)]
    for a, v in zip(arrs, f):
        so._view(a, rl, SIZE, (0, 0, 0))[...] = v
    dd, hs = domain(4, radius, [dtype] * 8, boundary, bcs)  # p, vx, vy, vz, bx, by, bz, K
    try:
        for q, a in zip(hs, f):
            load(dd, q.id, "curr", a)
        p, v, bq, K = hs[0], hs[1:4], hs[4:7], hs[7]
        for step in range(10):
            dd.apply_system(v_sys, [(q, "curr") for q in v], [p] + [(q, "curr") for q in v] + list(bq))
            dd.apply_system(p_sys, [(p, "curr")], list(v) + [(p, "curr"), K])
            for terms, ins, outs in ((v_terms, arrs[:7], arrs[1:4]), (p_terms, arrs[1:4] + [arrs[0], arrs[7]], arrs[:1])):
                od.exchange()
                bo.apply_boundary(od, bcs)
                yo.apply_box(terms, ins, outs, rl, SIZE)
            for q in range(4):
                assert same(gather(dd, hs[q].id), so._view(arrs[q], rl, SIZE, (0, 0, 0)).copy()), (step, q)
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("stagger", [-1, 0, 1])
def test_curl_grad_is_zero(stagger, dtype):
    """Integer-valued u (|u| < 2^16) and h = 0.5, 0.25: every value is exact, so curl(grad u) is 0 with no tolerance."""
    dtype = np.dtype(dtype)
    h = (0.5, 0.25, 0.5)
    rng = np.random.default_rng(90)
    u = rng.integers(-(2**16) + 1, 2**16, SIZE[::-1]).astype(dtype)
    dd, hs = domain(4, sb.Radius.face_edge_corner(1, 0, 0), [dtype] * 7)
    try:
        load(dd, hs[0].id, "curr", u)
        g, c = hs[1:4], hs[4:7]
        dd.apply_system(sb.StencilSystem.grad(stagger, h, dtype), [(q, "curr") for q in g], [hs[0]])
        dd.apply_system(sb.StencilSystem.curl(stagger, h, dtype), [(q, "curr") for q in c], list(g))
        for q in c:
            out = gather(dd, q.id)
            assert np.array_equal(out, np.zeros_like(out))
    finally:
        dd.close()


def test_apply_system_errors_and_cache():
    dd, hs = domain(2, sb.Radius.face_edge_corner(1, 0, 0), [np.float64] * 4 + [np.float32])
    a, b, c, d, s = hs
    try:
        for q in (a, b, c, d):
            load(dd, q.id, "curr", np.zeros(SIZE[::-1]))
        grad = sb.StencilSystem.grad(1, (1, 1, 1), np.float64)
        dd.apply_system(grad, [b, c, d], [a])
        dd.apply_system(grad, [b, c, d], [a])
        assert len(dd._stencil_plans) == 1
        dd.apply_system(grad, [b, c, d], [a], exchange=False)
        assert len(dd._stencil_plans) == 2
        with pytest.raises(sb.StencilError, match="3 outputs, but 1 inputs and 2 outputs"):
            dd.apply_system(grad, [b, c], [a])
        with pytest.raises(sb.StencilError, match="float32"):
            dd.apply_system(grad, [b, c, s], [a])
        with pytest.raises(sb.StencilError, match="distinct"):
            dd.apply_system(grad, [b, b, d], [a])
        with pytest.raises(sb.StencilError, match="must be a curr buffer"):
            dd.apply_system(grad, [b, c, d], [(a, "next")])
        with pytest.raises(sb.StencilError, match="output 0 is input 0"):
            dd.apply_system(grad, [(a, "curr"), c, d], [a])
        with pytest.raises(sb.StencilError, match="is read by a term, but it is None"):
            dd.apply_system(grad, [b, c, d], [None])
        with pytest.raises(sb.StencilError, match="not a StencilSystem"):
            dd.apply_system(sb.StencilOp.laplacian(2, (1, 1, 1), np.float64), [b], [a])
        with pytest.raises(sb.StencilError, match="ghost box|face radius"):
            dd.apply_system(sb.StencilSystem([(0, 0, (2, 0, 0), 1.0)], np.float64), [b], [a])
        # an input no term reads may be None; an output may be an input read only at offset 0
        dd.apply_system(sb.StencilSystem([(0, 1, (0, 0, 0), 2.0)], np.float64, nin=2), [(b, "curr")], [None, (b, "curr")])
        with pytest.raises(sb.StencilError, match="call realize"):
            sb.DistributedDomain(8, 8, 8).apply_system(grad, [b, c, d], [a])
    finally:
        dd.close()
