"""GPU parity of coloured DistributedDomain.apply: red-black SOR sweeps in place (each colour one apply, f on aux) on 1,
2, 3, 4 and 8 uneven subdomains of one GPU, on odd global sizes, periodic and walled (Dirichlet ODD and VALUE faces and
an EVEN face), bit-identical to tests/colour_oracle.py after every colour pass -- so identical across partitions --
with exchange=True (interior || exchange -> exterior) and with exchange=False after a manual exchange(); the same
under SB_ALLOC_ALIGN=0; an 8-colour sweep of a 27-point relaxation; the damped update u + theta (div(kappa grad u) - f)
with kappa on a walled grid; and the red-black Gauss-Seidel contraction rate of a periodic Helmholtz problem."""
import math

import numpy as np
import pytest

import bc_oracle as bo
import colour_oracle as co
import stencil_b200 as sb
import stencil_op_oracle as so
from gpu_util import oracle_radius
from test_gpu_stencil_domain import gather, lo_of, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
SIZE = (25, 21, 19)  # odd on every axis: on a periodic axis a cell and its wrapped neighbour can share a colour


def domain(ndom, radius, dtypes, size=SIZE, boundary=(P, P, P), bcs=None):
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([0] * ndom)
    dd.set_radius(radius)
    hs = [dd.add_data(dt, f"q{i}") for i, dt in enumerate(dtypes)]
    dd.set_boundary(*boundary)
    for (q, f), (kind, c) in (bcs or {}).items():
        dd.set_boundary_condition(hs[q], sb.FACES[f], sb.BC(kind, c))
    dd.realize()
    return dd, hs


def sor_terms(omega=1.6, h=1.0, sigma=0.3):
    return co.relax(co.helmholtz(h, sigma), omega)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 3, 4, 8])
def test_sor_periodic(ndom, dtype):
    """10 red-black SOR sweeps, each colour an in-place apply; the oracle after every colour pass."""
    dtype = np.dtype(dtype)
    terms = sor_terms()
    op = sb.StencilOp(terms, dtype)
    rng = np.random.default_rng(ndom)
    u0, f = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    for overlap in (True, False):
        dd, (hu, hf) = domain(ndom, sb.Radius.face_edge_corner(1, 0, 0), [dtype, dtype])
        try:
            load(dd, hu.id, "curr", u0)
            load(dd, hf.id, "curr", f)
            want = u0
            for sweep in range(10):
                for c in range(2):
                    if overlap:
                        dd.apply(op, (hu, "curr"), hu, hf, colour=(2, c))
                    else:
                        dd.exchange()
                        dd.apply(op, (hu, "curr"), hu, hf, exchange=False, colour=(2, c))
                    want = co.apply_periodic(terms, want, f, [], want, 2, c)
                    assert same(gather(dd, hu.id), want), (sweep, c, overlap)
        finally:
            dd.close()


def low_side_radius():
    """Radius 1 on the -x, -y and -z faces only: what an upwind op needs."""
    r = sb.Radius.face_edge_corner(0, 0, 0)
    for d in ((-1, 0, 0), (0, -1, 0), (0, 0, -1)):
        r.set_dir(d, 1)
    return r


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 3, 8])
def test_upwind_one_sided_radius(ndom, dtype):
    """An upwind relaxation (offsets -x, -y, -z) in place on a radius that is 1 on the low faces and 0 on the high ones,
    periodic with odd lengths: the wrapped ghost of x = 0 holds cell n - 1, of the same colour.  exchange() sends the
    high-side slabs that the low-side ghosts read, so the overlapped interior must not write them; the exterior then
    reads their old values, as the rule says.  Bits after every colour pass, with and without the overlap."""
    dtype = np.dtype(dtype)
    A = [(0, (0, 0, 0), 4.0), (0, (-1, 0, 0), -1.0), (0, (0, -1, 0), -0.75), (0, (0, 0, -1), -0.5)]
    terms = co.relax(A, 1.3)
    op = sb.StencilOp(terms, dtype)
    rng = np.random.default_rng(60 + ndom)
    u0, f = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    for overlap in (True, False):
        dd, (hu, hf) = domain(ndom, low_side_radius(), [dtype, dtype])
        try:
            load(dd, hu.id, "curr", u0)
            load(dd, hf.id, "curr", f)
            want = u0
            for sweep in range(6):
                for c in range(2):
                    if overlap:
                        dd.apply(op, (hu, "curr"), hu, hf, colour=(2, c))
                    else:
                        dd.exchange()
                        dd.apply(op, (hu, "curr"), hu, hf, exchange=False, colour=(2, c))
                    want = co.apply_periodic(terms, want, f, [], want, 2, c)
                    assert same(gather(dd, hu.id), want), (sweep, c, overlap)
        finally:
            dd.close()


def test_in_place_interior_keeps_clear_of_sent_slabs(monkeypatch):
    """The overlapped interior of an in-place apply is cut by the radius of both sides of each axis, so it writes none of
    the high-side slabs exchange() sends; an out-of-place apply keeps the interior the domain reports."""
    from stencil_b200 import stencil_op

    boxes = []
    init = stencil_op.StencilPlan.__init__

    def record(self, device, op, dst, src, aux, acc_origin, zsize, bx, *rest):
        boxes.append((dst.ptr == src.ptr, [tuple(map(tuple, b)) for b in bx]))
        init(self, device, op, dst, src, aux, acc_origin, zsize, bx, *rest)

    monkeypatch.setattr(stencil_op.StencilPlan, "__init__", record)
    dd, (hu, hf) = domain(2, low_side_radius(), [np.float64, np.float64])
    try:
        op = sb.StencilOp(co.relax([(0, (0, 0, 0), 4.0), (0, (-1, 0, 0), -1.0)], 1.0), np.float64)
        load(dd, hu.id, "curr", np.zeros(SIZE[::-1]))
        load(dd, hf.id, "curr", np.zeros(SIZE[::-1]))
        dd.apply(op, (hu, "curr"), hu, hf, colour=(2, 0))
        dd.apply(op, (hu, "next"), hu, hf, colour=(2, 0))
        interiors = [b for b in boxes if len(b[1]) == 1]  # each domain's interior plan, then its exterior plan
        assert len(interiors) == 4
        for k, d in enumerate(dd.domains()):
            lo, hi = d.get_compute_region()
            ilo = tuple(lo[a] + 1 for a in range(3))
            assert dd.get_interior()[k] == (ilo, tuple(hi))
            assert interiors[k] == (True, [(ilo, tuple(hi[a] - 1 for a in range(3)))])
            assert interiors[2 + k] == (False, [(ilo, tuple(hi))])
    finally:
        dd.close()


def test_sor_periodic_reference_placement(monkeypatch):
    """SB_ALLOC_ALIGN=0: allocations at the start of their blocks (rows of another 16-byte phase)."""
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    test_sor_periodic(3, np.float64)
    test_sor_periodic(4, np.float32)


WALL_BCS = {(0, 0): (bo.ODD, 0.0), (0, 1): (bo.VALUE, 0.5), (0, 2): (bo.EVEN, 0.0), (0, 3): (bo.ODD, 0.25), (0, 4): (bo.VALUE, -0.25),
            (0, 5): (bo.ODD, 0.0)}


def oracle_domain(radius, dtypes, boundary, arrays):
    od = bo.Domains(SIZE, oracle_radius(radius), dtypes, n_subdomains=1, periodic=[b == P for b in boundary])
    rl = lo_of(radius)
    for a, v in zip(od.arrays[(0, 0, 0)], arrays):
        so._view(a, rl, SIZE, (0, 0, 0))[...] = v
    return od, rl


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("boundary", [(F, F, F), (F, P, F)])
def test_sor_walls(ndom, dtype, boundary):
    """Walled on every face, or on x and z: ODD, VALUE and EVEN faces filled by exchange(), 10 sweeps."""
    dtype = np.dtype(dtype)
    terms = sor_terms(1.5, 0.5, 0.0)
    op = sb.StencilOp(terms, dtype)
    radius = sb.Radius.face_edge_corner(1, 0, 0)
    bcs = {k: v for k, v in WALL_BCS.items() if boundary[k[1] // 2] == F}
    rng = np.random.default_rng(20 + ndom)
    u, f = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    od, rl = oracle_domain(radius, [dtype, dtype], boundary, [u, f])
    ua, fa = od.arrays[(0, 0, 0)]
    origin = tuple(-v for v in rl)
    dd, (hu, hf) = domain(ndom, radius, [dtype, dtype], SIZE, boundary, bcs)
    try:
        load(dd, hu.id, "curr", u)
        load(dd, hf.id, "curr", f)
        for sweep in range(10):
            for c in range(2):
                od.exchange()
                bo.apply_boundary(od, bcs)
                co.apply_box(terms, ua, fa, [], ua, rl, SIZE, origin, 2, c)
                dd.apply(op, (hu, "curr"), hu, hf, colour=(2, c))
                assert same(gather(dd, hu.id), so._view(ua, rl, SIZE, (0, 0, 0)).copy()), (sweep, c)
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 3, 8])
def test_eight_colour_box27(ndom, dtype):
    """One 8-colour sweep of a 27-point relaxation (radius 1 on faces, edges and corners), then a second."""
    dtype = np.dtype(dtype)
    rng = np.random.default_rng(5)
    A = [(0, (x, y, z), float(rng.uniform(-1, 0))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]
    terms = co.relax(A + [(0, (0, 0, 0), 30.0)], 1.2)
    op = sb.StencilOp(terms, dtype)
    u0, f = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    dd, (hu, hf) = domain(ndom, sb.Radius.face_edge_corner(1, 1, 1), [dtype, dtype])
    try:
        load(dd, hu.id, "curr", u0)
        load(dd, hf.id, "curr", f)
        want = u0
        for _ in range(2):
            for c in range(8):
                dd.apply(op, (hu, "curr"), hu, hf, colour=(8, c))
                want = co.apply_periodic(terms, want, f, [], want, 8, c)
                assert same(gather(dd, hu.id), want), c
    finally:
        dd.close()


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4])
def test_damped_div_grad_walls(ndom, dtype):
    """u <- u + theta (div(kappa grad u) - f), red then black, in place; kappa in three quantities with EVEN faces, u with
    VALUE faces, walls on x and z."""
    dtype = np.dtype(dtype)
    theta = 0.02
    import vstencil_oracle as vo

    terms = [(0, (0, 0, 0), 1.0)] + [(s, o, theta * w, k, c) for s, o, w, k, c in vo.div_grad((0.9, 1.0, 1.1))] + [(1, (0, 0, 0), -theta)]
    op = sb.StencilOp(terms, dtype)
    boundary = (F, P, F)
    radius = sb.Radius.face_edge_corner(1, 0, 0)
    bcs = {(0, 0): (bo.VALUE, 1.0), (0, 1): (bo.VALUE, -0.5), (0, 4): (bo.VALUE, 0.25), (0, 5): (bo.VALUE, 0.0)}
    for q in (2, 3, 4):
        for fc in (0, 1, 4, 5):
            bcs[(q, fc)] = (bo.EVEN, 0.0)
    rng = np.random.default_rng(40 + ndom)
    u, f = rng.uniform(-1, 1, SIZE[::-1]).astype(dtype), rng.uniform(-1, 1, SIZE[::-1]).astype(dtype)
    ks = [rng.uniform(0.2, 2.0, SIZE[::-1]).astype(dtype) for _ in range(3)]
    od, rl = oracle_domain(radius, [dtype] * 5, boundary, [u, f] + ks)
    arrs = od.arrays[(0, 0, 0)]
    origin = tuple(-v for v in rl)
    dd, hs = domain(ndom, radius, [dtype] * 5, SIZE, boundary, bcs)
    try:
        load(dd, hs[0].id, "curr", u)
        load(dd, hs[1].id, "curr", f)
        for q, k in zip(hs[2:], ks):
            load(dd, q.id, "curr", k)
        for sweep in range(5):
            for c in range(2):
                od.exchange()
                bo.apply_boundary(od, bcs)
                co.apply_box(terms, arrs[0], arrs[1], arrs[2:], arrs[0], rl, SIZE, origin, 2, c)
                dd.apply(op, (hs[0], "curr"), hs[0], hs[1], coefs=hs[2:], colour=(2, c))
                assert same(gather(dd, hs[0].id), so._view(arrs[0], rl, SIZE, (0, 0, 0)).copy()), (sweep, c)
    finally:
        dd.close()


def test_helmholtz_contraction_two_subdomains():
    """Periodic FP64 -lap u + sigma u = f, even sizes, sigma h^2 = 0.06: red-black Gauss-Seidel contracts the update by
    rho_J^2 per sweep within 1 %, on 2 subdomains."""
    size = (8, 6, 10)
    sigma = 0.06
    rho_j = 6.0 / (6.0 + sigma)
    terms = co.relax(co.helmholtz(1.0, sigma), 1.0)
    op = sb.StencilOp(terms, np.float64)
    f = np.random.default_rng(9).uniform(-1, 1, size[::-1])
    dd, (hu, hf) = domain(2, sb.Radius.face_edge_corner(1, 0, 0), [np.float64, np.float64], size)
    try:
        load(dd, hu.id, "curr", np.zeros(size[::-1]))
        load(dd, hf.id, "curr", f)
        prev, norms = gather(dd, hu.id), []
        for _ in range(400):
            for c in range(2):
                dd.apply(op, (hu, "curr"), hu, hf, colour=(2, c))
            cur = gather(dd, hu.id)
            norms.append(float(np.linalg.norm(cur - prev)))
            prev = cur
        rate = norms[-1] / norms[-2]
        assert abs(rate / rho_j**2 - 1) < 0.01, (rate, rho_j**2)
    finally:
        dd.close()


def test_colour_errors_and_cache():
    dd, (h, f, g) = domain(2, sb.Radius.face_edge_corner(2, 0, 0), [np.float64, np.float64, np.float32])
    try:
        sor = sb.StencilOp(sor_terms(), np.float64)
        load(dd, h.id, "curr", np.zeros(SIZE[::-1]))
        load(dd, f.id, "curr", np.zeros(SIZE[::-1]))
        dd.apply(sor, (h, "curr"), h, f, colour=(2, 0))
        dd.apply(sor, (h, "curr"), h, f, colour=(2, 0))
        assert len(dd._stencil_plans) == 1
        dd.apply(sor, (h, "curr"), h, f, colour=(2, 1))
        assert len(dd._stencil_plans) == 2
        dd.apply(sor, h, h, f, colour=(2, 1))  # out of place: another plan
        assert len(dd._stencil_plans) == 3
        with pytest.raises(sb.StencilError, match="dst must not be src"):
            dd.apply(sor, (h, "curr"), h, f)
        with pytest.raises(sb.StencilError, match="dst must not be src"):
            dd.apply(sor, (h, "curr"), h, f, colour=(1, 0))
        for bad in ((3, 0), (2, 2), (8, -1), (0, 0)):
            with pytest.raises(sb.StencilError, match="colour"):
                dd.apply(sor, (h, "curr"), h, f, colour=bad)
        with pytest.raises(sb.StencilError, match="own colour under 2"):
            dd.apply(sb.StencilOp.laplacian(4, (1, 1, 1), np.float64), (h, "curr"), h, colour=(2, 0))
        with pytest.raises(sb.StencilError, match="must not be dst"):
            dd.apply(sb.StencilOp([(0, (1, 0, 0), 1.0, 0, (0, 0, 0))], np.float64), (h, "curr"), h, coefs=[h], colour=(2, 0))
    finally:
        dd.close()
