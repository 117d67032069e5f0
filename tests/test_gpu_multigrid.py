"""GPU tests of DistributedDomain.restrict_to(op=...) and stencil_b200.Multigrid: the fused residual-restriction on 1, 2,
3, 4 and 8 subdomains, periodic and walled, with and without exchange, under SB_ALLOC_ALIGN=0 and 1, bit for bit
against tests/mg_oracle.py; Multigrid.cycle() bit for bit against the numpy cycle after every cycle on every partition
(FP64 and FP32 ODD(0) Poisson, FP64 inhomogeneous ODD(c), EVEN walls with sigma > 0, periodic Helmholtz, a 27-point
op under 8 colours); the queued cycle against the same sequence of public synchronising calls; the factor per cycle
on 64^3 .. 256^3 FP64 ODD(0) Poisson; solve() reaching its rtol; the constructor's errors; and subdomains on two GPUs
where the machine has them."""
import numpy as np
import pytest
import torch

import colour_oracle as co
import mg_oracle as mo
import stencil_b200 as sb
import transfer_oracle as to
from test_gpu_stencil_domain import gather, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
PARTS = [1, 2, 3, 4, 8]
ODDC = {0: ("odd", 0.0), 1: ("odd", 0.25), 2: ("odd", -0.5), 3: ("odd", 1.0), 4: ("odd", 0.125), 5: ("odd", -1.0)}
ODD0 = {f: ("odd", 0.0) for f in range(6)}
EVEN = {f: ("even", 0.0) for f in range(6)}


def fine_size(ndom):
    return (96, 32, 32) if ndom == 3 else (32, 32, 32)


def sb_bc(w):
    return sb.BC.ODD(w[1]) if w[0] == "odd" else sb.BC.EVEN()


def domain(size, gpus, dtype, names, periodic=True, walls=None, radius=1):
    dd = sb.DistributedDomain(*size)
    dd.set_gpus(list(gpus))
    dd.set_radius(sb.Radius.constant(radius))
    hs = [dd.add_data(dtype, n) for n in names]
    dd.set_boundary(*((P,) * 3 if periodic else (F,) * 3))
    for fc, w in (walls or {}).items():
        dd.set_boundary_condition(hs[0], sb.FACES[fc], sb_bc(w))
    dd.realize()
    return dd, hs


def padded(a, periodic, walls):
    out = np.zeros(tuple(n + 2 for n in a.shape), a.dtype)
    out[1:-1, 1:-1, 1:-1] = a
    mo.fill_ghosts(out, (periodic,) * 3, walls or {})
    return out


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("periodic", [True, False])
@pytest.mark.parametrize("exchange", [True, False])
@pytest.mark.parametrize("align", ["1", "0"])
def test_restrict_op(ndom, dtype, periodic, exchange, align, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    dtype = np.dtype(dtype)
    size = fine_size(ndom)
    csize = tuple(n // 2 for n in size)
    walls = None if periodic else ODDC
    fd, (u, f) = domain(size, [0] * ndom, dtype, ["u", "f"], periodic, walls)
    cd, (w,) = domain(csize, [0] * ndom, dtype, ["w"], periodic)
    try:
        A = co.helmholtz(1.0 / size[0], 0.5)
        res = sb.StencilOp(to.residual_terms(A), dtype)
        rng = np.random.default_rng(ndom)
        uh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        fh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        load(fd, u.id, "curr", uh)
        load(fd, f.id, "curr", fh)
        if not exchange:
            fd.exchange()
        fd.restrict_to(cd, (w, "curr"), u, op=res, aux=(f, "curr"), exchange=exchange)
        want = np.empty(csize[::-1], dtype)
        fp = np.zeros(tuple(n + 2 for n in fh.shape), dtype)
        fp[1:-1, 1:-1, 1:-1] = fh
        mo.restrict_op_box(want, (0, 0, 0), to.residual_terms(A), padded(uh, periodic, walls), fp, (-1, -1, -1), (0, 0, 0), csize)
        assert same(gather(cd, w.id), want)
        # no aux term: the plain op into next
        neg = sb.StencilOp([(0, t[1], -t[2]) for t in A], dtype)
        fd.restrict_to(cd, w, u, op=neg)
        mo.restrict_op_box(want, (0, 0, 0), [(0, t[1], -t[2]) for t in A], padded(uh, periodic, walls), None, (-1, -1, -1), (0, 0, 0), csize)
        assert same(gather(cd, w.id, "next"), want)
    finally:
        fd.close()
        cd.close()


def helmholtz_at(size, sigma):
    return lambda l: co.helmholtz(2.0 ** l / size[0], sigma)


def twenty_seven_at(size):
    def A(l):
        h2 = (2.0 ** l / size[0]) ** 2
        return [(0, (0, 0, 0), 88.0 / (26 * h2))] + [(0, (x, y, z), -(1.0 + 0.1 * (abs(x) + abs(y) + abs(z))) / (26 * h2))
                                                    for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]
    return A


CASES = {  # name: (dtype, periodic, walls, sigma, 27-point)
    "odd0-f64": (np.float64, False, ODD0, 0.0, False),
    "odd0-f32": (np.float32, False, ODD0, 0.0, False),
    "oddc-f64": (np.float64, False, ODDC, 0.0, False),
    "even-f64": (np.float64, False, EVEN, 1.0, False),
    "periodic-f64": (np.float64, True, None, 1.0, False),
    "27pt-f64": (np.float64, True, None, 1.0, True),
}


def solver(size, gpus, case, levels=4):
    dtype, periodic, walls, sigma, p27 = CASES[case]
    dtype = np.dtype(dtype)
    A_at = twenty_seven_at(size) if p27 else helmholtz_at(size, sigma)
    dd, (u, f, r) = domain(size, gpus, dtype, ["u", "f", "r"], periodic, walls)
    mg = sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp(A_at(l), dtype), levels=levels)
    ref = mo.hierarchy(size, levels, A_at, dtype, (periodic,) * 3, walls or {}, m=mg.colours)
    fh = np.random.default_rng(7).uniform(-1, 1, size[::-1]).astype(dtype)
    load(dd, f.id, "curr", fh)
    load(dd, u.id, "curr", np.zeros(size[::-1], dtype))
    ref[0].interior(ref[0].f)[...] = fh
    return dd, (u, f, r), mg, ref


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_cycle_bits(ndom, case):
    size = fine_size(ndom)
    dd, (u, f, r), mg, ref = solver(size, [0] * ndom, case)
    try:
        assert len(mg.levels) == 4 and mg.colours == (8 if CASES[case][4] else 2)
        for cyc in range(3):
            mg.cycle()
            mo.vcycle(ref)
            assert same(gather(dd, u.id), ref[0].interior(ref[0].u).copy()), cyc
    finally:
        mg.close()
        dd.close()


def test_cycle_bits_reference_placement(monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    test_cycle_bits(4, "oddc-f64")


@pytest.mark.parametrize("ndom", [2, 8])
def test_queued_equals_public_calls(ndom):
    """Two queued cycles against the same sequence of public synchronising calls on a second solver's domains."""
    size = fine_size(ndom)
    dd, (u, f, r), mg, _ = solver(size, [0] * ndom, "oddc-f64")
    dd2, (u2, f2, r2), mg2, _ = solver(size, [0] * ndom, "oddc-f64")
    try:
        lv = mg2.levels

        def smooth(L, n):
            for _ in range(n):
                for c in range(2):
                    L.dd.apply(L.gs, (L.u, "curr"), L.u, (L.f, "curr"), colour=(2, c))

        def cyc(l):
            L = lv[l]
            if l == len(lv) - 1:
                smooth(L, 30)
                return
            smooth(L, 2)
            Cl = lv[l + 1]
            L.dd.restrict_to(Cl.dd, (Cl.f, "curr"), L.u, op=L.res, aux=(L.f, "curr"))
            load(Cl.dd, Cl.u.id, "curr", np.zeros(Cl.dd.size()[::-1]))
            cyc(l + 1)
            L.dd.prolong_from(Cl.dd, (L.u, "curr"), (Cl.u, "curr"), aux=(L.u, "curr"))
            smooth(L, 2)

        for k in range(2):
            mg.cycle()
            cyc(0)
            assert same(gather(dd, u.id), gather(dd2, u2.id)), k
    finally:
        mg.close()
        mg2.close()
        dd.close()
        dd2.close()


def test_factor_per_cycle_is_h_independent():
    """V(2,2) on FP64 ODD(0) Poisson down to 4^3: after the first cycle every factor is <= 0.15, and the factors at
    64^3, 128^3 and 256^3 agree within 0.02."""
    fs = {}
    for n in (64, 128, 256):
        levels = int(np.log2(n)) - 1
        dd, (u, f, r), mg, _ = solver((n, n, n), [0], "odd0-f64", levels=levels)
        try:
            hist = [mg.residual_norm()]
            for _ in range(5):
                mg.cycle()
                hist.append(mg.residual_norm())
            fs[n] = [hist[k + 1] / hist[k] for k in range(5)]
        finally:
            mg.close()
            dd.close()
    for n, fac in fs.items():
        assert max(fac[1:]) <= 0.15, (n, fac)
    for k in range(1, 5):
        vals = [fs[n][k] for n in fs]
        assert max(vals) - min(vals) < 0.02, (k, fs)


def test_solve_reaches_rtol():
    dd, (u, f, r), mg, _ = solver((64, 64, 64), [0, 0], "oddc-f64", levels=5)
    try:
        fn = dd.reduce(f, "curr", exact=True).l2()
        hist = mg.solve(1e-8, 20)
        assert hist[-1] <= 1e-8 * fn and len(hist) <= 15, hist
        assert all(hist[k + 1] < hist[k] for k in range(len(hist) - 1)), hist
    finally:
        mg.close()
        dd.close()


def test_constructor_errors():
    A = lambda l: sb.StencilOp(co.helmholtz(1.0, 0.0), np.float64)  # noqa: E731
    dd, (u, f, r) = domain((16, 16, 16), [0], np.float64, ["u", "f", "r"], False, {0: ("odd", 0.0)})
    try:
        with pytest.raises(sb.StencilError, match="needs a boundary condition"):
            sb.Multigrid(dd, u, f, r, A)
    finally:
        dd.close()
    dd = sb.DistributedDomain(16, 16, 16)
    dd.set_gpus([0])
    dd.set_radius(1)
    u, f, r = (dd.add_data(np.float64) for _ in range(3))
    dd.set_boundary(F)
    for fc in range(6):
        dd.set_boundary_condition(u, sb.FACES[fc], sb.BC.VALUE(0.0))
    dd.realize()
    try:
        with pytest.raises(sb.StencilError, match="VALUE walls"):
            sb.Multigrid(dd, u, f, r, A)
    finally:
        dd.close()
    dd, (u, f, r, g) = domain((17, 16, 16), [0], np.float64, ["u", "f", "r", "g"])
    try:
        with pytest.raises(sb.StencilError, match="cannot be coarsened once"):
            sb.Multigrid(dd, u, f, r, A)
    finally:
        dd.close()
    dd, (u, f, r, g) = domain((16, 16, 16), [0], np.float64, ["u", "f", "r", "g"], radius=2)
    try:
        with pytest.raises(sb.StencilError, match="three different quantities"):
            sb.Multigrid(dd, u, f, u, A)
        with pytest.raises(sb.StencilError, match="must be a StencilOp in float64"):
            sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp(co.helmholtz(1.0, 0.0), np.float32))
        with pytest.raises(sb.StencilError, match="reaches 2 cells"):
            sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp([(0, (0, 0, 0), 1.0), (0, (2, 0, 0), 0.1)], np.float64))
        with pytest.raises(sb.StencilError, match="coefficient or aux terms"):
            sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp([(0, (0, 0, 0), 1.0), (1, (0, 0, 0), 0.1)], np.float64))
        with pytest.raises(sb.StencilError, match="coefficient or aux terms"):
            sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp.div_grad((1.0, 1.0, 1.0), np.float64))
        with pytest.raises(sb.StencilError, match="levels must be >= 2"):
            sb.Multigrid(dd, u, f, r, A, levels=1)
    finally:
        dd.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_cycle_bits_two_gpus():
    dd, (u, f, r), mg, ref = solver((32, 32, 32), [0, 1, 0, 1], "oddc-f64")
    try:
        for cyc in range(2):
            mg.cycle()
            mo.vcycle(ref)
            assert same(gather(dd, u.id), ref[0].interior(ref[0].u).copy()), cyc
    finally:
        mg.close()
        dd.close()
