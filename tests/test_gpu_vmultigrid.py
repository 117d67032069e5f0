"""GPU tests of multigrid for variable-coefficient operators on a DistributedDomain (DESIGN.md section 2.12): relax(),
restrict_to(op=..., coefs=...) and restrict_to(face=a) on 1, 2, 3, 4 and 8 subdomains, periodic and walled, under
SB_ALLOC_ALIGN=0 and 1, bit for bit against tests/vmg_oracle.py; Multigrid.cycle() with coefficient fields bit for bit
against the numpy cycle after each of 3 cycles on every partition (FP64 and FP32 ODD(0), ODD(c), EVEN walls with a cell
field sigma, periodic Helmholtz); the queued cycle against the same sequence of public synchronising calls;
update_coefficients() after kappa changes against a freshly built solver; the factor per cycle at 64^3 .. 256^3 and
solve() on smooth kappa; the constructor's errors; and subdomains on two GPUs where the machine has them."""
import numpy as np
import pytest
import torch

import mg_oracle as mo
import stencil_b200 as sb
import vmg_oracle as vm
from test_gpu_stencil_domain import gather, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
PARTS = [1, 2, 3, 4, 8]
ODDC = {0: ("odd", 0.0), 1: ("odd", 0.25), 2: ("odd", -0.5), 3: ("odd", 1.0), 4: ("odd", 0.125), 5: ("odd", -1.0)}
ODD0 = {f: ("odd", 0.0) for f in range(6)}
EVEN = {f: ("even", 0.0) for f in range(6)}
KVALUE = {f: ("value", 1.0 + 0.25 * f) for f in range(6)}  # kappa pinned on every wall face


def fine_size(ndom):
    return (96, 32, 32) if ndom == 3 else (32, 32, 32)


def sb_bc(w):
    return {"odd": sb.BC.ODD, "even": lambda c: sb.BC.EVEN(), "value": sb.BC.VALUE}[w[0]](w[1])


def domain(size, gpus, dtype, names, periodic, walls, coef_walls, ncoef):
    """A domain of the quantities names, then kx, ky, kz (and sigma with ncoef = 4); u (the first) gets walls, every
    coefficient coef_walls."""
    dd = sb.DistributedDomain(*size)
    dd.set_gpus(list(gpus))
    dd.set_radius(sb.Radius.constant(1))
    hs = [dd.add_data(dtype, n) for n in names]
    ks = [dd.add_data(dtype, n) for n in ("kx", "ky", "kz", "sigma")[:ncoef]]
    dd.set_boundary(*((P,) * 3 if periodic else (F,) * 3))
    if not periodic:
        for fc, w in walls.items():
            dd.set_boundary_condition(hs[0], sb.FACES[fc], sb_bc(w))
        for k in ks:
            for fc, w in coef_walls.items():
                dd.set_boundary_condition(k, sb.FACES[fc], sb_bc(w))
    dd.realize()
    return dd, hs, ks


def fields(size, dtype, kind, ncoef, seed=0):
    """Padded kappa fields (and sigma) of the unit-spaced grid size."""
    ks = vm.kappa_faces(size, 1.0 / 32, kind, dtype)
    if ncoef == 4:
        ks.append(np.random.default_rng(seed + 11).uniform(0.5, 2.0, tuple(n + 2 for n in size[::-1])).astype(dtype))
    return ks


def padded(a, periodic, walls):
    out = np.zeros(tuple(n + 2 for n in a.shape), a.dtype)
    out[1:-1, 1:-1, 1:-1] = a
    vm.fill_ghosts(out, (periodic,) * 3, walls or {})
    return out


def interior(a):
    return a[1:-1, 1:-1, 1:-1].copy()


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("periodic", [True, False])
@pytest.mark.parametrize("align", ["1", "0"])
def test_relax_and_restrictions(ndom, dtype, periodic, align, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    dtype = np.dtype(dtype)
    size = fine_size(ndom)
    csize = tuple(n // 2 for n in size)
    walls, cw = (None, {}) if periodic else (ODDC, KVALUE)
    fd, (u, f, r), ks = domain(size, [0] * ndom, dtype, ["u", "f", "r"], periodic, walls or {}, cw, 4)
    cd, (w,), _ = domain(csize, [0] * ndom, dtype, ["w"], periodic, {}, {}, 0)
    try:
        A = vm.helmholtz_div_grad(1.0 / 32, sigma_field=True)
        op = sb.StencilOp(A, dtype)
        rng = np.random.default_rng(ndom)
        uh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        fh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        kh = [interior(k) for k in fields(size, dtype, "smooth", 4, ndom)]
        load(fd, u.id, "curr", uh)
        load(fd, f.id, "curr", fh)
        for q, a in zip(ks, kh):
            load(fd, q.id, "curr", a)
        up = padded(uh, periodic, walls)
        fp = padded(fh, periodic, walls)
        kp = [padded(a, periodic, cw) for a in kh]
        # weighted Jacobi out of place into r, then a red-black sweep in place
        fd.relax(op, (r, "curr"), u, f, coefs=ks, omega=0.75)
        want = np.full(up.shape, np.nan, dtype)
        vm.diag_box(A, 0.75, up, fp, kp, want, (1, 1, 1), size, (-1, -1, -1), 1, 0)
        assert same(gather(fd, r.id), interior(want))
        for c in range(2):
            fd.relax(op, (u, "curr"), u, f, coefs=ks, colour=(2, c))
            vm.fill_ghosts(up, (periodic,) * 3, walls or {})
            vm.diag_box(A, 1.0, up, fp, kp, up, (1, 1, 1), size, (-1, -1, -1), 2, c)
            assert same(gather(fd, u.id), interior(up)), c
        # the fused residual-restriction with coefficients, with and without the overlapped exchange
        res = vm.vresidual_terms(A)
        for exchange in (True, False):
            if not exchange:
                fd.exchange()
            fd.restrict_to(cd, (w, "curr"), u, op=sb.StencilOp(res, dtype), aux=(f, "curr"), coefs=ks, exchange=exchange)
            want = np.empty(csize[::-1], dtype)
            vm.fill_ghosts(up, (periodic,) * 3, walls or {})
            vm.restrict_vop_box(want, (0, 0, 0), res, up, fp, kp, (-1, -1, -1), (0, 0, 0), csize)
            assert same(gather(cd, w.id), want), exchange
        # the face restriction of each kappa field, and the 8-cell one of sigma
        for axis in range(3):
            fd.restrict_to(cd, (w, "curr"), (ks[axis], "curr"), face=axis)
            want = np.empty(csize[::-1], dtype)
            vm.face_restrict_box(want, (0, 0, 0), kh[axis], (0, 0, 0), axis, (0, 0, 0), csize)
            assert same(gather(cd, w.id), want), axis
    finally:
        fd.close()
        cd.close()


CASES = {  # name: (dtype, periodic, u walls, coefficient walls, kappa, sigma field)
    "odd0-f64": (np.float64, False, ODD0, EVEN, "smooth", False),
    "odd0-f32": (np.float32, False, ODD0, EVEN, "smooth", False),
    "oddc-f64": (np.float64, False, ODDC, KVALUE, "smooth", False),
    "even-sigma-f64": (np.float64, False, EVEN, EVEN, "smooth", True),
    "jump-f64": (np.float64, False, ODD0, EVEN, "jump", False),
    "periodic-f64": (np.float64, True, None, {}, "smooth", True),
}


def solver(size, gpus, case, levels=4, seed=7):
    dtype, periodic, walls, cw, kind, sig = CASES[case]
    dtype = np.dtype(dtype)
    ncoef = 4 if sig else 3
    kinds = ("x", "y", "z", "cell")[:ncoef]
    h = 1.0 / 32

    def A_at(l):
        return vm.helmholtz_div_grad(h * 2 ** l, sigma_field=sig)

    dd, (u, f, r), ks = domain(size, gpus, dtype, ["u", "f", "r"], periodic, walls or {}, cw, ncoef)
    kp = fields(size, dtype, kind, ncoef)
    for q, a in zip(ks, kp):
        load(dd, q.id, "curr", interior(a))
    fh = np.random.default_rng(seed).uniform(-1, 1, size[::-1]).astype(dtype)
    load(dd, f.id, "curr", fh)
    load(dd, u.id, "curr", np.zeros(size[::-1], dtype))
    mg = sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp(A_at(l), dtype), levels=levels, coefs=ks, coef_kinds=kinds)
    ref = vm.hierarchy(size, levels, A_at, dtype, (periodic,) * 3, walls or {}, [dict(cw) for _ in range(ncoef)], m=mg.colours)
    ref[0].interior(ref[0].f)[...] = fh
    for a, b in zip(ref[0].k, kp):
        a[...] = b
    vm.update_coefficients(ref, kinds)
    return dd, (u, f, r), ks, mg, ref


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_cycle_bits(ndom, case):
    size = fine_size(ndom)
    dd, (u, f, r), ks, mg, ref = solver(size, [0] * ndom, case)
    try:
        assert len(mg.levels) == 4 and mg.colours == 2
        for cyc in range(3):
            mg.cycle()
            vm.vcycle(ref)
            assert same(gather(dd, u.id), ref[0].interior(ref[0].u).copy()), cyc
        assert mg.residual_norm() == pytest.approx(ref[0].residual_norm(), rel=1e-12 if CASES[case][0] is np.float64 else 1e-5)
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
    dd, (u, f, r), ks, mg, _ = solver(size, [0] * ndom, "even-sigma-f64")
    dd2, (u2, f2, r2), ks2, mg2, _ = solver(size, [0] * ndom, "even-sigma-f64")
    try:
        lv = mg2.levels

        def smooth(L, n):
            for _ in range(n):
                for c in range(2):
                    L.dd.relax(L.A, (L.u, "curr"), L.u, L.f, coefs=L.coefs, colour=(2, c))

        def cyc(l):
            L = lv[l]
            if l == len(lv) - 1:
                smooth(L, 30)
                return
            smooth(L, 2)
            Cl = lv[l + 1]
            L.dd.restrict_to(Cl.dd, (Cl.f, "curr"), L.u, op=L.res, aux=(L.f, "curr"), coefs=L.coefs)
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


def test_update_coefficients_equals_fresh_solver():
    """kappa changes after a cycle: update_coefficients() then a cycle gives the bits of a solver built on the new kappa
    from the same u."""
    size = (32, 32, 32)
    dd, (u, f, r), ks, mg, _ = solver(size, [0, 0], "odd0-f64")
    dd2, (u2, f2, r2), ks2, mg2, _ = solver(size, [0, 0], "odd0-f64")
    try:
        mg.cycle()
        new = [interior(k) * (1.0 + 0.5 * np.cos(np.arange(32))[None, None, :]) for k in fields(size, np.float64, "jump", 3)]
        for q, a in zip(ks, new):
            load(dd, q.id, "curr", a)
        mg.update_coefficients()
        mg2.close()
        for q, a in zip(ks2, new):
            load(dd2, q.id, "curr", a)
        load(dd2, u2.id, "curr", gather(dd, u.id))
        mg2 = sb.Multigrid(dd2, u2, f2, r2, lambda l: sb.StencilOp(vm.helmholtz_div_grad(2.0 ** l / 32), np.float64), levels=4, coefs=ks2)
        for L, L2 in zip(mg.levels[1:], mg2.levels[1:]):
            for k, k2 in zip(L.coefs, L2.coefs):
                assert same(gather(L.dd, k.id), gather(L2.dd, k2.id))
        mg.cycle()
        mg2.cycle()
        assert same(gather(dd, u.id), gather(dd2, u2.id))
    finally:
        mg.close()
        mg2.close()
        dd.close()
        dd2.close()


def test_factor_per_cycle():
    """V(2,2) on FP64 -div(kappa grad u) = f, smooth kappa, ODD(0) walls, down to 4^3: after the first cycle every factor
    is <= 0.2 at 64^3, 128^3 and 256^3 (h-independent; the numpy cycle gives 0.07 - 0.13 at 16^3 - 64^3)."""
    fs = {}
    for n in (64, 128, 256):
        levels = int(np.log2(n)) - 1
        dd, (u, f, r), ks, mg, _ = solver((n, n, n), [0], "odd0-f64", levels=levels)
        try:
            hist = [mg.residual_norm()]
            for _ in range(5):
                mg.cycle()
                hist.append(mg.residual_norm())
            fs[n] = [hist[k + 1] / hist[k] for k in range(5)]
        finally:
            mg.close()
            dd.close()
    print("factors", fs)
    for n, fac in fs.items():
        assert max(fac[1:]) <= 0.2, (n, fac)


def test_solve_reaches_rtol():
    """Smooth kappa, ODD(0) walls: 10^-8 ||f|| within 14 cycles (measured factors 0.02 - 0.13), every cycle lowering the
    residual."""
    dd, (u, f, r), ks, mg, _ = solver((64, 64, 64), [0, 0], "odd0-f64", levels=5)
    try:
        fn = dd.reduce(f, "curr", exact=True).l2()
        hist = mg.solve(1e-8, 20)
        assert hist[-1] <= 1e-8 * fn and len(hist) <= 15, hist
        assert all(hist[k + 1] < hist[k] for k in range(len(hist) - 1)), hist
    finally:
        mg.close()
        dd.close()


def test_constructor_errors():
    A = lambda l: sb.StencilOp(vm.helmholtz_div_grad(2.0 ** l / 16), np.float64)  # noqa: E731
    dd, (u, f, r), ks = domain((16, 16, 16), [0], np.float64, ["u", "f", "r"], False, ODD0, {}, 3)
    try:
        with pytest.raises(sb.StencilError, match="coefficient 0 needs a boundary condition"):
            sb.Multigrid(dd, u, f, r, A, coefs=ks)
    finally:
        dd.close()
    dd, (u, f, r), ks = domain((16, 16, 16), [0], np.float64, ["u", "f", "r"], True, {}, {}, 3)
    try:
        with pytest.raises(sb.StencilError, match="coefficient or aux terms"):
            sb.Multigrid(dd, u, f, r, A)
        with pytest.raises(sb.StencilError, match="coefficient or aux terms"):
            sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp([(0, (0, 0, 0), 1.0), (1, (0, 0, 0), 0.1)], np.float64), coefs=ks)
        with pytest.raises(sb.StencilError, match="coef_kinds"):
            sb.Multigrid(dd, u, f, r, A, coefs=ks, coef_kinds=("x", "y", "w"))
        with pytest.raises(sb.StencilError, match="coef_kinds"):
            sb.Multigrid(dd, u, f, r, A, coefs=ks[:2])
        with pytest.raises(sb.StencilError, match="reads 3 coefficient fields, but 2"):
            sb.Multigrid(dd, u, f, r, A, coefs=ks[:2], coef_kinds=("x", "y"))
        with pytest.raises(sb.StencilError, match="other than u, f and r"):
            sb.Multigrid(dd, u, f, r, A, coefs=[ks[0], ks[1], u])
        with pytest.raises(sb.StencilError, match="different quantities"):
            sb.Multigrid(dd, u, f, r, A, coefs=[ks[0], ks[1], ks[1]])
        with pytest.raises(sb.StencilError, match="no term at offset"):
            sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp([t for t in vm.helmholtz_div_grad(1.0) if any(t[1])], np.float64), coefs=ks)
    finally:
        dd.close()


def test_relax_errors():
    dd, (u, f, r), ks = domain((16, 16, 16), [0], np.float64, ["u", "f", "r"], True, {}, {}, 3)
    try:
        op = sb.StencilOp(vm.helmholtz_div_grad(1.0), np.float64)
        with pytest.raises(sb.StencilError, match="dst must not be src"):
            dd.relax(op, (u, "curr"), u, f, coefs=ks)
        with pytest.raises(sb.StencilError, match="A has a term on aux"):
            dd.relax(sb.StencilOp([(0, (0, 0, 0), 1.0), (1, (0, 0, 0), 1.0)], np.float64), r, u, f)
        with pytest.raises(sb.StencilError, match="no term at offset"):
            dd.relax(sb.StencilOp([(0, (1, 0, 0), 1.0)], np.float64), r, u, f)
        with pytest.raises(sb.StencilError, match="omega"):
            dd.relax(op, r, u, f, coefs=ks, omega=float("nan"))
        with pytest.raises(sb.StencilError, match="face"):
            dd.restrict_to(dd, r, u, face=3)
    finally:
        dd.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_cycle_bits_two_gpus():
    dd, (u, f, r), ks, mg, ref = solver((32, 32, 32), [0, 1, 0, 1], "oddc-f64")
    try:
        for cyc in range(2):
            mg.cycle()
            vm.vcycle(ref)
            assert same(gather(dd, u.id), ref[0].interior(ref[0].u).copy()), cyc
    finally:
        mg.close()
        dd.close()
