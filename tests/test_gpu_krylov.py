"""GPU tests of multigrid-preconditioned CG on a DistributedDomain (DESIGN.md section 2.13): dd.dot on 1, 2, 3, 4 and 8
subdomains under SB_ALLOC_ALIGN=0 and 1 (the same bits on every partition, equal to math.fsum); PCG.solve() bit for bit
against tests/krylov_oracle.py on every partition, x after each of 3 iterations and the sqrt(rho) history, FP64 and
FP32 (ODD(0) Poisson, inhomogeneous ODD(c) Poisson, EVEN walls with a sigma field, periodic Helmholtz, smooth and jump
kappa with VALUE kappa walls, and no preconditioner); a solve after dd.swap(); the jump problem at 64^3 and 128^3
reaching 1e-8 within the CPU bound's 30 iterations; update_coefficients() against a freshly built solver; the
constructor's errors and the breakdown of an indefinite op; and subdomains on two GPUs where the machine has them."""
import math

import numpy as np
import pytest
import torch

import krylov_oracle as ko
import mg_oracle as mo
import stencil_b200 as sb
import vmg_oracle as vm
from test_gpu_stencil_domain import gather, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
PARTS = [1, 2, 3, 4, 8]
ODD0 = {f: ("odd", 0.0) for f in range(6)}
ODDC = {0: ("odd", 0.0), 1: ("odd", 0.25), 2: ("odd", -0.5), 3: ("odd", 1.0), 4: ("odd", 0.125), 5: ("odd", -1.0)}
EVEN = {f: ("even", 0.0) for f in range(6)}
KVALUE = {f: ("value", 1.0 + 0.25 * f) for f in range(6)}


def fine_size(ndom):
    return (96, 32, 32) if ndom == 3 else (32, 32, 32)


def sb_bc(w):
    return {"odd": sb.BC.ODD, "even": lambda c: sb.BC.EVEN(), "value": sb.BC.VALUE}[w[0]](w[1])


def poisson(h, sigma=0.0):
    """-lap u (+ sigma u): the 7-point stencil with one centre term."""
    t = [(0, (0, 0, 0), 6.0 / h**2 + sigma)]
    for a in range(3):
        for s in (-1, 1):
            o = [0, 0, 0]
            o[a] = s
            t.append((0, tuple(o), -1.0 / h**2))
    return t


CASES = {  # name: (dtype, periodic, x walls, coefficient walls, kappa (None: constant coefficients), sigma, precond)
    "poisson-odd0-f64": (np.float64, False, ODD0, None, None, 0.0, True),
    "poisson-odd0-f32": (np.float32, False, ODD0, None, None, 0.0, True),
    "poisson-oddc-f64": (np.float64, False, ODDC, None, None, 0.0, True),
    "even-sigma-f64": (np.float64, False, EVEN, EVEN, "smooth", "field", True),
    "helmholtz-periodic-f64": (np.float64, True, {}, None, None, 10.0, True),
    "helmholtz-periodic-f32": (np.float32, True, {}, None, None, 10.0, True),
    "smooth-kvalue-f64": (np.float64, False, ODD0, KVALUE, "smooth", None, True),
    "smooth-kvalue-f32": (np.float32, False, ODD0, KVALUE, "smooth", None, True),
    "jump-kvalue-f64": (np.float64, False, ODD0, KVALUE, "jump", None, True),
    "noprec-oddc-f64": (np.float64, False, ODDC, None, None, 0.0, False),
}


class Setup:
    """A domain of x, f, r, z, p, q (p and z with the homogeneous walls) and the coefficient fields, a PCG on it and
    the numpy solver of the same problem."""

    def __init__(self, size, gpus, case, levels=4, seed=7, n_h=32, sign=1.0):
        dtype, periodic, walls, cw, kappa, sigma, precond = CASES[case]
        self.dtype = dtype = np.dtype(dtype)
        self.size, self.periodic, self.walls, self.precond = size, periodic, walls, precond
        self.cw = {} if periodic or cw is None else cw
        h = 1.0 / n_h
        ncoef = 0 if kappa is None else 4 if sigma == "field" else 3
        self.kinds = ("x", "y", "z", "cell")[:ncoef]
        if kappa is None:
            A_at = lambda l: [t[:2] + (sign * t[2],) for t in poisson(h * 2**l, sigma)]  # noqa: E731
        else:
            A_at = lambda l: [t[:2] + (sign * t[2],) + tuple(t[3:]) for t in vm.helmholtz_div_grad(h * 2**l, sigma_field=sigma == "field")]  # noqa: E731
        self.A_at = A_at
        dd = self.dd = sb.DistributedDomain(*size)
        dd.set_gpus(list(gpus))
        dd.set_radius(sb.Radius.constant(1))
        self.x, self.f, self.r, self.z, self.p, self.q = (dd.add_data(dtype, n) for n in "xfrzpq")
        self.ks = [dd.add_data(dtype, n) for n in ("kx", "ky", "kz", "sigma")[:ncoef]]
        dd.set_boundary(*((P,) * 3 if periodic else (F,) * 3))
        if not periodic:
            hom = ko.homogeneous(walls)
            for fc in range(6):
                dd.set_boundary_condition(self.x, sb.FACES[fc], sb_bc(walls[fc]))
                for v in (self.p, self.z):
                    dd.set_boundary_condition(v, sb.FACES[fc], sb_bc(hom[fc]))
                for k in self.ks:
                    dd.set_boundary_condition(k, sb.FACES[fc], sb_bc(cw[fc]))
        dd.realize()
        rng = np.random.default_rng(seed)
        self.fh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        self.x0 = rng.uniform(-0.5, 0.5, size[::-1]).astype(dtype)
        self.kp = []
        if ncoef:
            self.kp = vm.kappa_faces(size, h, kappa, dtype)
            if ncoef == 4:
                self.kp.append(np.random.default_rng(seed + 11).uniform(0.5, 2.0, tuple(n + 2 for n in size[::-1])).astype(dtype))
        for q, a in zip(self.ks, self.kp):
            load(dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1]))
        load(dd, self.f.id, "curr", self.fh)
        self.reset()
        op_at = lambda l: sb.StencilOp(A_at(l), dtype)  # noqa: E731
        self.cg = sb.PCG(dd, self.x, self.f, self.r, self.z if precond else None, self.p, self.q, op_at, precond="multigrid" if precond else None,
                         coefs=self.ks or None, coef_kinds=self.kinds or None, levels=levels)
        self.levels = levels

    def reset(self):
        load(self.dd, self.x.id, "curr", self.x0)

    def oracle(self):
        hom = ko.homogeneous(self.walls)
        per = (self.periodic,) * 3
        m = self.cg.mg.colours if self.cg.mg is not None else 2
        if self.kp:
            cw = [dict(self.cw) for _ in self.kp]
            lv = vm.hierarchy(self.size, self.levels, self.A_at, self.dtype, per, hom, cw, m=m)
            for a, b in zip(lv[0].k, self.kp):
                a[...] = b
            vm.update_coefficients(lv, self.kinds)
        else:
            lv = mo.hierarchy(self.size, self.levels, self.A_at, self.dtype, per, hom, m=m)
        s = ko.PCG(lv, self.walls, precond=self.precond)
        s.I(s.f)[...] = self.fh
        s.I(s.x)[...] = self.x0
        return s

    def close(self):
        self.cg.close()
        self.dd.close()


def run_bits(setup, iters=3):
    """x after 1 .. iters iterations (each a solve from the same first guess) and the history, against the oracle."""
    ref = setup.oracle()
    hist_ref = [math.sqrt(ref.start())]
    xs = []
    for k in range(iters):
        hist_ref.append(math.sqrt(ref.iterate(k)))
        xs.append(ref.I(ref.x).copy())
    for k in range(1, iters + 1):
        setup.reset()
        hist = setup.cg.solve(0.0, k)
        assert setup.cg.breakdown is None
        assert hist == hist_ref[: k + 1], (k, hist, hist_ref)
        assert same(gather(setup.dd, setup.x.id), xs[k - 1]), k
    return hist_ref


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_pcg_bits(ndom, case):
    s = Setup(fine_size(ndom), [0] * ndom, case)
    try:
        assert s.cg.mg is None or (len(s.cg.mg.levels) == 4 and s.cg.mg.colours == 2)
        run_bits(s)
    finally:
        s.close()


@pytest.mark.parametrize("ndom", [1, 4])
@pytest.mark.parametrize("case", ["poisson-oddc-f64", "poisson-odd0-f32"])
def test_swap_after_construction(ndom, case):
    """dd.swap() once after the solver has built and used its passes: with x and f loaded into the new curr buffers,
    every pass follows them, and the solve gives the oracle's bits."""
    s = Setup(fine_size(ndom), [0] * ndom, case)
    try:
        s.cg.solve(0.0, 2)
        s.dd.swap()
        load(s.dd, s.f.id, "curr", s.fh)
        run_bits(s)
    finally:
        s.close()


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("align", ["1", "0"])
def test_dot_every_partition(ndom, dtype, align, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    dtype = np.dtype(dtype)
    size = fine_size(ndom)
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([0] * ndom)
    dd.set_radius(sb.Radius.constant(1))
    a, b = dd.add_data(dtype, "a"), dd.add_data(dtype, "b")
    dd.realize()
    try:
        rng = np.random.default_rng(1)
        ah = (rng.uniform(-1, 1, size[::-1]) * 10.0 ** rng.integers(-8, 8, size[::-1])).astype(dtype)
        bh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        load(dd, a.id, "curr", ah)
        load(dd, b.id, "curr", bh)
        got = dd.dot(a, b)
        assert got == ko.dot(ah, bh)
        assert dd.dot(a, a) == ko.dot(ah, ah) == dd.reduce(a, exact=True).sumsq
        assert dd.dot(b, a) == got
    finally:
        dd.close()


@pytest.mark.parametrize("n", [64, 128])
def test_jump_reaches_1e8(n):
    """The 10^3 jump on ODD(0) walls, full hierarchy: 1e-8 of ||f|| within 30 iterations (the CPU bound)."""
    s = Setup((n, n, n), [0], "jump-kvalue-f64", levels=None, n_h=n)
    try:
        load(s.dd, s.x.id, "curr", np.zeros((n, n, n)))
        hist = s.cg.solve(1e-8, 30)
        assert hist[-1] <= 1e-8 * hist[0] and len(hist) - 1 <= 30, [v / hist[0] for v in hist]
        assert s.cg.residual_norm() <= 1e-7 * hist[0]
    finally:
        s.close()


def test_update_coefficients_equals_fresh_solver():
    s = Setup((32, 32, 32), [0] * 2, "smooth-kvalue-f64")
    t = None
    try:
        s.cg.solve(0.0, 1)
        for q, a in zip(s.ks, s.kp):
            load(s.dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1] * 2.5 + 0.5))
        s.cg.update_coefficients()
        s.reset()
        hist = s.cg.solve(0.0, 3)
        t = Setup((32, 32, 32), [0] * 2, "smooth-kvalue-f64")
        for q, a in zip(t.ks, t.kp):
            load(t.dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1] * 2.5 + 0.5))
        t.cg.update_coefficients()
        assert t.cg.solve(0.0, 3) == hist
        assert same(gather(s.dd, s.x.id), gather(t.dd, t.x.id))
    finally:
        s.close()
        if t is not None:
            t.close()


def test_constructor_errors_and_breakdown():
    s = Setup((32, 32, 32), [0], "poisson-oddc-f64")
    try:
        dd, A = s.dd, lambda l: sb.StencilOp(s.A_at(l), np.float64)
        with pytest.raises(sb.StencilError, match="must be 6 different quantities"):
            sb.PCG(dd, s.x, s.f, s.r, s.p, s.p, s.q, A)
        with pytest.raises(sb.StencilError, match=r"p needs BC\(ODD, 0.0\) on face \(1, 0, 0\)"):
            sb.PCG(dd, s.p, s.f, s.r, s.z, s.x, s.q, A)  # the roles of x and p swapped: p carries ODD(c)
        with pytest.raises(sb.StencilError, match="op_at\\(0\\) must be a StencilOp in float64"):
            sb.PCG(dd, s.x, s.f, s.r, s.z, s.p, s.q, lambda l: sb.StencilOp(s.A_at(l), np.float32))
        with pytest.raises(sb.StencilError, match="reads 3 coefficient fields, but 0 were given"):
            sb.PCG(dd, s.x, s.f, s.r, s.z, s.p, s.q, lambda l: sb.StencilOp(vm.helmholtz_div_grad(1 / 32), np.float64))
    finally:
        s.close()
    for case in ("poisson-odd0-f64", "noprec-oddc-f64"):
        s = Setup((32, 32, 32), [0] * 2, case, sign=-1.0)
        try:
            hist = s.cg.solve(1e-8, 10)
            assert s.cg.breakdown == 0 and len(hist) == 1, (case, hist)
        finally:
            s.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus():
    s = Setup((32, 32, 32), [0, 1], "smooth-kvalue-f64")
    try:
        run_bits(s)
    finally:
        s.close()
