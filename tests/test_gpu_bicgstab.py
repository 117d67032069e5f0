"""GPU tests of multigrid-preconditioned BiCGStab on a DistributedDomain (DESIGN.md section 2.14): BiCGStab.solve() bit
for bit against tests/bicgstab_oracle.py on every partition of test_gpu_krylov.PARTS, x after each of 3 iterations and
the history (convection-diffusion on ODD(0) walls in FP64 and FP32, on ODD(c) walls, EVEN walls with a sigma field,
periodic with sigma, jump kappa with convection in FP64 and smooth kappa with convection in FP32); Multigrid.cycle on
another pair against a Multigrid built on that pair; a solve after dd.swap(); the jump problem with convection at 64^3
and 128^3 reaching 1e-8 within 12 iterations; update_coefficients() against a freshly built solver; the constructor's
errors; and subdomains on two GPUs where the machine has them."""
import math

import numpy as np
import pytest
import torch

import bicgstab_oracle as bo
import krylov_oracle as ko
import mg_oracle as mo
import stencil_b200 as sb
import vmg_oracle as vm
from test_gpu_krylov import EVEN, KVALUE, ODD0, ODDC, PARTS, P, F, fine_size, poisson, sb_bc
from test_gpu_stencil_domain import gather, load, same

pytestmark = pytest.mark.gpu

B = (4.0, 2.4, 1.2)  # the convection velocity


def conv(h, b=B):
    """Central differences of b . grad u on spacing h."""
    t = []
    for a in range(3):
        e = [0, 0, 0]
        e[a] = 1
        t.append((0, tuple(e), b[a] / (2 * h)))
        t.append((0, tuple(-v for v in e), -b[a] / (2 * h)))
    return t


CASES = {  # name: (dtype, periodic, x walls, coefficient walls, kappa (None: constant coefficients), sigma)
    "cd-odd0-f64": (np.float64, False, ODD0, None, None, 0.0),
    "cd-odd0-f32": (np.float32, False, ODD0, None, None, 0.0),
    "cd-oddc-f64": (np.float64, False, ODDC, None, None, 0.0),
    "even-sigma-f64": (np.float64, False, EVEN, EVEN, "smooth", "field"),
    "periodic-sigma-f64": (np.float64, True, {}, None, None, 10.0),
    "jump-conv-f64": (np.float64, False, ODD0, KVALUE, "jump", None),
    "smooth-conv-f32": (np.float32, False, ODD0, KVALUE, "smooth", None),
}


class Setup:
    """A domain of the nine vectors (phat and shat with the homogeneous walls) and the coefficient fields, a BiCGStab on
    it and the numpy solver of the same problem."""

    def __init__(self, size, gpus, case, levels=4, seed=7, n_h=32):
        dtype, periodic, walls, cw, kappa, sigma = CASES[case]
        self.dtype = dtype = np.dtype(dtype)
        self.size, self.periodic, self.walls = size, periodic, walls
        self.cw = {} if periodic or cw is None else cw
        h = 1.0 / n_h
        ncoef = 0 if kappa is None else 4 if sigma == "field" else 3
        self.kinds = ("x", "y", "z", "cell")[:ncoef]
        if kappa is None:
            A_at = lambda l: poisson(h * 2**l, sigma) + conv(h * 2**l)  # noqa: E731
        else:
            A_at = lambda l: vm.helmholtz_div_grad(h * 2**l, sigma_field=sigma == "field") + conv(h * 2**l)  # noqa: E731
        self.A_at = A_at
        dd = self.dd = sb.DistributedDomain(*size)
        dd.set_gpus(list(gpus))
        dd.set_radius(sb.Radius.constant(1))
        self.vecs = {n: dd.add_data(dtype, n) for n in sb.BiCGStab.NAMES}
        self.x, self.f = self.vecs["x"], self.vecs["f"]
        self.ks = [dd.add_data(dtype, n) for n in ("kx", "ky", "kz", "sigma")[:ncoef]]
        dd.set_boundary(*((P,) * 3 if periodic else (F,) * 3))
        if not periodic:
            hom = ko.homogeneous(walls)
            for fc in range(6):
                dd.set_boundary_condition(self.x, sb.FACES[fc], sb_bc(walls[fc]))
                for v in (self.vecs["phat"], self.vecs["shat"]):
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
        self.op_at = lambda l: sb.StencilOp(A_at(l), dtype)  # noqa: E731
        self.bi = sb.BiCGStab(dd, *(self.vecs[n] for n in sb.BiCGStab.NAMES), self.op_at, coefs=self.ks or None, coef_kinds=self.kinds or None,
                              levels=levels)
        self.levels = levels

    def reset(self):
        load(self.dd, self.x.id, "curr", self.x0)

    def hierarchy(self):
        hom = ko.homogeneous(self.walls)
        per = (self.periodic,) * 3
        m = self.bi.mg.colours
        if self.kp:
            lv = vm.hierarchy(self.size, self.levels, self.A_at, self.dtype, per, hom, [dict(self.cw) for _ in self.kp], m=m)
            for a, b in zip(lv[0].k, self.kp):
                a[...] = b
            vm.update_coefficients(lv, self.kinds)
        else:
            lv = mo.hierarchy(self.size, self.levels, self.A_at, self.dtype, per, hom, m=m)
        return lv

    def oracle(self):
        s = bo.BiCGStab(self.hierarchy(), self.walls)
        s.I(s.f)[...] = self.fh
        s.I(s.x)[...] = self.x0
        return s

    def close(self):
        self.bi.close()
        self.dd.close()


def run_bits(setup, iters=3):
    """x after 1 .. iters iterations (each a solve from the same first guess) and the history, against the oracle."""
    ref = setup.oracle()
    hist_ref = [math.sqrt(ref.start())]
    xs = []
    for k in range(iters):
        assert ref.iterate(k, 0.0, hist_ref)
        xs.append(ref.I(ref.x).copy())
    for k in range(1, iters + 1):
        setup.reset()
        hist = setup.bi.solve(0.0, k)
        assert setup.bi.breakdown is None
        assert hist == hist_ref[: k + 1], (k, hist, hist_ref)
        assert same(gather(setup.dd, setup.x.id), xs[k - 1]), k
    return hist_ref


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("case", sorted(CASES))
def test_bicgstab_bits(ndom, case):
    s = Setup(fine_size(ndom), [0] * ndom, case)
    try:
        assert len(s.bi.mg.levels) == 4 and s.bi.mg.colours == 2
        run_bits(s)
    finally:
        s.close()


@pytest.mark.parametrize("ndom", [1, 4])
@pytest.mark.parametrize("case", ["jump-conv-f64", "cd-odd0-f32"])
def test_cycle_on_another_pair(ndom, case):
    """Multigrid.cycle(u=shat, f=r) on the solver's preconditioner gives the bits of a Multigrid built on (shat, r)."""
    s = Setup(fine_size(ndom), [0] * ndom, case)
    mg2 = None
    try:
        V = s.vecs
        rng = np.random.default_rng(5)
        rh = rng.uniform(-1, 1, s.size[::-1]).astype(s.dtype)
        load(s.dd, V["r"].id, "curr", rh)
        load(s.dd, V["phat"].id, "curr", np.zeros_like(rh))
        load(s.dd, V["p"].id, "curr", rng.uniform(-1, 1, s.size[::-1]).astype(s.dtype))
        load(s.dd, V["shat"].id, "curr", np.zeros_like(rh))
        s.bi.mg.cycle(u=V["shat"], f=V["r"])
        got = gather(s.dd, V["shat"].id)
        assert not same(got, np.zeros_like(got))
        load(s.dd, V["shat"].id, "curr", np.zeros_like(rh))
        mg2 = sb.Multigrid(s.dd, V["shat"], V["r"], V["t"], s.op_at, coefs=s.ks or None, coef_kinds=s.kinds or None, levels=4)
        mg2.cycle()
        assert same(gather(s.dd, V["shat"].id), got)
        assert same(gather(s.dd, V["phat"].id), np.zeros_like(rh))  # the constructor pair is untouched
        with pytest.raises(sb.StencilError, match="give both u and f"):
            s.bi.mg.cycle(u=V["shat"])
        with pytest.raises(sb.StencilError, match="two different quantities"):
            s.bi.mg.cycle(u=V["shat"], f=V["shat"])
        if not s.periodic:
            with pytest.raises(sb.StencilError, match="u needs .* the constructor u's BC"):
                s.bi.mg.cycle(u=V["v"], f=V["r"])  # v carries no BC
        if s.ks:
            with pytest.raises(sb.StencilError, match="must not be coefficient fields"):
                s.bi.mg.cycle(u=V["shat"], f=s.ks[0])
    finally:
        if mg2 is not None:
            mg2.close()
        s.close()


@pytest.mark.parametrize("ndom", [1, 4])
@pytest.mark.parametrize("case", ["cd-oddc-f64", "cd-odd0-f32"])
def test_swap_after_construction(ndom, case):
    s = Setup(fine_size(ndom), [0] * ndom, case)
    try:
        s.bi.solve(0.0, 2)
        s.dd.swap()
        load(s.dd, s.f.id, "curr", s.fh)
        run_bits(s)
    finally:
        s.close()


@pytest.mark.parametrize("n", [64, 128])
def test_jump_convection_reaches_1e8(n):
    """The 10^3 jump with convection on ODD(0) walls, full hierarchy: 1e-8 of ||f|| within 12 iterations."""
    s = Setup((n, n, n), [0], "jump-conv-f64", levels=None, n_h=n)
    try:
        load(s.dd, s.x.id, "curr", np.zeros((n, n, n)))
        hist = s.bi.solve(1e-8, 12)
        assert s.bi.breakdown is None
        assert hist[-1] <= 1e-8 * math.sqrt(ko.dot(s.fh, s.fh)) and len(hist) - 1 <= 12, [v / hist[0] for v in hist]
        assert s.bi.residual_norm() <= 1e-7 * hist[0]
    finally:
        s.close()


def test_update_coefficients_equals_fresh_solver():
    s = Setup((32, 32, 32), [0] * 2, "smooth-conv-f32")
    t = None
    try:
        s.bi.solve(0.0, 1)
        for q, a in zip(s.ks, s.kp):
            load(s.dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1] * 2.5 + 0.5))
        s.bi.update_coefficients()
        s.reset()
        hist = s.bi.solve(0.0, 3)
        t = Setup((32, 32, 32), [0] * 2, "smooth-conv-f32")
        for q, a in zip(t.ks, t.kp):
            load(t.dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1] * 2.5 + 0.5))
        t.bi.update_coefficients()
        assert t.bi.solve(0.0, 3) == hist
        assert same(gather(s.dd, s.x.id), gather(t.dd, t.x.id))
    finally:
        s.close()
        if t is not None:
            t.close()


def test_constructor_errors():
    s = Setup((32, 32, 32), [0], "cd-oddc-f64")
    try:
        dd, V = s.dd, s.vecs
        args = [V[n] for n in sb.BiCGStab.NAMES]
        with pytest.raises(sb.StencilError, match="must be 9 different quantities"):
            sb.BiCGStab(dd, *args[:8], V["p"], s.op_at)
        with pytest.raises(sb.StencilError, match=r"phat needs BC\(ODD, 0.0\) on face \(1, 0, 0\)"):
            sb.BiCGStab(dd, V["phat"], *args[1:6], V["x"], *args[7:], s.op_at)  # x and phat swapped: phat carries ODD(c)
        with pytest.raises(sb.StencilError, match="op_at\\(0\\) must be a StencilOp in float64"):
            sb.BiCGStab(dd, *args, lambda l: sb.StencilOp(s.A_at(l), np.float32))
        with pytest.raises(sb.StencilError, match="reads 3 coefficient fields, but 0 were given"):
            sb.BiCGStab(dd, *args, lambda l: sb.StencilOp(vm.helmholtz_div_grad(1 / 32), np.float64))
    finally:
        s.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpus():
    s = Setup((32, 32, 32), [0, 1], "jump-conv-f64")
    try:
        run_bits(s)
    finally:
        s.close()
