"""GPU tests of the C++ solvers against the numpy oracles (DESIGN.md section 2.14): bin/test_solver_parity
(tests/cpp/test_solver_parity.cu) runs stencil::Multigrid<T>, stencil::PCG<T> and stencil::BiCGStab<T> on case
directories this module writes from the case tables of test_gpu_multigrid.py, test_gpu_vmultigrid.py, test_gpu_krylov.py
and test_gpu_bicgstab.py (ops as hex-float term lists, inputs as raw arrays), and every result must be the bits of
tests/mg_oracle.py, vmg_oracle.py, krylov_oracle.py and bicgstab_oracle.py: u after each of 3 cycles, update_coefficients()
after kappa changes, a cycle on a second pair, num_levels() and colours(); x and the history (as doubles) after solves
of 1, 2 and 3 iterations, breakdown(), and a solve after dd.swap(); PCG and BiCGStab on -A; and, on a walled case with
ODD(c) walls on u and VALUE walls on kappa, single passes of apply, relax, the coefficient residual restriction, the face
restriction and the prolongation.  Every case runs on 1, 2, 3, 4 and 8 subdomains of one process; one case per solver
under bin/sb_mpirun with 2 and 4 ranks (ranks share the GPU on a one-GPU machine); one under SB_ALLOC_ALIGN=0.  The
oracles do not depend on the partition, so each is computed once per grid size."""
import math
import os
import subprocess

import numpy as np
import pytest

import bicgstab_oracle as bo
import krylov_oracle as ko
import mg_oracle as mo
import transfer_oracle as to
import vmg_oracle as vm
import vstencil_oracle as vo
from test_gpu_bicgstab import CASES as BICG_CASES, conv
from test_gpu_colour_multirank import BIN, mpirun_env
from test_gpu_krylov import CASES as PCG_CASES, poisson
from test_gpu_multigrid import CASES as MG_CASES, fine_size, helmholtz_at, twenty_seven_at
from test_gpu_stencil_domain import same
from test_gpu_vmultigrid import CASES as VMG_CASES, KVALUE, ODDC, fields, padded

pytestmark = pytest.mark.gpu

PARTS = [1, 2, 3, 4, 8]
LEVELS = 4
ITERS = 3
KSCALE = 2.5  # the factor of the coefficient fields before update_coefficients()
EXE = os.path.join(BIN, "test_solver_parity")


def interior(a):
    return np.ascontiguousarray(a[1:-1, 1:-1, 1:-1])


def pad(a):
    out = np.zeros(tuple(n + 2 for n in a.shape), a.dtype)
    out[1:-1, 1:-1, 1:-1] = a
    return out


def negated(A_at):
    return lambda l: [t[:2] + (-t[2],) + tuple(t[3:]) for t in A_at(l)]


class Case:
    """One case directory: the problem for the harness, and what the oracle says it must write."""

    def __init__(self, name, solver, size, dtype, periodic, kinds=(), precond=True):
        self.name, self.solver, self.size, self.dtype, self.periodic = name, solver, tuple(size), np.dtype(dtype), periodic
        self.kinds, self.precond = tuple(kinds), precond
        self.bcs, self.ops, self.inputs, self.files = [], [], {}, {}
        self.want, self.info = {}, {}

    def walls(self, names, walls):
        for q in names:
            for fc, (kind, c) in sorted((walls or {}).items()):
                self.bcs.append((q, fc, kind, c))

    def write(self, root):
        d = os.path.join(root, self.name)
        os.makedirs(d, exist_ok=True)
        lines = [f"size {self.size[0]} {self.size[1]} {self.size[2]}", f"dtype {'f64' if self.dtype == np.float64 else 'f32'}",
                 f"periodic {int(self.periodic)}", f"solver {self.solver}", f"precond {int(self.precond)}", f"levels {LEVELS}", "nu 2 2 30",
                 f"iters {ITERS}", "coef_kinds " + " ".join(self.kinds), "inputs " + " ".join(sorted(self.inputs))]
        lines += [f"bc {q} {fc} {kind} {float(c).hex()}" for q, fc, kind, c in self.bcs]
        for l, A in enumerate(self.ops):
            lines.append(f"op {l} {len(A)}")
            for t in A:
                s, o, w, k, c = vo.split(t)
                lines.append(f"{s} {o[0]} {o[1]} {o[2]} {float(w).hex()} {k} {c[0]} {c[1]} {c[2]}")
        with open(os.path.join(d, "case.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
        for n, a in list(self.inputs.items()) + list(self.files.items()):
            np.ascontiguousarray(a, self.dtype).astype(self.dtype.newbyteorder("<")).tofile(os.path.join(d, n + ".bin"))
        return d


# ----------------------------------------------------------------------------------------------- the cases
def multigrid(c, lv, cycle, m, kp=()):
    """3 cycles from u = 0, then (with coefficient fields) kappa scaled, update_coefficients() and a cycle, then a cycle on
    a second pair."""
    shape, T = c.size[::-1], c.dtype.type
    rng = np.random.default_rng(7)
    fh = rng.uniform(-1, 1, shape).astype(c.dtype)
    c.inputs.update(u=np.zeros(shape, c.dtype), f=fh)
    for i, k in enumerate(kp):
        c.inputs[f"k{i}"] = interior(k)
    lv[0].interior(lv[0].f)[...] = fh
    for k in range(1, ITERS + 1):
        cycle(lv)
        c.want[f"cycle{k}"] = interior(lv[0].u)
    if kp:
        for i, k in enumerate(lv[0].k):
            k[...] = k * T(KSCALE)
            c.files[f"ks{i}"] = interior(k)
        vm.update_coefficients(lv, c.kinds)
        cycle(lv)
        c.want["update"] = interior(lv[0].u)
    rng = np.random.default_rng(5)
    u2, f2 = (pad(rng.uniform(-1, 1, shape).astype(c.dtype)) for _ in range(2))
    c.files.update(u2=interior(u2), f2=interior(f2))
    bo.cycle_pair(lv, u2, f2, cycle)
    c.want["pair"] = interior(u2)
    c.info.update(levels=[LEVELS], colours=[m])
    return c


def mg_case(name, size):
    dtype, periodic, walls, sigma, p27 = MG_CASES[name]
    A_at = twenty_seven_at(size) if p27 else helmholtz_at(size, sigma)
    m = 8 if p27 else 2  # the 27-point op reads every neighbour, so red-black does not apply
    c = Case("mg-" + name, "mg", size, dtype, periodic)
    c.ops = [A_at(l) for l in range(LEVELS)]
    c.walls(["u", "u2"], walls)
    lv = mo.hierarchy(size, LEVELS, A_at, np.dtype(dtype), (periodic,) * 3, walls or {}, m=m)
    return multigrid(c, lv, mo.vcycle, m)


def vmg_case(name, size):
    dtype, periodic, walls, cw, kind, sig = VMG_CASES[name]
    ncoef = 4 if sig else 3
    c = Case("vmg-" + name, "mg", size, dtype, periodic, ("x", "y", "z", "cell")[:ncoef])
    A_at = lambda l: vm.helmholtz_div_grad(2.0**l / 32, sigma_field=sig)  # noqa: E731
    c.ops = [A_at(l) for l in range(LEVELS)]
    c.walls(["u", "u2"], walls)
    c.walls([f"k{i}" for i in range(ncoef)], cw)
    lv = vm.hierarchy(size, LEVELS, A_at, c.dtype, (periodic,) * 3, walls or {}, [dict(cw) for _ in range(ncoef)], m=2)
    kp = fields(size, c.dtype, kind, ncoef)
    for a, b in zip(lv[0].k, kp):
        a[...] = b
    vm.update_coefficients(lv, c.kinds)
    return multigrid(c, lv, vm.vcycle, 2, kp)


def solves(c, s, fh, x0, bicg):
    """The oracle of solve(0, k) from x0 for k = 1 .. ITERS and of the solve after dd.swap(): one run, with the history
    and x kept after every iteration; a breakdown ends the run (every later solve stops there too)."""
    I = s.I
    I(s.f)[...] = fh
    I(s.x)[...] = x0
    hist = [math.sqrt(s.start())]
    hists, xs, bd = [list(hist)], [I(s.x).copy()], None
    for k in range(ITERS):
        if bicg:
            ok = s.iterate(k, 0.0, hist)
        else:
            rho = s.iterate(k)
            ok = rho is not None
            if ok:
                hist.append(math.sqrt(rho))
        hists.append(list(hist))
        xs.append(I(s.x).copy())
        if not ok:
            bd = s.breakdown
            break
    for key, n in [(str(k), k) for k in range(1, ITERS + 1)] + [("_swap", ITERS)]:
        i = min(n, len(hists) - 1)
        c.want["swap" if key == "_swap" else "x" + key] = xs[i]
        c.info["hist" + key] = hists[i]
        c.info["breakdown" + key] = [bd if bd is not None and bd < n else -1]
    c.inputs.update(x=x0, f=fh)
    return c


def krylov_data(c, size, dtype, kappa, sigma, h):
    """fh, x0 and the padded coefficient fields of test_gpu_krylov.Setup and test_gpu_bicgstab.Setup."""
    rng = np.random.default_rng(7)
    fh = rng.uniform(-1, 1, size[::-1]).astype(dtype)
    x0 = rng.uniform(-0.5, 0.5, size[::-1]).astype(dtype)
    kp = []
    if kappa is not None:
        kp = vm.kappa_faces(size, h, kappa, dtype)
        if sigma == "field":
            kp.append(np.random.default_rng(7 + 11).uniform(0.5, 2.0, tuple(n + 2 for n in size[::-1])).astype(dtype))
    for i, k in enumerate(kp):
        c.inputs[f"k{i}"] = interior(k)
    return fh, x0, kp


def krylov_hierarchy(c, size, A_at, walls, cw, kp):
    per, hom = (c.periodic,) * 3, ko.homogeneous(walls)
    if not kp:
        return mo.hierarchy(size, LEVELS, A_at, c.dtype, per, hom, m=2)
    lv = vm.hierarchy(size, LEVELS, A_at, c.dtype, per, hom, [dict(cw) for _ in kp], m=2)
    for a, b in zip(lv[0].k, kp):
        a[...] = b
    vm.update_coefficients(lv, c.kinds)
    return lv


def pcg_case(name, size, sign=1.0):
    dtype, periodic, walls, cw, kappa, sigma, precond = PCG_CASES[name]
    cw = {} if periodic or cw is None else cw
    ncoef = 0 if kappa is None else 4 if sigma == "field" else 3
    c = Case(("pcg-" if sign > 0 else "pcg-neg-") + name, "pcg", size, dtype, periodic, ("x", "y", "z", "cell")[:ncoef], precond)
    h = 1.0 / 32
    if kappa is None:
        A_at = lambda l: poisson(h * 2**l, sigma)  # noqa: E731
    else:
        A_at = lambda l: vm.helmholtz_div_grad(h * 2**l, sigma_field=sigma == "field")  # noqa: E731
    if sign < 0:
        A_at = negated(A_at)
    c.ops = [A_at(l) for l in range(LEVELS)]
    c.walls(["x"], walls)
    c.walls(["p", "z"], ko.homogeneous(walls))
    c.walls([f"k{i}" for i in range(ncoef)], cw)
    fh, x0, kp = krylov_data(c, size, c.dtype, kappa, sigma, h)
    if precond:
        c.info.update(levels=[LEVELS], colours=[2])
    return solves(c, ko.PCG(krylov_hierarchy(c, size, A_at, walls, cw, kp), walls, precond=precond), fh, x0, False)


def bicg_case(name, size, sign=1.0):
    dtype, periodic, walls, cw, kappa, sigma = BICG_CASES[name]
    cw = {} if periodic or cw is None else cw
    ncoef = 0 if kappa is None else 4 if sigma == "field" else 3
    c = Case(("bicgstab-" if sign > 0 else "bicgstab-neg-") + name, "bicgstab", size, dtype, periodic, ("x", "y", "z", "cell")[:ncoef])
    h = 1.0 / 32
    if kappa is None:
        A_at = lambda l: poisson(h * 2**l, sigma) + conv(h * 2**l)  # noqa: E731
    else:
        A_at = lambda l: vm.helmholtz_div_grad(h * 2**l, sigma_field=sigma == "field") + conv(h * 2**l)  # noqa: E731
    if sign < 0:
        A_at = negated(A_at)
    c.ops = [A_at(l) for l in range(LEVELS)]
    c.walls(["x"], walls)
    c.walls(["phat", "shat"], ko.homogeneous(walls))
    c.walls([f"k{i}" for i in range(ncoef)], cw)
    fh, x0, kp = krylov_data(c, size, c.dtype, kappa, sigma, h)
    c.info.update(levels=[LEVELS], colours=[2])
    return solves(c, bo.BiCGStab(krylov_hierarchy(c, size, A_at, walls, cw, kp), walls), fh, x0, True)


def passes_case(size):
    """Single passes on -div(kappa grad u), u with ODD(c) walls (a different c per face), kappa with VALUE walls."""
    dtype, periodic, walls, cw, kind, _ = VMG_CASES["oddc-f64"]
    assert walls is ODDC and cw is KVALUE and not periodic
    c = Case("passes-oddc-f64", "passes", size, dtype, periodic, ("x", "y", "z"))
    A = vm.helmholtz_div_grad(1.0 / 32)
    c.ops = [A]
    c.walls(["u"], walls)
    c.walls(["k0", "k1", "k2"], cw)
    c.walls(["cu"], mo.coarse_walls(walls))
    per, csize = (periodic,) * 3, tuple(n // 2 for n in size)
    rng = np.random.default_rng(3)
    uh, fh = (rng.uniform(-1, 1, size[::-1]).astype(dtype) for _ in range(2))
    cuh = rng.uniform(-1, 1, csize[::-1]).astype(dtype)
    kh = [interior(k) for k in fields(size, np.dtype(dtype), kind, 3)]
    c.inputs.update(u=uh, f=fh, k0=kh[0], k1=kh[1], k2=kh[2])
    c.files["cu"] = cuh
    up, fp = padded(uh, periodic, walls), padded(fh, periodic, walls)
    kp = [padded(a, periodic, cw) for a in kh]
    out = np.zeros_like(up)
    vo.apply_box(A, up, None, kp, out, (1, 1, 1), size)
    c.want["apply"] = interior(out)
    for col in range(2):
        vm.fill_ghosts(up, per, walls)
        vm.diag_box(A, 1.0, up, fp, kp, up, (1, 1, 1), size, (-1, -1, -1), 2, col)
        c.want[f"relax{col}"] = interior(up)
    vm.fill_ghosts(up, per, walls)
    want = np.empty(csize[::-1], dtype)
    vm.restrict_vop_box(want, (0, 0, 0), vm.vresidual_terms(A), up, fp, kp, (-1, -1, -1), (0, 0, 0), csize)
    c.want["restrict"] = want
    for a in range(3):
        want = np.empty(csize[::-1], dtype)
        vm.face_restrict_box(want, (0, 0, 0), kh[a], (0, 0, 0), a, (0, 0, 0), csize)
        c.want[f"face{a}"] = want
    cup = padded(cuh, periodic, mo.coarse_walls(walls))
    to.prolong_box(up, (-1, -1, -1), cup, (-1, -1, -1), (0, 0, 0), size, aux=up)
    c.want["prolong"] = interior(up)
    return c


BUILDERS = {"mg-" + n: (mg_case, n) for n in MG_CASES}
BUILDERS.update({"vmg-" + n: (vmg_case, n) for n in VMG_CASES})
BUILDERS.update({"pcg-" + n: (pcg_case, n) for n in PCG_CASES})
BUILDERS.update({"bicgstab-" + n: (bicg_case, n) for n in BICG_CASES})
# -A: PCG breaks down at once (<p, A p> < 0), with and without the preconditioner; BiCGStab on -A as its oracle says
BUILDERS.update({"pcg-neg-" + n: (lambda n, s: pcg_case(n, s, -1.0), n) for n in ("poisson-odd0-f64", "noprec-oddc-f64")})
BUILDERS["bicgstab-neg-cd-odd0-f64"] = (lambda n, s: bicg_case(n, s, -1.0), "cd-odd0-f64")
BUILDERS["passes-oddc-f64"] = (lambda n, s: passes_case(s), None)
NAMES = sorted(BUILDERS)
MPI_CASES = ["vmg-oddc-f64", "pcg-jump-kvalue-f64", "bicgstab-jump-conv-f64", "passes-oddc-f64"]


@pytest.fixture(scope="module")
def cases(tmp_path_factory):
    """size -> {name: (case directory, Case)}, built on first use"""
    root, built = tmp_path_factory.mktemp("cases"), {}

    def get(size):
        if size not in built:
            d = str(root / "x".join(map(str, size)))
            built[size] = {}
            for name in NAMES:
                make, arg = BUILDERS[name]
                c = make(arg, size)
                assert c.name == name
                built[size][name] = (c.write(d), c)
        return built[size]

    return get


def run(cmd, env=None):
    if not os.path.exists(EXE):
        pytest.fail("bin/test_solver_parity not built -- run `make`")
    out = subprocess.run(cmd, env=env or mpirun_env(), capture_output=True, text=True, timeout=1200)
    assert out.returncode == 0 and "done" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.fixture(scope="module", params=PARTS)
def partition(request, cases, tmp_path_factory):
    """Every case on ndom subdomains of one process: (output root, the cases)."""
    ndom = request.param
    cs = cases(fine_size(ndom))
    out = str(tmp_path_factory.mktemp(f"out{ndom}"))
    run([EXE, "--single", str(ndom), out] + [cs[n][0] for n in NAMES])
    return out, cs


def check(out, c):
    d = os.path.join(out, c.name)
    for n, want in sorted(c.want.items()):
        got = np.fromfile(os.path.join(d, n + ".bin"), c.dtype.newbyteorder("<")).astype(c.dtype).reshape(want.shape)
        assert same(got, np.ascontiguousarray(want)), f"{c.name}: {n} differs in {int(np.sum(got != want))} cells, max |diff| {np.nanmax(np.abs(got - want))}"
    info = {}
    with open(os.path.join(d, "info.txt")) as f:
        for line in f:
            k, *v = line.split()
            info[k] = v
    assert sorted(info) == sorted(c.info), (c.name, sorted(info), sorted(c.info))
    for k, want in c.info.items():
        got = [float.fromhex(v) for v in info[k]] if k.startswith("hist") else [int(v) for v in info[k]]
        assert got == want, (c.name, k, got, want)


@pytest.mark.parametrize("name", NAMES)
def test_cpp_solver_bits(partition, name):
    out, cs = partition
    check(out, cs[name][1])


def test_breakdown_cases():
    """The -A cases take the breakdown branch: PCG at its first iteration, with and without the preconditioner."""
    for n in ("poisson-odd0-f64", "noprec-oddc-f64"):
        c = pcg_case(n, (16, 16, 16), -1.0)
        assert c.info["breakdown1"] == [0] and len(c.info["hist3"]) == 1, c.info


@pytest.mark.parametrize("ranks", [2, 4])
def test_cpp_solvers_under_sb_mpirun(tmp_path, cases, ranks):
    cs = cases((32, 32, 32))
    run([os.path.join(BIN, "sb_mpirun"), "-n", str(ranks), EXE, "--ranks", str(tmp_path)] + [cs[n][0] for n in MPI_CASES])
    for n in MPI_CASES:
        check(str(tmp_path), cs[n][1])


def test_cpp_solvers_reference_placement(tmp_path, cases):
    cs = cases((32, 32, 32))
    env = dict(mpirun_env(), SB_ALLOC_ALIGN="0")
    run([EXE, "--single", "4", str(tmp_path), cs["vmg-oddc-f64"][0], cs["passes-oddc-f64"][0]], env=env)
    for n in ("vmg-oddc-f64", "passes-oddc-f64"):
        check(str(tmp_path), cs[n][1])
