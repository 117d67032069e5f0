"""Time of the BiCGStab Krylov kernels (SB_KRYLOV_BICG_P, SB_KRYLOV_UPDATE with c) and of the Python BiCGStab on one GPU.

    python scripts/time_bicgstab.py [--iters 30] [--warmup 5] [--solver-iters 8]

512^3, radius 1.  Workloads, each launch alternated with dst.copy_(src) of one field (the copy ceiling):
  (a) BICG_P p = r + T(beta) (p - T(omega) v), FP64 and FP32, against torch's three in-place ops
      p.sub_(v, alpha=omega).mul_(beta).add_(r) on tensors of the same size;
  (b) UPDATE with c (x += T(s) p, r -= T(s) q with <r, r> and <c, r>) against UPDATE followed by the one-pair DOT <c, r>,
      FP64 and FP32.
Each kernel timing is the trimean of --iters CUDA-event timings after --warmup untimed rounds.  Then, 256^3 FP64
-div(kappa grad x) + b . grad x = f with a 10^3 jump in kappa, ODD(0) walls, V(2,2) to 4^3, from Python:
  (c) one BiCGStab iteration against two cycles of its preconditioner (median of 3);
  (d) BiCGStab's wall time to 1e-8 of ||f||, then Multigrid.cycle() repeated and PCG iterations (on the same
      non-symmetric op) for the same wall time, each from x = 0; the relative true residual ||f - A x|| / ||f|| each
      leaves (residual_norm()).
The C++ solver is timed by bin/test_bicgstab_multigpu --time N C.
Prints one JSON line per workload with the GPU's name and power limit."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from time_boundary import gpu_info  # noqa: E402
from time_krylov import alternate  # noqa: E402

B = (4.0, 2.4, 1.2)


def kernels(sb, torch, dtype, name, limit, args):
    n = 512
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(1)
    x, p, r, q, c = (dd.add_data(dtype, k) for k in "xprqc")
    dd.realize()
    d = dd.domains()[0]
    rng = np.random.default_rng(1)
    for h in (x, p, r, q, c):
        d.quantity_from_host(h.id, rng.standard_normal(d.raw_size()[::-1]).astype(dtype))
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    src = torch.randn(n**3, dtype=tdt, device="cuda")
    dst = torch.empty_like(src)
    tp, tr, tv = (torch.randn(n**3, dtype=tdt, device="cuda") for _ in range(3))
    s = torch.cuda.Stream()
    tag = "FP64" if dtype == np.float64 else "FP32"
    es = np.dtype(dtype).itemsize
    copy = lambda: dst.copy_(src)  # noqa: E731
    K = sb._lib
    bp = dd.krylov_plans(K.KRYLOV_BICG_P, (p, r, q))[0]
    bp.s, bp.t = 0.5, 0.25  # |p| stays bounded over many launches

    def torch_three():
        tp.sub_(tv, alpha=0.25).mul_(0.5).add_(tr)

    t_bp, t_th, t_c = alternate(torch, s, [lambda: bp.launch(s), torch_three, copy], args)
    print(json.dumps(dict(workload=f"(a) 512^3 {tag} BICG_P", gpu=name, power_limit=limit, iters=args.iters, bicg_p_ms=round(t_bp, 4),
                          torch_three_ops_ms=round(t_th, 4), bicg_p_over_torch=round(t_bp / t_th, 3), copy_ms_per_field=round(t_c, 4),
                          bicg_p_GBps=round(bp.bytes / (t_bp * 1e-3) / 1e9, 1), copy_GBps=round(2 * n**3 * es / (t_c * 1e-3) / 1e9, 1))),
          flush=True)
    upc = dd.krylov_plans(K.KRYLOV_UPDATE, (x, p, r, q, c))[0]
    up = dd.krylov_plans(K.KRYLOV_UPDATE, (x, p, r, q))[0]
    cr = dd.krylov_plans(K.KRYLOV_DOT, (c, r))[0]
    upc.s = up.s = 1e-3

    def pair():
        up.launch(s)
        cr.launch(s)

    t_upc, t_pair, t_c = alternate(torch, s, [lambda: upc.launch(s), pair, copy], args)
    print(json.dumps(dict(workload=f"(b) 512^3 {tag} UPDATE with c", gpu=name, power_limit=limit, iters=args.iters, update_c_ms=round(t_upc, 4),
                          update_plus_dot_ms=round(t_pair, 4), update_c_over_pair=round(t_upc / t_pair, 3), copy_ms_per_field=round(t_c, 4),
                          update_c_GBps=round(upc.bytes / (t_upc * 1e-3) / 1e9, 1))), flush=True)
    dd.close()
    del src, dst, tp, tr, tv
    torch.cuda.empty_cache()


def conv(h):
    return [(0, tuple(sg * (a == j) for j in range(3)), sg * B[a] / (2 * h)) for a in range(3) for sg in (1, -1)]


def solvers(sb, torch, name, limit, args):
    import vmg_oracle as vm
    from test_gpu_stencil_domain import load

    n, dtype = 256, np.float64
    h = 1.0 / n
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(1)
    V = {k: dd.add_data(dtype, k) for k in sb.BiCGStab.NAMES}
    z, q = dd.add_data(dtype, "z"), dd.add_data(dtype, "q")
    ks = [dd.add_data(dtype, k) for k in ("kx", "ky", "kz")]
    dd.set_boundary(sb.Boundary.FIXED)
    for fc in sb.FACES:
        for k in ("x", "phat", "shat"):
            dd.set_boundary_condition(V[k], fc, sb.BC.ODD(0.0))
        for k in (z, V["p"]):  # PCG's p and z
            dd.set_boundary_condition(k, fc, sb.BC.ODD(0.0))
        for k in ks:
            dd.set_boundary_condition(k, fc, sb.BC.EVEN())
    dd.realize()
    d = dd.domains()[0]
    for k, a in zip(ks, vm.kappa_faces(n, h, "jump", dtype)):
        load(dd, k.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1]))
    load(dd, V["f"].id, "curr", np.random.default_rng(0).uniform(-1, 1, (n, n, n)))
    zero = np.zeros(d.raw_size()[::-1], dtype)
    A_at = lambda l: sb.StencilOp(vm.helmholtz_div_grad(h * 2**l) + conv(h * 2**l), dtype)  # noqa: E731
    bi = sb.BiCGStab(dd, *(V[k] for k in sb.BiCGStab.NAMES), A_at, coefs=ks)
    nf = dd.reduce(V["f"], "curr", exact=True).l2()

    def timed_solve(fn):
        d.quantity_from_host(V["x"].id, zero)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    bi.solve(0.0, 2)  # warm-up: plans, first launches
    t_it = []
    for _ in range(3):
        t0, _ = timed_solve(lambda: bi.solve(0.0, 0))
        t1, _ = timed_solve(lambda: bi.solve(0.0, args.solver_iters))
        t_it.append((t1 - t0) / args.solver_iters)
    t_it = float(np.median(t_it))
    d.quantity_from_host(V["phat"].id, zero)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(args.solver_iters):
        bi.mg.cycle()
    t_cyc = (time.perf_counter() - t0) / args.solver_iters
    print(json.dumps(dict(workload="(c) 256^3 FP64 jump kappa + convection, V(2,2) to 4^3: stencil_b200.BiCGStab iteration vs two cycles of its "
                          "preconditioner", gpu=name, power_limit=limit, ms_per_iteration=round(t_it * 1e3, 2), ms_per_vcycle=round(t_cyc * 1e3, 2),
                          ratio_to_two_cycles=round(t_it / (2 * t_cyc), 3))), flush=True)
    t_bi, hist = timed_solve(lambda: bi.solve(1e-8, 30))
    res_bi = bi.residual_norm()
    bi.close()
    # Multigrid and PCG on the same op, given the same wall time
    mg = sb.Multigrid(dd, V["x"], V["f"], V["r"], A_at, coefs=ks)
    mg.solve(0.0, 1)

    def mg_for(seconds):
        t0 = time.perf_counter()
        while time.perf_counter() - t0 < seconds:
            mg.cycle()
        return mg.residual_norm()

    t_mg, res_mg = timed_solve(lambda: mg_for(t_bi))
    mg.close()
    cg = sb.PCG(dd, V["x"], V["f"], V["r"], z, V["p"], q, A_at, coefs=ks)
    cg.solve(0.0, 1)

    def cg_for(seconds):
        t0, k = time.perf_counter(), 0
        cg._start()
        res = math.inf
        while time.perf_counter() - t0 < seconds:
            rho = cg._iterate(k)
            if rho is None:
                break
            res = math.sqrt(rho)
            k += 1
        return res, k

    t_cg, (_, k_cg) = timed_solve(lambda: cg_for(t_bi))
    res_cg = cg.residual_norm()
    cg.close()
    print(json.dumps(dict(workload="(d) 256^3 FP64 jump kappa + convection to 1e-8, V(2,2) to 4^3: BiCGStab time, and what Multigrid and PCG "
                          "leave in that time", gpu=name, power_limit=limit, bicgstab_s=round(t_bi, 3), bicgstab_iterations=len(hist) - 1,
                          bicgstab_rel_residual=res_bi / nf, multigrid_s=round(t_mg, 3), multigrid_rel_residual=res_mg / nf, pcg_s=round(t_cg, 3),
                          pcg_iterations=k_cg, pcg_rel_residual=res_cg / nf, pcg_breakdown=cg.breakdown)), flush=True)
    dd.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--solver-iters", type=int, default=8)
    ap.add_argument("--skip-solvers", action="store_true")
    args = ap.parse_args()
    import torch

    import stencil_b200 as sb

    if not torch.cuda.is_available():
        raise SystemExit("time_bicgstab.py needs a CUDA device")
    name, limit = gpu_info()
    for dtype in (np.float64, np.float32):
        kernels(sb, torch, dtype, name, limit, args)
    if not args.skip_solvers:
        solvers(sb, torch, name, limit, args)


if __name__ == "__main__":
    main()
