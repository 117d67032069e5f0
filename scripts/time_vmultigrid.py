"""Rates of the variable-coefficient multigrid kernels (DESIGN.md section 2.12) and the cost of a stencil_b200.Multigrid
cycle with coefficient fields on one GPU.

    python scripts/time_vmultigrid.py [--iters 40] [--warmup 5] [--cycles 8]

(a) The diagonal relaxation (sb_stencil_dplan_create): one in-place red pass of -div(kappa grad u) = f over 512^3 cells
(ghost width 1), FP64 and FP32, alternated with the coloured damped pass u + theta (div(kappa grad u) - f) of
tests/test_gpu_colour_op.py on the same fields (sb_stencil_cplan_create, red, in place).
(b) The fused residual-restriction with coefficients (sb_transfer_voplan_create) of r = f + div(kappa grad u) from
512^3 into 256^3, against the residual as one sb_stencil_vplan_create launch into a scratch allocation plus the
512^3 -> 256^3 restriction.
(c) The face restriction (sb_transfer_fplan_create) of a 512^3 field for each axis against the 8-cell restriction of
the same field.
Each launch is alternated in the same loop with dst.copy_(src) over two 512^3 allocations (the copy ceiling, bytes =
read + write).  Every timing is the trimean of --iters launches timed one by one with CUDA events on one stream, after
--warmup untimed ones.
(d) Cycles: -div(kappa grad u) = f on 256^3 FP64 cells, ODD(0) walls, EVEN kappa walls, f = uniform(-1, 1) with seed
256, V(2,2) down to 4^3 with 30 coarsest sweeps, kappa smooth (tests/vmg_oracle.kappa_faces) and with a 10^3 jump:
Multigrid.cycle() from u = 0 with the residual after each cycle, then red-black diagonal relaxation sweeps from u = 0
for the wall time of those cycles, then the constant-coefficient cycle (-lap u = f) on the same grid for the ratio; then
the C++ stencil::Multigrid<double> cycle, smooth kappa and constant coefficients, on the same grid size and configuration
(bin/test_vmultigrid_multigpu --time, its own seeded right-hand side and kappa).
Prints the GPU's name, power limit and SM clock, then one JSON line per workload."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from time_boundary import gpu_info, timed, trimean  # noqa: E402
from time_system_op import sm_clock  # noqa: E402

N = 512


def alternate(args, s, runs, a, b):
    """Trimean ms of each launch function in runs (a dict) and of the copy ceiling, alternated launch by launch."""
    import torch

    ts = {k: [] for k in list(runs) + ["copy"]}
    for it in range(args.warmup + args.iters):
        for k, fn in runs.items():
            x = timed(s, fn)
            if it >= args.warmup:
                ts[k].append(x)
        with torch.cuda.stream(s):
            x = timed(s, lambda: b.copy_(a))
        if it >= args.warmup:
            ts["copy"].append(x)
    return {k: trimean(v) for k, v in ts.items()}


def kernels(args, name, limit):
    import numpy as np
    import torch

    import stencil_b200 as sb
    import vmg_oracle as vm
    import vstencil_oracle as vo
    from stencil_b200._lib import Pitched

    s = torch.cuda.Stream()
    n, m, c = N, N + 2, N // 2
    for dtype, tdt in ((np.float64, torch.float64), (np.float32, torch.float32)):
        es = np.dtype(dtype).itemsize
        P = lambda t, k: Pitched(t.data_ptr(), k * es, k)  # noqa: E731
        u, f = torch.rand(m, m, m, dtype=tdt, device="cuda"), torch.rand(m, m, m, dtype=tdt, device="cuda")
        ks = [0.5 + torch.rand(m, m, m, dtype=tdt, device="cuda") for _ in range(3)]
        a, b = torch.rand(n, n, n, dtype=tdt, device="cuda"), torch.empty(n, n, n, dtype=tdt, device="cuda")
        box = [((0, 0, 0), (n, n, n))]
        K = [P(k, m) for k in ks]
        A = sb.StencilOp(vm.helmholtz_div_grad(1.0 / n), dtype)
        theta = 0.02
        damped = sb.StencilOp([(0, (0, 0, 0), 1.0)] + [(s_, o, theta * w, k, cc) for s_, o, w, k, cc in vo.div_grad((1.0 / n,) * 3)]
                              + [(1, (0, 0, 0), -theta)], dtype)
        diag = sb.StencilPlan(0, A, P(u, m), P(u, m), P(f, m), (-1, -1, -1), m, box, K, (2, 0), omega=1.0)
        damp = sb.StencilPlan(0, damped, P(u, m), P(u, m), P(f, m), (-1, -1, -1), m, box, K, (2, 0))
        t = alternate(args, s, {"diag": lambda: diag.launch(s), "damped": lambda: damp.launch(s)}, a, b)
        ceil = 2 * a.numel() * es / (t["copy"] * 1e-3)
        print(json.dumps(dict(workload=f"(a) 512^3 in-place red diagonal relaxation of -div(kappa grad u), {np.dtype(dtype).name}", gpu=name,
                              power_limit=limit, iters=args.iters, bytes=diag.bytes, kernel_ms=round(t["diag"], 4),
                              GBps=round(diag.bytes / (t["diag"] * 1e-3) / 1e9, 1), damped_pass_ms=round(t["damped"], 4),
                              diag_over_damped=round(t["diag"] / t["damped"], 3), target_1_10_met=bool(t["diag"] <= 1.10 * t["damped"]),
                              copy_ms=round(t["copy"], 4), copy_ceiling_GBps=round(ceil / 1e9, 1),
                              share_of_copy_ceiling=round(diag.bytes / (t["diag"] * 1e-3) / ceil, 3))), flush=True)
        for p in (diag, damp):
            p.destroy()
        # (b) the fused coefficient residual-restriction against the vplan residual plus the restriction
        r = torch.empty(m, m, m, dtype=tdt, device="cuda")
        coarse = torch.empty(c, c, c, dtype=tdt, device="cuda")
        res = sb.StencilOp(vm.vresidual_terms(vm.helmholtz_div_grad(1.0 / n)), dtype)
        fused = sb.TransferPlan.fused(0, res, P(coarse, c), (0, 0, 0), c, P(u, m), (-1, -1, -1), m, P(f, m), [((0, 0, 0), (c, c, c))], K)
        apply = sb.StencilPlan(0, res, P(r, m), P(u, m), P(f, m), (-1, -1, -1), m, box, K)
        restrict = sb.TransferPlan(0, dtype, 0, P(coarse, c), (0, 0, 0), c, P(r, m), (-1, -1, -1), m, None, (0, 0, 0), (c, c, c))
        t = alternate(args, s, {"fused": lambda: fused.launch(s), "apply": lambda: apply.launch(s), "restrict": lambda: restrict.launch(s)}, a, b)
        ceil = 2 * a.numel() * es / (t["copy"] * 1e-3)
        rate = fused.bytes / (t["fused"] * 1e-3)
        print(json.dumps(dict(workload=f"(b) 512^3 -> 256^3 fused residual-restriction of -div(kappa grad u), {np.dtype(dtype).name}", gpu=name,
                              power_limit=limit, iters=args.iters, bytes=fused.bytes, kernel_ms=round(t["fused"], 4), GBps=round(rate / 1e9, 1),
                              residual_apply_ms=round(t["apply"], 4), restriction_ms=round(t["restrict"], 4),
                              fused_over_unfused=round(t["fused"] / (t["apply"] + t["restrict"]), 3),
                              target_0_6_met=bool(t["fused"] <= 0.6 * (t["apply"] + t["restrict"])), copy_ms=round(t["copy"], 4),
                              share_of_copy_ceiling=round(rate / ceil, 3))), flush=True)
        for p in (fused, apply, restrict):
            p.destroy()
        # (c) the face restriction per axis against the 8-cell restriction of the same field
        plans = {"cell": sb.TransferPlan(0, dtype, 0, P(coarse, c), (0, 0, 0), c, P(a, n), (0, 0, 0), n, None, (0, 0, 0), (c, c, c))}
        for ax in range(3):
            plans[f"face{ax}"] = sb.TransferPlan.face(0, dtype, ax, P(coarse, c), (0, 0, 0), c, P(a, n), (0, 0, 0), n, (0, 0, 0), (c, c, c))
        t = alternate(args, s, {k: (lambda p=p: p.launch(s)) for k, p in plans.items()}, a, b)
        print(json.dumps(dict(workload=f"(c) 512^3 -> 256^3 face restriction per axis, {np.dtype(dtype).name}", gpu=name, power_limit=limit,
                              iters=args.iters, eight_cell_ms=round(t["cell"], 4), face_ms=[round(t[f"face{ax}"], 4) for ax in range(3)],
                              face_over_eight_cell=[round(t[f"face{ax}"] / t["cell"], 3) for ax in range(3)],
                              target_no_slower_met=bool(all(t[f"face{ax}"] <= t["cell"] for ax in range(3))), copy_ms=round(t["copy"], 4))),
              flush=True)
        for p in plans.values():
            p.destroy()
        del u, f, ks, a, b, r, coarse
        torch.cuda.empty_cache()


def cycles(args, name, limit):
    import numpy as np

    import stencil_b200 as sb
    import vmg_oracle as vm
    from test_gpu_stencil_domain import load

    n = 256
    levels = int(np.log2(n)) - 1  # down to 4^3
    h = 1.0 / n
    f = np.random.default_rng(256).uniform(-1, 1, (n, n, n))
    fnorm = float(np.linalg.norm(f))
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(sb.Radius.constant(1))
    u, fq, r = (dd.add_data(np.float64, x) for x in ("u", "f", "r"))
    ks = [dd.add_data(np.float64, x) for x in ("kx", "ky", "kz")]
    dd.set_boundary(sb.Boundary.FIXED, sb.Boundary.FIXED, sb.Boundary.FIXED)
    for fc in sb.FACES:
        dd.set_boundary_condition(u, fc, sb.BC.ODD(0.0))
        for k in ks:
            dd.set_boundary_condition(k, fc, sb.BC.EVEN())
    dd.realize()
    load(dd, fq.id, "curr", f)
    zero = np.zeros((n, n, n))
    out = {}
    for kind in ("smooth", "jump"):
        for q, a in zip(ks, vm.kappa_faces(n, h, kind, np.float64)):
            load(dd, q.id, "curr", a[1:-1, 1:-1, 1:-1].copy())
        A = lambda l: sb.StencilOp(vm.helmholtz_div_grad(h * 2 ** l), np.float64)  # noqa: E731
        t0 = time.perf_counter()
        mg = sb.Multigrid(dd, u, fq, r, A, levels=levels, coefs=ks)
        build = time.perf_counter() - t0
        load(dd, u.id, "curr", zero)
        mg.cycle()  # warm-up: plans, streams, first launches
        load(dd, u.id, "curr", zero)
        res, times = [mg.residual_norm()], []
        for _ in range(args.cycles):
            t0 = time.perf_counter()
            mg.cycle()
            times.append(time.perf_counter() - t0)
            res.append(mg.residual_norm())
        t0 = time.perf_counter()
        mg.update_coefficients()
        upd = time.perf_counter() - t0
        # red-black diagonal relaxation for the same wall time
        load(dd, u.id, "curr", zero)
        op = A(0)
        budget, sweeps, t0 = sum(times), 0, time.perf_counter()
        while time.perf_counter() - t0 < budget:
            for c in range(2):
                dd.relax(op, (u, "curr"), u, fq, coefs=ks, colour=(2, c))
            sweeps += 1
        rb = mg.residual_norm()
        mg.close()
        rec = dict(workload=f"(d) 256^3 FP64 -div(kappa grad u) = f, {kind} kappa, ODD(0) walls, V(2,2) to 4^3, 30 coarsest sweeps: Multigrid.cycle()",
                   gpu=name, power_limit=limit, f_norm=fnorm, ms_per_cycle=[round(t * 1e3, 2) for t in times],
                   median_ms=round(float(np.median(times)) * 1e3, 2), residual=[float(f"{x:.4g}") for x in res],
                   factor=[round(res[k + 1] / res[k], 4) for k in range(args.cycles)], build_s=round(build, 2),
                   update_coefficients_ms=round(upd * 1e3, 2), red_black_sweeps_same_time=sweeps, red_black_residual=float(f"{rb:.4g}"))
        out[kind] = float(np.median(times))
        print(json.dumps(rec), flush=True)
    # the constant-coefficient cycle on the same grid
    import colour_oracle as co

    A = lambda l: sb.StencilOp(co.helmholtz(2.0 ** l / n, 0.0), np.float64)  # noqa: E731
    mg = sb.Multigrid(dd, u, fq, r, A, levels=levels)
    load(dd, u.id, "curr", zero)
    mg.cycle()
    times = []
    for _ in range(args.cycles):
        t0 = time.perf_counter()
        mg.cycle()
        times.append(time.perf_counter() - t0)
    mg.close()
    tc = float(np.median(times))
    print(json.dumps(dict(workload="(d) 256^3 FP64 -lap u = f, same grid and cycle: Multigrid.cycle()", gpu=name, power_limit=limit,
                          median_ms=round(tc * 1e3, 2), smooth_over_constant=round(out["smooth"] / tc, 3), jump_over_constant=round(out["jump"] / tc, 3),
                          target_2_5_met=bool(out["smooth"] <= 2.5 * tc))), flush=True)
    dd.close()
    # the C++ solver on the same grid (its own process, right-hand side and kappa)
    import subprocess

    out = subprocess.run([os.path.join(ROOT, "bin", "test_vmultigrid_multigpu"), "--time", str(n), str(args.cycles)], capture_output=True, text=True,
                         timeout=600)
    med = []
    for line in out.stdout.splitlines():
        if line.startswith("{"):
            rec = json.loads(line)
            rec.update(gpu=name, power_limit=limit, median_ms=round(float(np.median(rec["ms_per_cycle"])), 2))
            med.append(rec["median_ms"])
            print(json.dumps(rec), flush=True)
    if len(med) == 2:
        print(json.dumps(dict(workload="(d) C++ coefficient cycle over the C++ constant-coefficient cycle", gpu=name, power_limit=limit,
                              ratio=round(med[0] / med[1], 3), target_2_5_met=bool(med[0] <= 2.5 * med[1]))), flush=True)
    if out.returncode != 0:
        print(out.stdout[-2000:] + out.stderr[-2000:], flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cycles", type=int, default=8)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_vmultigrid.py measures on a CUDA device; none is available")
    name, limit = gpu_info()
    print(f"# {name}, power limit {limit}, SM clock (current, max) {sm_clock()}", flush=True)
    kernels(args, name, limit)
    cycles(args, name, limit)


if __name__ == "__main__":
    main()
