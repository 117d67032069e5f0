"""Rate of the multigrid transfer kernels (sb_transfer_plan_*) on one GPU against the copy ceiling of the same run, and
the cost and effect of V(2,2) cycles built on them (tests/mg_gpu.py).

    python scripts/time_transfer.py [--iters 40] [--warmup 5] [--cycles 12]

Kernels, each one launch over the whole region:
  512^3 -> 256^3 restriction, FP64 and FP32 (fine allocation 512^3, no ghost cells read);
  256^3 -> 512^3 prolongation in place (u <- u + P e), FP64 and FP32 (coarse allocation 258^3 with its ghost layer).
Each transfer launch is alternated with dst.copy_(src) over two 512^3 allocations (the copy ceiling, bytes = read +
write) and with the 7-point Laplacian over 512^3 cells (one tile-kernel launch).  Bytes: sb_transfer_plan_bytes (every
element the rule reads once, one written per cell of the box).  Every timing is the trimean of --iters launches timed
one by one with CUDA events on one stream, after --warmup untimed ones.

Solve: -lap u = f on 256^3 FP64 cells of a unit cube, f = uniform(-1, 1) with seed 256, Dirichlet ODD(0) on every face,
u = 0.  V(2,2) cycles (red-black Gauss-Seidel, 30 sweeps on the coarsest level of 4^3) until ||f - A u||_2 <= 1e-8 ||f||_2
or --cycles cycles: the wall time per cycle and per level, and the residual after each cycle.  Then red-black
Gauss-Seidel sweeps from u = 0 on the same grid for the same wall time, and their residual.
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


def kernels(args, name, limit):
    import numpy as np
    import torch

    import stencil_b200 as sb
    from stencil_b200._lib import Pitched

    s = torch.cuda.Stream()
    n, c, m = N, N // 2, N // 2 + 2
    lap_box = [((1, 1, 1), (N - 1, N - 1, N - 1))]
    for dtype, tdt in ((np.float64, torch.float64), (np.float32, torch.float32)):
        es = np.dtype(dtype).itemsize
        fine, fine2 = torch.rand(n, n, n, dtype=tdt, device="cuda"), torch.rand(n, n, n, dtype=tdt, device="cuda")
        coarse, ghosted = torch.rand(c, c, c, dtype=tdt, device="cuda"), torch.rand(m, m, m, dtype=tdt, device="cuda")
        cbytes = 2 * fine.numel() * es
        P = lambda t, k: Pitched(t.data_ptr(), k * es, k)  # noqa: E731
        lap = sb.StencilPlan(0, sb.StencilOp.laplacian(2, (1, 1, 1), dtype), P(fine2, n), P(fine, n), Pitched(None, 0, 0), (0, 0, 0), n, lap_box)
        work = [("512^3 -> 256^3 restriction", sb.TransferPlan(0, dtype, 0, P(coarse, c), (0, 0, 0), c, P(fine, n), (0, 0, 0), n, None, (0, 0, 0), (c,) * 3)),
                ("256^3 -> 512^3 prolongation in place", sb.TransferPlan(0, dtype, 1, P(fine2, n), (0, 0, 0), n, P(ghosted, m), (-1, -1, -1), m, P(fine2, n),
                                                                         (0, 0, 0), (n,) * 3))]
        for label, plan in work:
            tt, tc, tl = [], [], []
            for it in range(args.warmup + args.iters):
                a = timed(s, lambda: plan.launch(s))
                with torch.cuda.stream(s):
                    b = timed(s, lambda: fine2.copy_(fine))
                d = timed(s, lambda: lap.launch(s))
                if it >= args.warmup:
                    tt.append(a)
                    tc.append(b)
                    tl.append(d)
            t, tcopy, tlap = trimean(tt), trimean(tc), trimean(tl)
            ceil, rate = cbytes / (tcopy * 1e-3), plan.bytes / (t * 1e-3)
            rec = dict(workload=f"{label}, {np.dtype(dtype).name}", gpu=name, power_limit=limit, iters=args.iters, bytes=plan.bytes, kernel_ms=round(t, 4),
                       GBps=round(rate / 1e9, 1), copy_ms=round(tcopy, 4), copy_ceiling_GBps=round(ceil / 1e9, 1), share_of_copy_ceiling=round(rate / ceil, 3),
                       target_0_8_met=bool(rate / ceil >= 0.8), laplacian_512_ms=round(tlap, 4), laplacian_GBps=round(lap.bytes / (tlap * 1e-3) / 1e9, 1))
            print(json.dumps(rec), flush=True)
            plan.destroy()
        lap.destroy()
        del fine, fine2, coarse, ghosted
        torch.cuda.empty_cache()


def solve(args, name, limit):
    import numpy as np

    import mg_gpu
    from test_gpu_stencil_domain import load

    n = 256
    f = np.random.default_rng(256).uniform(-1, 1, (n, n, n))
    fnorm = float(np.linalg.norm(f))
    lv = mg_gpu.hierarchy((n, n, n), int(np.log2(n)) - 1, 0.0, np.float64, (mg_gpu.F,) * 3, [0])  # down to 4^3
    load(lv[0].dd, lv[0].f.id, "curr", f)
    for L in lv:
        load(L.dd, L.u.id, "curr", np.zeros(L.size[::-1]))
    per_level = [0.0] * len(lv)

    def timed_cycle(l=0):
        # as mg_gpu.vcycle, with the host time of each level's own work (every call returns when its work is complete)
        L = lv[l]
        t0 = time.perf_counter()
        if l == len(lv) - 1:
            L.smooth(30)
            per_level[l] += time.perf_counter() - t0
            return
        L.smooth(2)
        L.residual()
        C = lv[l + 1]
        L.dd.restrict_to(C.dd, (C.f, "curr"), (L.r, "curr"))
        C.dd.apply(C.zero, (C.u, "curr"), C.f, exchange=False)
        per_level[l] += time.perf_counter() - t0
        timed_cycle(l + 1)
        t0 = time.perf_counter()
        L.dd.prolong_from(C.dd, (L.u, "curr"), (C.u, "curr"), aux=(L.u, "curr"))
        L.smooth(2)
        per_level[l] += time.perf_counter() - t0

    timed_cycle()  # warm-up cycle: plans, streams, first launches
    for L in lv:
        load(L.dd, L.u.id, "curr", np.zeros(L.size[::-1]))
    per_level = [0.0] * len(lv)
    res, times, total = [lv[0].residual_norm()], [], 0.0
    while res[-1] > 1e-8 * fnorm and len(times) < args.cycles:
        t0 = time.perf_counter()
        timed_cycle()
        times.append(time.perf_counter() - t0)
        total += times[-1]
        res.append(lv[0].residual_norm())
    share2 = (per_level[0] + per_level[1]) / sum(per_level)
    rec = dict(workload="256^3 FP64 -lap u = f, ODD(0) walls, V(2,2) to 4^3", gpu=name, power_limit=limit, f_norm=fnorm, cycles=len(times),
               ms_per_cycle=[round(t * 1e3, 2) for t in times], residual=[float(f"{r:.4g}") for r in res],
               factor=[round(res[k + 1] / res[k], 4) for k in range(len(times))], wall_s_to_1e_8=round(total, 3) if res[-1] <= 1e-8 * fnorm else None,
               level_ms_per_cycle=[round(t * 1e3 / len(times), 2) for t in per_level], two_finest_share=round(share2, 3))
    print(json.dumps(rec), flush=True)
    # red-black Gauss-Seidel for the same wall time
    L = lv[0]
    load(L.dd, L.u.id, "curr", np.zeros((n, n, n)))
    L.smooth(1)  # warm-up
    load(L.dd, L.u.id, "curr", np.zeros((n, n, n)))
    sweeps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < total:
        L.smooth(1)
        sweeps += 1
    rec = dict(workload="256^3 FP64 -lap u = f, ODD(0) walls, red-black Gauss-Seidel for the same wall time", gpu=name, power_limit=limit,
               wall_s=round(time.perf_counter() - t0, 3), sweeps=sweeps, residual=float(f"{L.residual_norm():.4g}"), f_norm=fnorm)
    print(json.dumps(rec), flush=True)
    mg_gpu.close(lv)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cycles", type=int, default=12)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_transfer.py measures on a CUDA device; none is available")
    name, limit = gpu_info()
    print(f"# {name}, power limit {limit}, SM clock (current, max) {sm_clock()}", flush=True)
    kernels(args, name, limit)
    solve(args, name, limit)


if __name__ == "__main__":
    main()
