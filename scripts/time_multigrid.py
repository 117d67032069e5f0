"""Rate of the fused residual-restriction (sb_transfer_oplan_create) and the cost of a stencil_b200.Multigrid cycle on
one GPU.

    python scripts/time_multigrid.py [--iters 40] [--warmup 5] [--cycles 6]

(a) Kernels, FP64 and FP32, each one launch over the whole region: the fused residual-restriction r = f - A u of the
7-point ODD(0) Poisson operator from a 514^3 fine allocation (ghost width 1) into 256^3 coarse cells, alternated in the
same loop with its unfused form (the residual as one sb_stencil_plan over 512^3 cells into a scratch allocation, then
the 512^3 -> 256^3 restriction) and with dst.copy_(src) over two 512^3 allocations (the copy ceiling, bytes = read +
write).  Bytes: sb_transfer_plan_bytes (per coarse cell 8 src and 8 aux elements and one written).  Every timing is the
trimean of --iters launches timed one by one with CUDA events on one stream, after --warmup untimed ones.

(b) Cycles: -lap u = f on 256^3 FP64 cells, ODD(0) walls, f = uniform(-1, 1) with seed 256, V(2,2) down to 4^3 with 30
coarsest sweeps (DESIGN.md section 2.10's configuration): the tests/mg_gpu.py cycle (public synchronising calls) and
Multigrid.cycle() alternated, --cycles of each from u = 0, the wall time per cycle, the host time spent queueing a
Multigrid cycle, and the residual after each cycle; then the C++ stencil::Multigrid<double> cycle on the same grid size
and configuration (bin/test_multigrid_multigpu --time, its own seeded right-hand side and ODD(c) walls).
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

    import colour_oracle as co
    import stencil_b200 as sb
    import transfer_oracle as to
    from stencil_b200._lib import Pitched

    s = torch.cuda.Stream()
    n, m, c = N, N + 2, N // 2
    for dtype, tdt in ((np.float64, torch.float64), (np.float32, torch.float32)):
        es = np.dtype(dtype).itemsize
        u, f = torch.rand(m, m, m, dtype=tdt, device="cuda"), torch.rand(m, m, m, dtype=tdt, device="cuda")
        r = torch.empty(m, m, m, dtype=tdt, device="cuda")
        a, b = torch.rand(n, n, n, dtype=tdt, device="cuda"), torch.empty(n, n, n, dtype=tdt, device="cuda")
        coarse = torch.empty(c, c, c, dtype=tdt, device="cuda")
        P = lambda t, k: Pitched(t.data_ptr(), k * es, k)  # noqa: E731
        res = sb.StencilOp(to.residual_terms(co.helmholtz(1.0 / n, 0.0)), dtype)
        fused = sb.TransferPlan.fused(0, res, P(coarse, c), (0, 0, 0), c, P(u, m), (-1, -1, -1), m, P(f, m), [((0, 0, 0), (c, c, c))])
        apply = sb.StencilPlan(0, res, P(r, m), P(u, m), P(f, m), (-1, -1, -1), m, [((0, 0, 0), (n, n, n))])
        restrict = sb.TransferPlan(0, dtype, 0, P(coarse, c), (0, 0, 0), c, P(r, m), (-1, -1, -1), m, None, (0, 0, 0), (c, c, c))
        tf, ta, tr, tc = [], [], [], []
        for it in range(args.warmup + args.iters):
            x = timed(s, lambda: fused.launch(s))
            y = timed(s, lambda: apply.launch(s))
            z = timed(s, lambda: restrict.launch(s))
            with torch.cuda.stream(s):
                w = timed(s, lambda: b.copy_(a))
            if it >= args.warmup:
                tf.append(x)
                ta.append(y)
                tr.append(z)
                tc.append(w)
        t, tapp, tres, tcopy = trimean(tf), trimean(ta), trimean(tr), trimean(tc)
        ceil, rate = 2 * a.numel() * es / (tcopy * 1e-3), fused.bytes / (t * 1e-3)
        rec = dict(workload=f"512^3 -> 256^3 fused residual-restriction, 7-point, {np.dtype(dtype).name}", gpu=name, power_limit=limit,
                   iters=args.iters, bytes=fused.bytes, kernel_ms=round(t, 4), GBps=round(rate / 1e9, 1), copy_ms=round(tcopy, 4),
                   copy_ceiling_GBps=round(ceil / 1e9, 1), share_of_copy_ceiling=round(rate / ceil, 3), target_0_8_met=bool(rate / ceil >= 0.8),
                   residual_apply_ms=round(tapp, 4), restriction_ms=round(tres, 4), fused_over_unfused=round(t / (tapp + tres), 3),
                   target_0_6_met=bool(t <= 0.6 * (tapp + tres)))
        print(json.dumps(rec), flush=True)
        for p in (fused, apply, restrict):
            p.destroy()
        del u, f, r, a, b, coarse
        torch.cuda.empty_cache()


def cycles(args, name, limit):
    import numpy as np

    import colour_oracle as co
    import mg_gpu
    import stencil_b200 as sb
    from test_gpu_stencil_domain import load

    n = 256
    levels = int(np.log2(n)) - 1  # down to 4^3
    f = np.random.default_rng(256).uniform(-1, 1, (n, n, n))
    fnorm = float(np.linalg.norm(f))
    lv = mg_gpu.hierarchy((n, n, n), levels, 0.0, np.float64, (mg_gpu.F,) * 3, [0])
    load(lv[0].dd, lv[0].f.id, "curr", f)
    L0 = lv[0]
    A = lambda l: sb.StencilOp(co.helmholtz(2.0 ** l / n, 0.0), np.float64)  # noqa: E731
    mg = sb.Multigrid(L0.dd, L0.u, L0.f, L0.r, A, levels=levels)

    def reset():
        for L in lv:
            load(L.dd, L.u.id, "curr", np.zeros(L.size[::-1]))

    reset()
    mg_gpu.vcycle(lv)  # warm-up: plans, streams, first launches
    mg.cycle()
    queue_ms = []

    def timed_mg():
        t0 = time.perf_counter()
        mg.cycle(wait=False)
        queue_ms.append((time.perf_counter() - t0) * 1e3)
        mg.wait()

    out = {}
    for rnd in range(2):  # alternate the two cycles, twice
        for label, run in (("tests/mg_gpu.py cycle (public synchronising calls)", lambda: mg_gpu.vcycle(lv)), ("Multigrid.cycle()", mg.cycle)):
            reset()
            res, times = [lv[0].residual_norm()], []
            for _ in range(args.cycles):
                t0 = time.perf_counter()
                run()
                times.append(time.perf_counter() - t0)
                res.append(lv[0].residual_norm())
            out.setdefault(label, []).append((times, res))
    reset()
    for _ in range(args.cycles):
        timed_mg()
    for label, runs in out.items():
        times = [t for tt, _ in runs for t in tt]
        rec = dict(workload=f"256^3 FP64 -lap u = f, ODD(0) walls, V(2,2) to 4^3, 30 coarsest sweeps: {label}", gpu=name, power_limit=limit,
                   f_norm=fnorm, ms_per_cycle=[round(t * 1e3, 2) for t in times], median_ms=round(float(np.median(times)) * 1e3, 2),
                   residual=[float(f"{r:.4g}") for r in runs[-1][1]], factor=[round(runs[-1][1][k + 1] / runs[-1][1][k], 4) for k in range(args.cycles)])
        print(json.dumps(rec), flush=True)
    a = float(np.median([t for tt, _ in out["tests/mg_gpu.py cycle (public synchronising calls)"] for t in tt]))
    b = float(np.median([t for tt, _ in out["Multigrid.cycle()"] for t in tt]))
    print(json.dumps(dict(workload="Multigrid.cycle() over the mg_gpu.py cycle", gpu=name, power_limit=limit, ratio=round(b / a, 3),
                          target_0_5_met=bool(b <= 0.5 * a), host_queue_ms_per_cycle=[round(t, 2) for t in queue_ms])), flush=True)
    mg.close()
    mg_gpu.close(lv)
    # the C++ solver on the same grid (its own process; the right-hand side is the test's seeded pattern, not this one)
    import subprocess

    out = subprocess.run([os.path.join(ROOT, "bin", "test_multigrid_multigpu"), "--time", str(n), str(args.cycles)], capture_output=True, text=True,
                         timeout=600)
    for line in out.stdout.splitlines():
        if line.startswith("{"):
            rec = json.loads(line)
            rec.update(gpu=name, power_limit=limit, median_ms=round(float(np.median(rec["ms_per_cycle"])), 2))
            print(json.dumps(rec), flush=True)
    if out.returncode != 0:
        print(out.stdout[-2000:] + out.stderr[-2000:], flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cycles", type=int, default=6)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_multigrid.py measures on a CUDA device; none is available")
    name, limit = gpu_info()
    print(f"# {name}, power limit {limit}, SM clock (current, max) {sm_clock()}", flush=True)
    kernels(args, name, limit)
    cycles(args, name, limit)


if __name__ == "__main__":
    main()
