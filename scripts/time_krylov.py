"""Time of the Krylov vector kernels (sb_krylov_plan_*) and of the Python PCG iteration on one GPU.

    python scripts/time_krylov.py [--iters 30] [--warmup 5] [--pcg-iters 10]

512^3, radius 1.  Workloads, each launch alternated with dst.copy_(src) of one field (the copy ceiling):
  (a) UPDATE x += T(s) p, r -= T(s) q with <r, r>, FP64 and FP32, against the unfused sequence: two torch in-place
      axpys on tensors of the same size plus the exact SCALAR reduction of r;
  (b) the two-pair DOT <z, r>, <z, q> against two one-pair DOT launches, and the one-pair DOT against the exact SCALAR
      reduction of one field, FP64 and FP32.
Then one PCG iteration of 256^3 -lap x = f (ODD(0) walls, V(2,2) to 4^3) from Python, FP64 and FP32, against the cycle
of its preconditioner, and with gamma and delta taken the other way (one two-pair DOT or two one-pair DOTs),
alternated (median of 3).  Each kernel timing is the trimean of --iters CUDA-event timings after --warmup untimed
rounds.  Prints one JSON line per workload with the GPU's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_boundary import gpu_info, timed, trimean  # noqa: E402


def alternate(torch, s, fns, args):
    """Trimean of each fn's CUDA-event time, the fns alternated round by round."""
    ts = [[] for _ in fns]
    with torch.cuda.stream(s):
        for it in range(args.warmup + args.iters):
            for t, fn in zip(ts, fns):
                v = timed(s, fn)
                if it >= args.warmup:
                    t.append(v)
    return [trimean(t) for t in ts]


def kernels(sb, torch, dtype, name, limit, args):
    n = 512
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(1)
    x, p, r, q, z = (dd.add_data(dtype, k) for k in "xprqz")
    dd.realize()
    d = dd.domains()[0]
    rng = np.random.default_rng(1)
    for h in (x, p, r, q, z):
        d.quantity_from_host(h.id, rng.standard_normal(d.raw_size()[::-1]).astype(dtype))
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    src = torch.randn(n**3, dtype=tdt, device="cuda")
    dst = torch.empty_like(src)
    tx, tp, tr, tq = (torch.randn(n**3, dtype=tdt, device="cuda") for _ in range(4))
    s = torch.cuda.Stream()
    tag = "FP64" if dtype == np.float64 else "FP32"
    es = np.dtype(dtype).itemsize
    copy = lambda: dst.copy_(src)  # noqa: E731
    K = sb._lib
    up = dd.krylov_plans(K.KRYLOV_UPDATE, (x, p, r, q))[0]
    up.s = 1e-3  # a small step keeps the data in range over many launches
    red = dd.reduce_plans([("scalar", r)], exact=True)[0]

    def unfused():
        tx.add_(tp, alpha=1e-3)
        tr.add_(tq, alpha=-1e-3)
        red.launch(s)

    t_up, t_un, t_c = alternate(torch, s, [lambda: up.launch(s), unfused, copy], args)
    print(json.dumps(dict(workload=f"(a) 512^3 {tag} UPDATE with <r, r>", gpu=name, power_limit=limit, iters=args.iters, update_ms=round(t_up, 4),
                          unfused_ms=round(t_un, 4), update_over_unfused=round(t_up / t_un, 3), copy_ms_per_field=round(t_c, 4),
                          update_GBps=round(up.bytes / (t_up * 1e-3) / 1e9, 1), copy_GBps=round(2 * n**3 * es / (t_c * 1e-3) / 1e9, 1))), flush=True)
    d2 = dd.krylov_plans(K.KRYLOV_DOT, (z, r, q))[0]
    d1a, d1b = dd.krylov_plans(K.KRYLOV_DOT, (z, r))[0], dd.krylov_plans(K.KRYLOV_DOT, (z, q))[0]
    rz = dd.reduce_plans([("scalar", z)], exact=True)[0]

    def two_one_pair():
        d1a.launch(s)
        d1b.launch(s)

    t2, t11, t1, tred, t_c = alternate(torch, s, [lambda: d2.launch(s), two_one_pair, lambda: d1a.launch(s), lambda: rz.launch(s), copy], args)
    print(json.dumps(dict(workload=f"(b) 512^3 {tag} DOT", gpu=name, power_limit=limit, iters=args.iters, two_pair_ms=round(t2, 4),
                          two_one_pair_ms=round(t11, 4), two_pair_over_two_one_pair=round(t2 / t11, 3), one_pair_ms=round(t1, 4),
                          exact_scalar_reduce_ms=round(tred, 4), one_pair_over_reduce=round(t1 / tred, 3), copy_ms_per_field=round(t_c, 4),
                          two_pair_GBps=round(d2.bytes / (t2 * 1e-3) / 1e9, 1))), flush=True)
    dd.close()
    del src, dst, tx, tp, tr, tq
    torch.cuda.empty_cache()


def pcg_iteration(sb, torch, dtype, name, limit, args):
    n = 256
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(1)
    x, f, r, z, p, q = (dd.add_data(dtype, k) for k in "xfrzpq")
    dd.set_boundary(sb.Boundary.FIXED)
    for fc in sb.FACES:
        for h in (x, z, p):
            dd.set_boundary_condition(h, fc, sb.BC.ODD(0.0))
    dd.realize()
    d = dd.domains()[0]
    d.quantity_from_host(f.id, np.random.default_rng(2).uniform(-1, 1, d.raw_size()[::-1]).astype(dtype))
    zero = np.zeros(d.raw_size()[::-1], dtype)

    def A_at(l):
        return sb.StencilOp.laplacian(2, (2.0**l / n,) * 3, dtype).scaled(-1.0)

    cg = sb.PCG(dd, x, f, r, z, p, q, A_at)
    tag = "FP64" if dtype == np.float64 else "FP32"

    def per_iteration():
        d.quantity_from_host(x.id, zero)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        cg.solve(0.0, 0)
        t_start = time.perf_counter() - t0
        d.quantity_from_host(x.id, zero)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hist = cg.solve(0.0, args.pcg_iters)
        return (time.perf_counter() - t0 - t_start) / args.pcg_iters, hist

    cg.solve(0.0, 2)  # warm-up: plans, events, first launches
    # gamma and delta by one two-pair DOT (the FP64 choice) or two one-pair DOTs (the FP32 choice), alternated
    default = cg._split_gamma_delta
    t_it, t_alt = [], []
    for _ in range(3):
        cg._split_gamma_delta = default
        t, hist = per_iteration()
        t_it.append(t)
        cg._split_gamma_delta = not default
        t_alt.append(per_iteration()[0])
    cg._split_gamma_delta = default
    t_it, t_alt = float(np.median(t_it)), float(np.median(t_alt))
    t0 = time.perf_counter()
    for _ in range(args.pcg_iters):
        cg.mg.cycle()
    t_cyc = (time.perf_counter() - t0) / args.pcg_iters
    print(json.dumps(dict(workload=f"256^3 {tag} -lap x = f, ODD(0) walls, V(2,2) to 4^3: stencil_b200.PCG iteration vs its preconditioner's cycle()",
                          gpu=name, power_limit=limit, gamma_delta="two one-pair DOTs" if default else "one two-pair DOT",
                          ms_per_iteration=round(t_it * 1e3, 2), ms_per_iteration_other_gamma_delta=round(t_alt * 1e3, 2),
                          ms_per_vcycle=round(t_cyc * 1e3, 2), ratio=round(t_it / t_cyc, 3),
                          factor_per_iteration=round((hist[-1] / hist[0]) ** (1.0 / args.pcg_iters), 4))), flush=True)
    cg.close()
    dd.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--pcg-iters", type=int, default=10)
    args = ap.parse_args()
    import torch

    import stencil_b200 as sb

    if not torch.cuda.is_available():
        raise SystemExit("time_krylov.py needs a CUDA device")
    name, limit = gpu_info()
    for dtype in (np.float64, np.float32):
        kernels(sb, torch, dtype, name, limit, args)
    for dtype in (np.float64, np.float32):
        pcg_iteration(sb, torch, dtype, name, limit, args)


if __name__ == "__main__":
    main()
