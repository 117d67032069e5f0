"""Exchanges of a quantity subset against full exchanges (DESIGN.md section 2.15), on the GPU, one JSON line per
workload, with the card's name and power limit read in the same run.

exchange: the bench_exchange shape (512^3 total, radius 2, 3 x float32) on 1, 2 and 4 subdomains of GPU 0 (and on all
GPUs where there are several): dd.exchange() against dd.exchange(only=[one quantity]), alternated, each with the
payload bytes of its copy plans (exchange_bytes).
solvers: one stencil_b200.PCG iteration and one Multigrid.cycle() on 256^3 FP64 -div(kappa grad x) = f with a 10^3
jump in kappa, on 1 and 4 subdomains.  "full" runs every exchange of the solver over every quantity (the behaviour
before subset exchanges, restored for the measurement by making every read set the full set), "subset" the solver as
it is; the two are alternated in one process.
usage: time_exchange_subset.py [--reps N] [--iters K]"""
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

from time_boundary import gpu_info, trimean  # noqa: E402


def exchange_times(sb, torch, gpus, args, name, limit):
    dd = sb.DistributedDomain(512, 512, 512)
    dd.set_gpus(gpus)
    dd.set_radius(2)
    hs = [dd.add_data(np.float32, f"q{i}") for i in range(3)]
    dd.realize()
    ways = {"full": None, "one quantity": [hs[0]]}
    for only in ways.values():
        for _ in range(5):
            dd.exchange(only=only)
    ts = {k: [] for k in ways}
    for _ in range(args.reps):
        for k, only in ways.items():
            for d in dd.domains():
                torch.cuda.synchronize(d.gpu())
            t0 = time.perf_counter()
            dd.exchange(only=only)
            ts[k].append(time.perf_counter() - t0)
    out = dict(workload=f"exchange 512^3 r2 3 x float32, {len(gpus)} subdomains on GPUs {sorted(set(gpus))}", gpu=name, power_limit=limit)
    for k, only in ways.items():
        out[k] = dict(us=round(trimean(ts[k]) * 1e6, 1), bytes=dd.exchange_bytes(only))
    out["time_ratio"] = round(out["one quantity"]["us"] / out["full"]["us"], 3)
    out["bytes_ratio"] = round(out["one quantity"]["bytes"] / max(out["full"]["bytes"], 1), 3)
    print(json.dumps(out), flush=True)
    dd.close()


def solver_times(sb, torch, ndom, args, name, limit):
    n = 256
    dtype = np.float64
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0] * ndom)
    dd.set_radius(1)
    x, f, r, z, p, q = (dd.add_data(dtype, k) for k in "xfrzpq")
    ks = [dd.add_data(dtype, k) for k in ("kx", "ky", "kz")]
    dd.set_boundary(sb.Boundary.FIXED)
    for fc in sb.FACES:
        for h in (x, z, p):
            dd.set_boundary_condition(h, fc, sb.BC.ODD(0.0))
        for h in ks:
            dd.set_boundary_condition(h, fc, sb.BC.EVEN())
    dd.realize()
    rng = np.random.default_rng(2)
    for d in dd.domains():
        raw, org, sz = d.raw_size(), d.origin(), d.size()
        d.quantity_from_host(f.id, rng.uniform(-1, 1, raw[::-1]))
        xs = org[0] - 1 + np.arange(raw[0])  # a 10^3 jump in kappa across the plane x = n / 2
        kap = np.broadcast_to(np.where(xs < n // 2, 1.0, 1000.0), raw[::-1]).copy()
        for h in ks:
            d.quantity_from_host(h.id, kap)
    A_at = lambda l: sb.StencilOp.div_grad((2.0**l / n,) * 3, dtype).scaled(-1.0)  # noqa: E731
    cg = sb.PCG(dd, x, f, r, z, p, q, A_at, coefs=ks)
    zero = [np.zeros(d.raw_size()[::-1], dtype) for d in dd.domains()]
    subset_sel = sb.DistributedDomain._exchange_sel

    def full_sel(self, name, exchange, reads):
        v = subset_sel(self, name, exchange, reads)
        return True if isinstance(v, tuple) else v

    def reset():
        for d, z0 in zip(dd.domains(), zero):
            d.quantity_from_host(x.id, z0)
        torch.cuda.synchronize()

    def pcg_iteration():
        reset()
        t0 = time.perf_counter()
        cg.solve(0.0, 0)
        t_start = time.perf_counter() - t0
        reset()
        t0 = time.perf_counter()
        cg.solve(0.0, args.iters)
        return (time.perf_counter() - t0 - t_start) / args.iters

    def cycle():
        t0 = time.perf_counter()
        for _ in range(args.iters):
            cg.mg.cycle()
        return (time.perf_counter() - t0) / args.iters

    ways = {"full": full_sel, "subset": subset_sel}
    ts = {(k, w): [] for k in ways for w in ("pcg", "cycle")}
    try:
        for sel in ways.values():  # warm-up: plans, events, first launches
            sb.DistributedDomain._exchange_sel = sel
            cg.solve(0.0, 2)
            cg.mg.cycle()
        for _ in range(3):
            for k, sel in ways.items():
                sb.DistributedDomain._exchange_sel = sel
                ts[(k, "pcg")].append(pcg_iteration())
                ts[(k, "cycle")].append(cycle())
    finally:
        sb.DistributedDomain._exchange_sel = subset_sel
    bytes_full = dd.exchange_bytes()
    bytes_one = dd.exchange_bytes([p])
    out = dict(workload=f"256^3 FP64 -div(kappa grad x) = f, 10^3 jump, {ndom} subdomains of GPU 0", gpu=name, power_limit=limit,
               exchange_bytes_full=bytes_full, exchange_bytes_one_vector=bytes_one, bytes_ratio=round(bytes_one / max(bytes_full, 1), 3))
    for k in ways:
        out[f"pcg_ms_{k}"] = round(float(np.median(ts[(k, "pcg")])) * 1e3, 2)
        out[f"cycle_ms_{k}"] = round(float(np.median(ts[(k, "cycle")])) * 1e3, 2)
    print(json.dumps(out), flush=True)
    cg.close()
    dd.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch

    import stencil_b200 as sb

    if not torch.cuda.is_available():
        raise SystemExit("time_exchange_subset.py needs a CUDA device")
    name, limit = gpu_info()
    layouts = [[0], [0, 0], [0, 0, 0, 0]]
    if torch.cuda.device_count() > 1:
        layouts.append(list(range(torch.cuda.device_count())))
    for gpus in layouts:
        exchange_times(sb, torch, gpus, args, name, limit)
    for ndom in (1, 4):
        solver_times(sb, torch, ndom, args, name, limit)


if __name__ == "__main__":
    main()
