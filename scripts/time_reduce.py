"""Rate of the reduction kernels on one GPU: bytes read (sb_reduce_plan_bytes) over kernel time.

    python scripts/time_reduce.py [--iters 50] [--warmup 5]

Workloads: (a) 512^3 FP64 SCALAR; (b) 512^3 FP64 DIFF, alternated launch by launch with sb_sqdiff over the same two
buffers (the residual the benchmark computes); (c) the astaroth diagnostics on 256^3 FP64 (8 SCALAR + 2 NORM3 items,
one plan).  Each timing is the trimean of --iters launches timed one by one with CUDA events on one stream, after
--warmup untimed launches.  Prints one JSON line per workload, with the GPU's name and power limit and the share of the
H100 SXM data-sheet bandwidth (3.35 TB/s)."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_boundary import gpu_info, timed, trimean  # noqa: E402

PEAK = 3.35e12


def domain(sb, n, radius, nq):
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(radius)
    hs = [dd.add_data(np.float64) for _ in range(nq)]
    dd.realize()
    rng = np.random.default_rng(1)
    for d in dd.domains():
        for q in range(nq):
            for which in ("curr", "next"):
                d.quantity_from_host(q, rng.uniform(-1, 1, d.raw_size()[::-1]), which)
    return dd, hs


def plan_for(sb, dd, items):
    return dd.reduce_plans(items)[0]


def record(label, name, limit, iters, plan, t_ms, **extra):
    gbps = plan.bytes / (t_ms * 1e-3) / 1e9
    rec = dict(workload=label, gpu=name, power_limit=limit, iters=iters, bytes_read=int(plan.bytes), kernel_ms=round(t_ms, 4),
               GBps=round(gbps, 1), share_of_3_35TBps=round(gbps * 1e9 / PEAK, 3))
    rec.update(extra)
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import ctypes as C

    import torch

    import stencil_b200 as sb
    from stencil_b200._lib import check, i3, lib, stream_ptr

    if not torch.cuda.is_available():
        raise SystemExit("time_reduce.py needs a CUDA device")
    name, limit = gpu_info()
    dd, hs = domain(sb, 512, 1, 1)
    s = torch.cuda.Stream()
    # (a) SCALAR
    plan = plan_for(sb, dd, [("scalar", hs[0])])
    ts = [timed(s, lambda: plan.launch(s)) for _ in range(args.warmup + args.iters)][args.warmup :]
    record("512^3 FP64 SCALAR", name, limit, args.iters, plan, trimean(ts))
    # (b) DIFF against sb_sqdiff, alternating
    plan = plan_for(sb, dd, [("diff", hs[0])])
    d = dd.domains()[0]
    lo, hi = d.get_compute_region()
    out = torch.zeros(1, dtype=torch.float64, device="cuda")
    sq_args = (d.curr_data(0), d.next_data(0), 8, i3(d.accessor_origin()), i3(lo), i3(hi), C.c_void_p(out.data_ptr()), stream_ptr(s))
    td_, tq = [], []
    for it in range(args.warmup + args.iters):
        a = timed(s, lambda: plan.launch(s))
        b = timed(s, lambda: check(lib().sb_sqdiff(*sq_args)))
        if it >= args.warmup:
            td_.append(a)
            tq.append(b)
    t_sq = trimean(tq)
    record("512^3 FP64 DIFF", name, limit, args.iters, plan, trimean(td_), sqdiff_ms=round(t_sq, 4),
           sqdiff_GBps=round(plan.bytes / (t_sq * 1e-3) / 1e9, 1))
    dd.close()
    torch.cuda.empty_cache()
    # (c) astaroth diagnostics, 256^3 FP64, radius 3
    from stencil_b200.astaroth import FIELDS

    dd, hs = domain(sb, 256, 3, len(FIELDS))
    items = [("scalar", h) for h in hs] + [("norm", hs[1], hs[2], hs[3]), ("norm", hs[4], hs[5], hs[6])]
    plan = plan_for(sb, dd, items)
    ts = [timed(s, lambda: plan.launch(s)) for _ in range(args.warmup + args.iters)][args.warmup :]
    record("astaroth 256^3 FP64 diagnostics (10 items)", name, limit, args.iters, plan, trimean(ts))
    dd.close()


if __name__ == "__main__":
    main()
