"""Cost of boundary conditions on one GPU: a periodic exchange (a) against the same grid with walls on every axis and
ODD(0.5) on every face (b).  On one subdomain (a) is the copy engine's self-wrap copies of the ghost shell and (b) is the
boundary-condition kernel writing the same ghost cells from the same number of source cells, so the two compare the new
kernel with the copy engine like for like.

    python scripts/time_boundary.py [--iters 30] [--warmup 5] [--periodic-only]

Shapes: the jacobi shape (512^3 FP64, faces r=1) and the bench_exchange shape (512^3, 3 x float, r=2).  Each timing is
the trimean of --iters exchanges timed one by one with CUDA events on the exchange stream, (a) and (b) alternating.  The
BC launch is also timed alone; its rate counts one read and one write per ghost cell it writes.  Prints one JSON line per
shape, with the GPU's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def trimean(v):
    q1, q2, q3 = np.percentile(np.asarray(v, dtype=np.float64), [25, 50, 75])
    return float((q1 + 2 * q2 + q3) / 4)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, limit = [s.strip() for s in out.stdout.strip().split(",")[:2]]
        return name, limit
    except Exception:
        import torch

        return torch.cuda.get_device_name(0), "unknown"


def make_domain(sb, n, radius, dtypes, walls):
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(radius)
    hs = [dd.add_data(dt) for dt in dtypes]
    if walls:
        dd.set_boundary(sb.Boundary.FIXED)
        for h in hs:
            for f in sb.FACES:
                dd.set_boundary_condition(h, f, sb.BC.ODD(0.5))
    dd.realize()
    for d in dd.domains():
        for q in range(len(dtypes)):
            d.quantity_from_host(q, np.random.default_rng(q).uniform(-1, 1, d.raw_size()[::-1]).astype(dtypes[q]))
    return dd


def timed(stream, fn):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    fn()
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--periodic-only", action="store_true", help="time (a) only (runs with libraries that lack boundary conditions)")
    args = ap.parse_args()
    import torch

    import stencil_b200 as sb

    if not torch.cuda.is_available():
        raise SystemExit("time_boundary.py needs a CUDA device")
    name, limit = gpu_info()
    shapes = [
        ("jacobi 512^3 FP64 faces r=1", 512, sb.Radius.face_edge_corner(1, 0, 0), [np.float64]),
        ("bench_exchange 512^3 3xf32 r=2", 512, sb.Radius.constant(2), [np.float32] * 3),
    ]
    for label, n, radius, dtypes in shapes:
        per = make_domain(sb, n, radius, dtypes, False)
        wal = None if args.periodic_only else make_domain(sb, n, radius, dtypes, True)
        sp = per.exchange_streams()[0]
        ta, tb, tbc = [], [], []
        for it in range(args.warmup + args.iters):
            t = timed(sp, per.exchange_async)
            if it >= args.warmup:
                ta.append(t)
            if wal is not None:
                sw = wal.exchange_streams()[0]
                t = timed(sw, wal.exchange_async)
                bc = wal._bc_plans[wal._parity][0]
                tl = timed(sw, lambda: bc.launch(sw))
                if it >= args.warmup:
                    tb.append(t)
                    tbc.append(tl)
        rec = dict(shape=label, gpu=name, power_limit=limit, iters=args.iters, periodic_ms=round(trimean(ta), 4),
                   periodic_bytes=int(per._plans[0][0].bytes))
        if wal is not None:
            bc_bytes = wal._bc_plans[0][0].bytes
            t_bc = trimean(tbc)
            rec.update(walled_ms=round(trimean(tb), 4), ratio=round(trimean(tb) / trimean(ta), 3), bc_launch_ms=round(t_bc, 4),
                       bc_bytes_written=int(bc_bytes), bc_GBps=round(2 * bc_bytes / (t_bc * 1e-3) / 1e9, 1))
        print(json.dumps(rec), flush=True)
        per.close()
        if wal is not None:
            wal.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
