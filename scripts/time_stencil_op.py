"""Rate of the linear stencil operator kernels on one GPU: algorithmic bytes (sb_stencil_plan_bytes: per cell one element
read of src, one of aux if present, one written) over kernel time.

    python scripts/time_stencil_op.py [--iters 50] [--warmup 5]

Workloads, each over the whole 512^3 compute region of one subdomain (one tile-kernel launch): FP64 7-point Laplacian,
FP64 order-8 Laplacian, FP64 27-point box, FP32 7-point Laplacian.  The FP64 7-point op is alternated launch by launch
with sb_jacobi3d over the same region (the fused jacobi kernel's step without the exchange), and its rate is reported as
a share of that kernel's.  Each timing is the trimean of --iters launches timed one by one with CUDA events on one stream,
after --warmup untimed launches.  Prints one JSON line per workload with the GPU's name and power limit and the share of
the H100 SXM data-sheet bandwidth (3.35 TB/s)."""
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
N = 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import stencil_b200 as sb
    from stencil_b200._lib import Pitched, check, i3, lib, stream_ptr

    if not torch.cuda.is_available():
        raise SystemExit("time_stencil_op.py needs a CUDA device")
    name, limit = gpu_info()
    s = torch.cuda.Stream()
    rng = np.random.default_rng(1)
    box27 = [(0, (x, y, z), float(rng.uniform(-1, 1))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1)]
    work = [
        ("512^3 FP64 7-point", np.float64, sb.Radius.face_edge_corner(1, 0, 0), lambda dt: sb.StencilOp.laplacian(2, (1, 1, 1), dt), True),
        ("512^3 FP64 order-8 Laplacian", np.float64, sb.Radius.face_edge_corner(4, 0, 0), lambda dt: sb.StencilOp.laplacian(8, (1, 1, 1), dt), False),
        ("512^3 FP64 27-point box", np.float64, sb.Radius.constant(1), lambda dt: sb.StencilOp(box27, dt), False),
        ("512^3 FP32 7-point", np.float32, sb.Radius.face_edge_corner(1, 0, 0), lambda dt: sb.StencilOp.laplacian(2, (1, 1, 1), dt), False),
    ]
    for label, dtype, radius, mk, vs_jacobi in work:
        dd = sb.DistributedDomain(N, N, N)
        dd.set_gpus([0])
        dd.set_radius(radius)
        h = dd.add_data(dtype)
        dd.realize()
        d = dd.domains()[0]
        for which in ("curr", "next"):
            d.quantity_from_host(h.id, rng.uniform(-1, 1, d.raw_size()[::-1]).astype(dtype), which)
        op = mk(dtype)
        lo, hi = d.get_compute_region()
        plan = sb.StencilPlan(d.gpu(), op, d.next_data(h.id), d.curr_data(h.id), Pitched(None, 0, 0), d.accessor_origin(), d.raw_size()[2], [(lo, hi)])
        rec = dict(workload=label, gpu=name, power_limit=limit, iters=args.iters, terms=len(op.terms), bytes=int(plan.bytes))
        to, tj = [], []
        jac = (d.next_data(h.id), d.curr_data(h.id), d.elem_size(h.id), i3(d.accessor_origin()), i3(lo), i3(hi), i3(lo), i3(hi), stream_ptr(s))
        for it in range(args.warmup + args.iters):
            a = timed(s, lambda: plan.launch(s))
            if it >= args.warmup:
                to.append(a)
            if vs_jacobi:
                b = timed(s, lambda: check(lib().sb_jacobi3d(*jac)))
                if it >= args.warmup:
                    tj.append(b)
        t = trimean(to)
        gbps = plan.bytes / (t * 1e-3) / 1e9
        rec.update(kernel_ms=round(t, 4), GBps=round(gbps, 1), share_of_3_35TBps=round(gbps * 1e9 / PEAK, 3))
        if vs_jacobi:
            tjm = trimean(tj)
            jbytes = N**3 * 2 * np.dtype(dtype).itemsize
            rec.update(jacobi_ms=round(tjm, 4), jacobi_GBps=round(jbytes / (tjm * 1e-3) / 1e9, 1), op_rate_over_jacobi=round((plan.bytes / t) / (jbytes / tjm), 3))
        print(json.dumps(rec), flush=True)
        plan.destroy()
        dd.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
