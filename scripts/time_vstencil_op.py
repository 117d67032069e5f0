"""Rate of the variable-coefficient stencil operator kernels on one GPU, against the plain FP64 7-point op and the copy
ceiling measured in the same run.

    python scripts/time_vstencil_op.py [--iters 50] [--warmup 5]

Workloads, each over the whole 512^3 compute region of one subdomain (one tile-kernel launch):
  * FP64 and FP32 heat step u + dt div(kappa grad u): 13 terms, 3 coefficient fields (kappa on the x / y / z faces),
    algorithmic bytes 5 elements per cell (u, three kappas, dst: 40 B at FP64);
  * FP64 c^2(x) lap4(u): 13 terms, one coefficient field read at offset 0 (24 B per cell).
Each launch is alternated with a launch of the plain FP64 7-point op (16 B per cell) and with dst.copy_(src) over two
514^3 FP64 buffers (the copy ceiling, bytes = read + write, as scripts/time_jacobi_feed.py measures it).  Every timing is
the trimean of --iters launches timed one by one with CUDA events on one stream, after --warmup untimed launches.  Prints
one JSON line per workload with the GPU's name and power limit, the algorithmic bytes (sb_stencil_plan_bytes), and each
rate as a share of the copy ceiling."""
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

N = 512


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import torch

    import stencil_b200 as sb
    from stencil_b200._lib import Pitched

    if not torch.cuda.is_available():
        raise SystemExit("time_vstencil_op.py needs a CUDA device")
    name, limit = gpu_info()
    s = torch.cuda.Stream()
    rng = np.random.default_rng(1)

    def heat(dt):
        kdt = sb.StencilOp.div_grad((1.0, 1.0, 1.0), dt).scaled(0.1)
        return sb.StencilOp(list(kdt.terms) + [(0, (0, 0, 0), 1.0)], dt)

    def c2lap4(dt):
        return sb.StencilOp([(0, o, w, 0, (0, 0, 0)) for _, o, w in sb.StencilOp.laplacian(4, (1, 1, 1), dt).terms], dt)

    work = [
        ("512^3 FP64 div(kappa grad u) heat step", np.float64, sb.Radius.face_edge_corner(1, 0, 0), heat),
        ("512^3 FP32 div(kappa grad u) heat step", np.float32, sb.Radius.face_edge_corner(1, 0, 0), heat),
        ("512^3 FP64 c^2 lap4", np.float64, sb.Radius.face_edge_corner(2, 0, 0), c2lap4),
    ]
    cn = N + 2
    csrc = torch.rand(cn, cn, cn, dtype=torch.float64, device="cuda")
    cdst = torch.empty_like(csrc)
    cbytes = 2 * csrc.numel() * 8
    for label, dtype, radius, mk in work:
        dd = sb.DistributedDomain(N, N, N)
        dd.set_gpus([0])
        dd.set_radius(radius)
        op = mk(dtype)
        h = dd.add_data(dtype)
        ks = [dd.add_data(dtype) for _ in range(op.ncoef)]
        p7 = dd.add_data(np.float64)
        dd.realize()
        d = dd.domains()[0]
        for q, low in [(h, -1.0), (p7, -1.0)] + [(k, 0.5) for k in ks]:
            for which in ("curr", "next"):
                d.quantity_from_host(q.id, rng.uniform(low, 1, d.raw_size()[::-1]).astype(dd.dtypes_[q.id]), which)
        lo, hi = d.get_compute_region()
        plan = sb.StencilPlan(d.gpu(), op, d.next_data(h.id), d.curr_data(h.id), Pitched(None, 0, 0), d.accessor_origin(), d.raw_size()[2],
                              [(lo, hi)], [d.curr_data(k.id) for k in ks])
        lap = sb.StencilOp.laplacian(2, (1, 1, 1), np.float64)
        plain = sb.StencilPlan(d.gpu(), lap, d.next_data(p7.id), d.curr_data(p7.id), Pitched(None, 0, 0), d.accessor_origin(), d.raw_size()[2],
                               [(lo, hi)])
        tv, tp, tc = [], [], []
        for it in range(args.warmup + args.iters):
            a = timed(s, lambda: plan.launch(s))
            b = timed(s, lambda: plain.launch(s))
            with torch.cuda.stream(s):
                c = timed(s, lambda: cdst.copy_(csrc))
            if it >= args.warmup:
                tv.append(a)
                tp.append(b)
                tc.append(c)
        t, t7, tcp = trimean(tv), trimean(tp), trimean(tc)
        ceil = cbytes / (tcp * 1e-3)
        rate, rate7 = plan.bytes / (t * 1e-3), plain.bytes / (t7 * 1e-3)
        rec = dict(workload=label, gpu=name, power_limit=limit, iters=args.iters, terms=len(op.terms), coef_fields=op.ncoef,
                   bytes=int(plan.bytes), bytes_per_cell=int(plan.bytes) // N**3, kernel_ms=round(t, 4), GBps=round(rate / 1e9, 1),
                   share_of_copy_ceiling=round(rate / ceil, 3), plain7_ms=round(t7, 4), plain7_GBps=round(rate7 / 1e9, 1),
                   plain7_share_of_copy_ceiling=round(rate7 / ceil, 3), rate_over_plain7=round(rate / rate7, 3), copy_ms=round(tcp, 4),
                   copy_ceiling_GBps=round(ceil / 1e9, 1))
        print(json.dumps(rec), flush=True)
        plan.destroy()
        plain.destroy()
        dd.close()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
