"""Time of the exact reductions (sb_reduce_exact_*) on one GPU, against the ordered plan and a copy on the same buffers.

    python scripts/time_reduce_exact.py [--iters 50] [--warmup 5]

512^3 FP64, radius 1.  Workloads: (a) SCALAR of 3 N(0,1) data; (b) DIFF of two such fields; (c) NORM3 of three;
(d) SCALAR of data whose exponents spread over the whole FP64 range (the path through the shared accumulator); then
(a) and (c) again on 512^3 FP32 fields: the same per-cell work over half the bytes, which tells a kernel bound by
arithmetic (about the same time as FP64) from one bound by bytes (about half).  Each
launch of the exact plan alternates with a launch of the ordered plan over the same items and with dst.copy_(src) of
one source field (the copy ceiling); each timing is the trimean of --iters CUDA-event timings after --warmup untimed
rounds.  Prints one JSON line per workload with the GPU's name and power limit."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    import stencil_b200 as sb

    if not torch.cuda.is_available():
        raise SystemExit("time_reduce_exact.py needs a CUDA device")
    name, limit = gpu_info()
    for dtype in (np.float64, np.float32):
        run_dtype(sb, torch, dtype, name, limit, args)


def run_dtype(sb, torch, dtype, name, limit, args):
    n = 512
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(1)
    hs = [dd.add_data(dtype) for _ in range(3)]
    dd.realize()
    d = dd.domains()[0]
    rng = np.random.default_rng(1)
    for q in range(3):
        for which in ("curr", "next"):
            d.quantity_from_host(q, (rng.standard_normal(d.raw_size()[::-1]) * 3.0).astype(dtype), which)
    src = torch.empty(n**3, dtype=torch.float64 if dtype == np.float64 else torch.float32, device="cuda")
    dst = torch.empty_like(src)
    s = torch.cuda.Stream()
    work = [("a SCALAR 3N(0,1)", [("scalar", hs[0])]), ("b DIFF", [("diff", hs[0])]), ("c NORM3", [("norm", hs[0], hs[1], hs[2])]),
            ("d SCALAR, exponents over the whole range", [("scalar", hs[0], "next")])]  # fmt: skip
    if dtype == np.float32:
        work = [work[0], work[2]]
    tag = "FP64" if dtype == np.float64 else "FP32"
    for label, items in work:
        if label.startswith("d"):
            raw = d.raw_size()[::-1]
            x = rng.standard_normal(raw) * np.ldexp(1.0, rng.integers(-1074, 1000, raw))
            d.quantity_from_host(0, x, "next")
        xplan, plan = dd.reduce_plans(items, exact=True)[0], dd.reduce_plans(items)[0]
        tx, tp, tc = [], [], []
        with torch.cuda.stream(s):
            for it in range(args.warmup + args.iters):
                a = timed(s, lambda: xplan.launch(s))
                b = timed(s, lambda: plan.launch(s))
                c = timed(s, lambda: dst.copy_(src))
                if it >= args.warmup:
                    tx.append(a)
                    tp.append(b)
                    tc.append(c)
        t_x, t_p, t_c = trimean(tx), trimean(tp), trimean(tc)
        print(json.dumps(dict(workload=f"512^3 {tag} {label}", gpu=name, power_limit=limit, iters=args.iters, bytes_read=int(xplan.bytes),
                              exact_ms=round(t_x, 4), ordered_ms=round(t_p, 4), exact_over_ordered=round(t_x / t_p, 3),
                              copy_ms_per_field=round(t_c, 4), exact_GBps=round(xplan.bytes / (t_x * 1e-3) / 1e9, 1))), flush=True)
    dd.close()
    torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
