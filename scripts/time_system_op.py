"""Rate of the linear stencil system kernels on one GPU, against the plain FP64 7-point op, the copy ceiling and the same
update written with torch tensor ops, all measured in the same run.

    python scripts/time_system_op.py [--iters 40] [--warmup 5]

Workloads, each over a 512^3 FP64 compute region in 514^3 allocations (one tile-kernel launch):
  (a) forward curl, 3 -> 3: 12 terms, 48 B per cell;
  (b) Yee E update in place, E = E + (dt / eps) curl- H: inputs 3 x H and 3 x E, outputs E; 15 terms, 72 B per cell;
  (c) forward grad, 1 -> 3: 6 terms, 32 B per cell.
Each launch is alternated with dst.copy_(src) over two 514^3 FP64 buffers (the copy ceiling, bytes = read + write), a
launch of the plain FP64 7-point op (16 B per cell) and the torch version of the workload on the same allocations.
Every timing is the trimean of --iters runs timed one by one with CUDA events on one stream, after --warmup untimed runs.
Prints the GPU's name, power limit and SM clock, then one JSON line per workload."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_boundary import gpu_info, timed, trimean  # noqa: E402

N = 512
H = (1.0, 0.9, 1.1)


def sm_clock() -> str:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip()
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()

    import numpy as np
    import torch

    import stencil_b200 as sb
    from stencil_b200._lib import Pitched

    if not torch.cuda.is_available():
        raise SystemExit("time_system_op.py needs a CUDA device")
    name, limit = gpu_info()
    s = torch.cuda.Stream()
    m = N + 2
    lo, hi = (1, 1, 1), (1 + N, 1 + N, 1 + N)
    I = slice(1, N + 1)

    def new():
        return torch.rand(m, m, m, dtype=torch.float64, device="cuda")

    def pitched(t):
        return Pitched(t.data_ptr(), m * 8, m)

    def at(t, o):
        """The interior of t shifted by o = (dx, dy, dz)."""
        return t[1 + o[2] : N + 1 + o[2], 1 + o[1] : N + 1 + o[1], 1 + o[0] : N + 1 + o[0]]

    def e(a, k):
        return tuple(k if b == a else 0 for b in range(3))

    def d_fwd(t, a):
        return (at(t, e(a, 1)) - at(t, (0, 0, 0))) * (1.0 / H[a])

    def d_bwd(t, a):
        return (at(t, (0, 0, 0)) - at(t, e(a, -1))) * (1.0 / H[a])

    c = 0.3
    curl_sys = sb.StencilSystem.curl(1, H, np.float64)
    ident = sb.StencilSystem([(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)], np.float64, nin=6)
    yee_sys = ident + sb.StencilSystem.curl(-1, H, np.float64).scaled(c)
    grad_sys = sb.StencilSystem.grad(1, H, np.float64)

    def curl_torch(ins, outs):
        for j in range(3):
            a, b = (j + 1) % 3, (j + 2) % 3
            outs[j][I, I, I] = d_fwd(ins[b], a) - d_fwd(ins[a], b)

    def yee_torch(ins, outs):
        for j in range(3):
            a, b = (j + 1) % 3, (j + 2) % 3
            outs[j][I, I, I] += c * (d_bwd(ins[b], a) - d_bwd(ins[a], b))

    def grad_torch(ins, outs):
        for j in range(3):
            outs[j][I, I, I] = d_fwd(ins[0], j)

    work = [
        ("(a) 512^3 FP64 forward curl, 3 -> 3", curl_sys, 3, None, curl_torch),
        ("(b) 512^3 FP64 Yee E update in place, E = E + (dt/eps) curl- H", yee_sys, 6, [3, 4, 5], yee_torch),
        ("(c) 512^3 FP64 forward grad, 1 -> 3", grad_sys, 1, None, grad_torch),
    ]
    print(json.dumps(dict(gpu=name, power_limit=limit, sm_clock_now_and_max=sm_clock())), flush=True)
    csrc, cdst = new(), torch.empty(m, m, m, dtype=torch.float64, device="cuda")
    cbytes = 2 * csrc.numel() * 8
    p_src, p_dst = new(), new()
    plain = sb.StencilPlan(0, sb.StencilOp.laplacian(2, (1, 1, 1), np.float64), pitched(p_dst), pitched(p_src), Pitched(None, 0, 0), (0, 0, 0), m,
                           [(lo, hi)])
    for label, system, nin, alias, torch_fn in work:
        ins = [new() for _ in range(nin)]
        outs = [ins[i] for i in alias] if alias else [new() for _ in range(system.nout)]
        plan = sb.SystemPlan(0, system, [pitched(t) for t in outs], [pitched(t) for t in ins], (0, 0, 0), m, [(lo, hi)])
        ts, t7, tt, tc = [], [], [], []
        for it in range(args.warmup + args.iters):
            a = timed(s, lambda: plan.launch(s))
            b = timed(s, lambda: plain.launch(s))
            with torch.cuda.stream(s):
                d = timed(s, lambda: torch_fn(ins, outs))
                e_ = timed(s, lambda: cdst.copy_(csrc))
            if it >= args.warmup:
                ts.append(a)
                t7.append(b)
                tt.append(d)
                tc.append(e_)
        t, tp, ttorch, tcp = trimean(ts), trimean(t7), trimean(tt), trimean(tc)
        ceil = cbytes / (tcp * 1e-3)
        rate, rate7 = plan.bytes / (t * 1e-3), plain.bytes / (tp * 1e-3)
        rec = dict(workload=label, gpu=name, power_limit=limit, iters=args.iters, terms=len(system.terms), inputs=nin, outputs=system.nout,
                   bytes_per_cell=int(plan.bytes) // N**3, kernel_ms=round(t, 4), GBps=round(rate / 1e9, 1), share_of_copy_ceiling=round(rate / ceil, 3),
                   plain7_ms=round(tp, 4), plain7_GBps=round(rate7 / 1e9, 1), rate_over_plain7=round(rate / rate7, 3), torch_ms=round(ttorch, 4),
                   speedup_over_torch=round(ttorch / t, 2), copy_ms=round(tcp, 4), copy_ceiling_GBps=round(ceil / 1e9, 1))
        print(json.dumps(rec), flush=True)
        plan.destroy()
        del ins, outs
        torch.cuda.empty_cache()
    plain.destroy()
    print(json.dumps(dict(sm_clock_now_and_max=sm_clock())), flush=True)


if __name__ == "__main__":
    main()
