"""Rate of coloured in-place application (sb_stencil_cplan_create) on one GPU, against the uncoloured launch of the same
op and the copy ceiling in the same run, and the cost and effect of Gauss-Seidel / SOR sweeps through
DistributedDomain.apply.

    python scripts/time_colour_op.py [--iters 40] [--warmup 5] [--sweeps 200]

Kernel workloads, 512^3 compute cells in 514^3 allocations (one tile-kernel launch), FP64 and FP32:
  7-point red pass / black pass: the SOR update of -lap u + sigma u = f in place (u read and written, f on aux);
  damped: u + theta (div(kappa grad u) - f) in place, kappa in 3 coefficient fields, red pass;
  27-point: a 27-point relaxation under 8 colours, colour 0.
Each coloured launch is alternated with (a) the uncoloured launch of the same op into a separate dst and (b)
dst.copy_(src) over two allocations (the copy ceiling, bytes = read + write).  Bytes per cell: every input read once,
plus one element written per cell of the colour (1/m of the cells).  Every timing is the trimean of --iters launches
timed one by one with CUDA events on one stream, after --warmup untimed ones.

Sweeps: a 256^3 FP64 Poisson problem -lap u = f walled on every face with Dirichlet ODD(0) (u = 0 on the wall face,
half a cell out: the ghost cell mirrors the cell as -u) and with VALUE(0) (the ghost cell holds 0), from u = 0: Jacobi
(relax(1), out-of-place apply + swap), red-black Gauss-Seidel and red-black SOR at omega_opt = 2 / (1 + sin(pi h)), each
through DistributedDomain.apply (exchange overlapped).  Reports the wall time per sweep over --sweeps sweeps and the
residual ||f - A u||_2, from reduce(), after 1, 5 and 10 times --sweeps sweeps.
Prints the GPU's name, power limit and SM clock, then one JSON line per workload."""
from __future__ import annotations

import argparse
import itertools
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_boundary import gpu_info, timed, trimean  # noqa: E402
from time_system_op import sm_clock  # noqa: E402

N = 512


def helmholtz(h, sigma):
    """A of -lap u + sigma u (order-2 Laplacian, spacing h), the centre first."""
    import numpy as np

    import stencil_b200 as sb

    lap = sb.StencilOp.laplacian(2, (h, h, h), np.float64).terms
    return [(0, (0, 0, 0), -lap[0][2] + sigma)] + [(0, o, -w) for _, o, w in lap[1:]]


def kernels(args, name, limit):
    import numpy as np
    import torch

    import stencil_b200 as sb
    from stencil_b200._lib import Pitched

    s = torch.cuda.Stream()
    m = N + 2
    box = [((1, 1, 1), (1 + N, 1 + N, 1 + N))]
    rng = np.random.default_rng(27)
    A27 = [(0, (x, y, z), float(rng.uniform(-1, 0))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]
    sor7 = sb.StencilOp(helmholtz(1.0, 0.06), np.float64).relax(1.6).terms
    sor27 = sb.StencilOp(A27 + [(0, (0, 0, 0), 30.0)], np.float64).relax(1.2).terms
    theta = 0.02
    damped = [(0, (0, 0, 0), 1.0)] + [(sr, o, theta * w, k, c) for sr, o, w, k, c in sb.StencilOp.div_grad((1, 1, 1), np.float64).terms] + [
        (1, (0, 0, 0), -theta)]
    work = [("7-point red pass", sor7, 2, 0, 0), ("7-point black pass", sor7, 2, 1, 0), ("damped div(kappa grad u), red pass", damped, 2, 0, 3),
            ("27-point, 8 colours, colour 0", sor27, 8, 0, 0)]
    for dtype, tdt in ((np.float64, torch.float64), (np.float32, torch.float32)):
        es = np.dtype(dtype).itemsize

        def new():
            return torch.rand(m, m, m, dtype=tdt, device="cuda")

        def pitched(t):
            return Pitched(t.data_ptr(), m * es, m)

        csrc, cdst = new(), new()
        cbytes = 2 * csrc.numel() * es
        for label, terms, ncol, c, nk in work:
            u, f, dst = new(), new(), new()
            ks = [new() + 0.5 for _ in range(nk)]
            op = sb.StencilOp(terms, dtype)
            K = [pitched(k) for k in ks] if nk else None
            col = sb.StencilPlan(0, op, pitched(u), pitched(u), pitched(f), (0, 0, 0), m, box, K, (ncol, c))
            plain = sb.StencilPlan(0, op, pitched(dst), pitched(u), pitched(f), (0, 0, 0), m, box, K)
            tc, tp, tcp = [], [], []
            for it in range(args.warmup + args.iters):
                a = timed(s, lambda: col.launch(s))
                b = timed(s, lambda: plain.launch(s))
                with torch.cuda.stream(s):
                    d = timed(s, lambda: cdst.copy_(csrc))
                if it >= args.warmup:
                    tc.append(a)
                    tp.append(b)
                    tcp.append(d)
            t, t0, tcopy = trimean(tc), trimean(tp), trimean(tcp)
            ceil = cbytes / (tcopy * 1e-3)
            rate, rate0 = col.bytes / (t * 1e-3), plain.bytes / (t0 * 1e-3)
            rec = dict(workload=f"512^3 {np.dtype(dtype).name} {label}", gpu=name, power_limit=limit, iters=args.iters, terms=len(terms), colours=ncol,
                       colour=c, bytes_per_cell=round(col.bytes / N**3, 3), kernel_ms=round(t, 4), GBps=round(rate / 1e9, 1),
                       share_of_copy_ceiling=round(rate / ceil, 3), uncoloured_ms=round(t0, 4), uncoloured_GBps=round(rate0 / 1e9, 1),
                       time_over_uncoloured=round(t / t0, 3), copy_ms=round(tcopy, 4), copy_ceiling_GBps=round(ceil / 1e9, 1))
            print(json.dumps(rec), flush=True)
            col.destroy()
            plain.destroy()
            del u, f, dst, ks
            torch.cuda.empty_cache()
        del csrc, cdst
        torch.cuda.empty_cache()


def sweeps(args, name, limit):
    import numpy as np
    import torch

    import stencil_b200 as sb

    n = 256
    h = 1.0 / (n + 1)
    A = helmholtz(h, 0.0)
    resid = sb.StencilOp([(1, (0, 0, 0), 1.0)] + [(0, o, -w) for _, o, w in A], np.float64)  # f - A u
    w_opt = 2.0 / (1.0 + math.sin(math.pi * h))
    f0 = np.random.default_rng(256).uniform(-1, 1, (n, n, n))
    runs = [("Jacobi (relax(1), out of place + swap)", 1.0, False), ("red-black Gauss-Seidel", 1.0, True),
            (f"red-black SOR, omega_opt = {w_opt:.6f}", w_opt, True)]
    for (label, omega, coloured), (bname, bc) in itertools.product(runs, (("ODD(0)", sb.BC.ODD(0.0)), ("VALUE(0)", sb.BC.VALUE(0.0)))):
        dd = sb.DistributedDomain(n, n, n)
        dd.set_gpus([0])
        dd.set_radius(sb.Radius.face_edge_corner(1, 0, 0))
        u, f, r = dd.add_data(np.float64), dd.add_data(np.float64), dd.add_data(np.float64)
        dd.set_boundary(sb.Boundary.FIXED)
        for fc in sb.FACES:
            dd.set_boundary_condition(u, fc, bc)
        dd.realize()
        for d in dd.domains():
            raw, p = d.raw_size(), d.halo_pos((0, 0, 0), True)
            a = np.zeros(raw[::-1])
            a[p[2] : p[2] + n, p[1] : p[1] + n, p[0] : p[0] + n] = f0
            d.quantity_from_host(f.id, a, "curr")
            d.quantity_from_host(f.id, a, "next")
            d.quantity_from_host(u.id, np.zeros(raw[::-1]), "curr")
            d.quantity_from_host(u.id, np.zeros(raw[::-1]), "next")
        op = sb.StencilOp(A, np.float64).relax(omega)

        def sweep():
            if coloured:
                for c in range(2):
                    dd.apply(op, (u, "curr"), u, f, colour=(2, c))
            else:
                dd.apply(op, u, u, f)
                dd.swap()

        for _ in range(2):  # builds the plans (Jacobi has one per swap parity)
            sweep()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.sweeps - 2):
            sweep()
        torch.cuda.synchronize()
        per = (time.perf_counter() - t0) / (args.sweeps - 2)
        residuals, done = {}, args.sweeps
        for k in sorted({args.sweeps, 5 * args.sweeps, 10 * args.sweeps}):
            for _ in range(k - done):
                sweep()
            done = k
            dd.apply(resid, (r, "curr"), u, f)
            residuals[k] = dd.reduce(r, "curr").l2()
        rec = dict(workload=f"256^3 FP64 Poisson, Dirichlet {bname} walls: {label}", gpu=name, power_limit=limit, timed_sweeps=args.sweeps - 2,
                   ms_per_sweep=round(per * 1e3, 4), residual_l2_after_sweeps=residuals, f_l2=float(np.linalg.norm(f0)))
        print(json.dumps(rec), flush=True)
        dd.close()
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--sweeps", type=int, default=200)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_colour_op.py needs a CUDA device")
    name, limit = gpu_info()
    print(json.dumps(dict(gpu=name, power_limit=limit, sm_clock_now_and_max=sm_clock())), flush=True)
    kernels(args, name, limit)
    sweeps(args, name, limit)
    print(json.dumps(dict(sm_clock_now_and_max=sm_clock())), flush=True)


if __name__ == "__main__":
    main()
