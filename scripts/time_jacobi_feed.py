"""How close the fused jacobi kernel runs to what the card can stream, on ONE GPU, in one process:

  * the card: name, power limit and max SM clock (read-only nvidia-smi query);
  * the copy ceiling on two 514^3 FP64 buffers (the 512^3 subdomain with its ghost layer, 1.086 GB each):
    dst.copy_(src) (a device-to-device memcpy) and one torch elementwise kernel with out=; bytes = read + write;
  * the fused step (Jacobi3D.step_fused) on 512^3 FP64.

Times are CUDA events around each call, reduced to the trimean of --reps samples.  With --ab LIB the script then
alternates bench.py between this tree's library and LIB (SB_LIB_PATH, e.g. a parent-commit build) for --pairs FP64
and --pairs FP32 pairs, then scripts/time_fused.py's 2- and 8-subdomain one-GPU stand-ins.

usage: python scripts/time_jacobi_feed.py [--reps 40] [--ab stencil_b200/_alt/libstencil_b200_parent.so] [--pairs 3]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def trimean(ts):
    q1, q2, q3 = np.percentile(ts, [25, 50, 75])
    return float((q1 + 2 * q2 + q3) / 4)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 -- the numbers below stand without it, labelled
        out = f"nvidia-smi unavailable ({e})"
    return out


def event_trimean(fn, stream, reps, warm=5):
    for _ in range(warm):
        fn()
    stream.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return trimean(ts)


def ceiling(reps):
    n = 514
    src = torch.rand(n, n, n, dtype=torch.float64, device="cuda")
    dst = torch.empty_like(src)
    nbytes = 2 * src.numel() * src.element_size()
    s = torch.cuda.current_stream()
    res = {}
    for name, fn in (("memcpy dst.copy_(src)", lambda: dst.copy_(src)), ("elementwise torch.mul(src, 0.5, out=dst)", lambda: torch.mul(src, 0.5, out=dst))):
        ms = event_trimean(fn, s, reps)
        res[name] = {"ms": ms, "gbs": nbytes / (ms * 1e-3) / 1e9}
        print(f"  {name:44s} {ms:.4f} ms  {res[name]['gbs']:.0f} GB/s  ({nbytes / 1e9:.3f} GB read + write)", flush=True)
    del src, dst
    torch.cuda.empty_cache()
    return res


def fused(reps):
    import stencil_b200 as sb
    from stencil_b200.jacobi import Jacobi3D, jacobi_radius

    n = 512
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0])
    dd.set_radius(jacobi_radius())
    h = dd.add_data(np.float64)
    dd.realize()
    jac = Jacobi3D(dd, h)
    jac.init(0.5)
    ms = event_trimean(jac.step_fused, jac.streams[0], reps)
    gbs = 16 * n**3 / (ms * 1e-3) / 1e9
    print(f"  fused 512^3 FP64 {ms:.4f} ms  {gbs:.0f} GB/s algorithmic", flush=True)
    jac.close()
    dd.close()
    return {"ms": ms, "gbs": gbs}


def bench(lib, extra=()):
    env = dict(os.environ)
    if lib:
        env["SB_LIB_PATH"] = os.path.abspath(lib)
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "200", "--warmup", "20", "--no-cpu-baseline", "--no-e2e", "--no-exchange-bench", *extra]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, cwd=ROOT)
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    if out.returncode or not line:
        print(out.stdout[-2000:], out.stderr[-2000:], flush=True)
        raise SystemExit(f"bench.py failed ({out.returncode})")
    r = json.loads(line[-1])
    par = (r.get("parity_check") or {}).get("bit_exact")
    clk = r.get("clocks") or {}
    print(f"  {('new' if not lib else 'alt'):3s} {' '.join(extra) or 'f64':12s} {r['ms_per_step']:.4f} ms/step  bit_exact={par}  "
          f"sm {clk.get('sm_mhz')}/{clk.get('sm_max_mhz')} MHz  limit {clk.get('power_limit_w')} W  {r.get('gpu')}", flush=True)
    return r["ms_per_step"], par


def stand_ins(lib):
    # 512^3 cut into 2 and into 8 subdomains on this GPU: every cut face is pushed as between ranks (EDGE = 2 kernel)
    env = dict(os.environ)
    if lib:
        env["SB_LIB_PATH"] = os.path.abspath(lib)
    res = []
    for only in ("2", "8"):
        env["ONLY"] = only
        out = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "time_fused.py"), "512", "30"], env=env, capture_output=True, text=True, cwd=ROOT)
        if out.returncode:
            print(out.stdout[-2000:], out.stderr[-2000:], flush=True)
            raise SystemExit("time_fused.py failed")
        ln = out.stdout.strip().splitlines()[-1]
        print(f"  {('new' if not lib else 'alt'):3s} {ln}", flush=True)
        res.append(float(ln.split("ms/step")[0].split()[-1]))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=40)
    ap.add_argument("--ab", default=None, help="library to alternate with this tree's (SB_LIB_PATH)")
    ap.add_argument("--pairs", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    print(f"card: {card()}", flush=True)
    print("copy ceiling, 2 x 514^3 FP64:", flush=True)
    ceil = ceiling(args.reps)
    top = max(v["gbs"] for v in ceil.values())
    r = fused(args.reps)
    print(f"    = {r['gbs'] / top:.3f} of the copy ceiling ({top:.0f} GB/s)", flush=True)
    if not args.ab:
        return
    print(f"A/B: bench.py --steps 200 --warmup 20, this tree ('new') vs {args.ab} ('alt'), alternating", flush=True)
    for name, extra in (("FP64", ()), ("FP32", ("--dtype", "f32"))):
        new, alt = [], []
        for _ in range(args.pairs):
            alt.append(bench(args.ab, extra)[0])
            new.append(bench(None, extra)[0])
        print(f"  {name} median new {np.median(new):.4f} alt {np.median(alt):.4f} ms/step ({np.median(new) / np.median(alt) - 1:+.1%}); "
              f"new {min(new):.4f}..{max(new):.4f}, alt {min(alt):.4f}..{max(alt):.4f}", flush=True)
    stand_ins(args.ab)
    stand_ins(None)
    print("copy ceiling again:", flush=True)
    ceiling(args.reps)


if __name__ == "__main__":
    main()
