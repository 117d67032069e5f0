"""Time the fused jacobi kernel variants on ONE GPU (same box, same run): the plain whole-region kernel as calibration,
the fused schedule on one 512^3 subdomain, and -- as a single-GPU stand-in for the multi-rank kernels -- the same 512^3
cut into 2 (x) and 8 (2x2x2) subdomains on this GPU, where every cut face is shipped (dense x arrays, ghost rows / planes)
between subdomains exactly as between ranks, minus the flags and the NVLink latency.
usage: python scripts/time_fused.py [n=512] [reps=30]"""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stencil_b200 as sb
from stencil_b200.jacobi import Jacobi3D, jacobi_radius

n = int(sys.argv[1]) if len(sys.argv) > 1 else 512
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 30
dtype = np.float64 if os.environ.get("DTYPE", "f64") == "f64" else np.float32


def run(ndom, label, fused=True, shape=None):
    dd = sb.DistributedDomain(*(shape or (n, n, n)))
    ngpu = int(os.environ.get("NGPU", "1"))  # NGPU=2: the subdomains alternate between two GPUs of this process (NVLink pushes)
    dd.set_gpus([i % ngpu for i in range(ndom)])
    dd.set_radius(jacobi_radius())
    h = dd.add_data(dtype)
    dd.realize()
    jac = Jacobi3D(dd, h)
    jac.init(0.5)
    step = jac.step_fused if fused else jac.launch_whole
    for _ in range(5):
        step()
    jac.synchronize()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        step()
    jac.synchronize()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / reps * 1e3
    es = np.dtype(dtype).itemsize
    cells = int(np.prod(shape)) if shape else n**3
    print(f"{label:58s} {ms:.4f} ms/step  {ms * n**3 / cells:.4f} ms per {n}^3  {2*es*cells/ms/1e6:.0f} GB/s", flush=True)
    jac.close()
    dd.close()
    return ms


only = os.environ.get("ONLY")  # e.g. ONLY=2 -> just the 2-subdomain case with the default kernel (for ncu)
if only:
    run(int(only), f"fused (default variant) subdomains={only}")
    sys.exit(0)
run(1, "plain whole-region kernel (calibration)", fused=False)
if os.environ.get("SPLITS", "1") == "1":
    # which face direction costs what: two 512^3 subdomains on this GPU, cut along x / y / z (the other two axes wrap in place)
    run(2, "fused, 2 x 512^3 cut along x (dense x lines)", shape=(2 * n, n, n))
    run(2, "fused, 2 x 512^3 cut along y", shape=(n, 2 * n, n))
    run(2, "fused, 2 x 512^3 cut along z", shape=(n, n, 2 * n))
    run(8, "fused, 8 x 512^3 cut along x, y and z", shape=(2 * n, 2 * n, 2 * n))
    sys.exit(0)
run(1, "fused, one 512^3 subdomain (every neighbour is the subdomain itself)")
