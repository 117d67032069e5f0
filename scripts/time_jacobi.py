"""Time the jacobi kernels alone (CUDA events) at one size and precision.
usage: python scripts/time_jacobi.py [n] [dtype] [reps]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stencil_b200 as sb
from stencil_b200.jacobi import Jacobi3D, jacobi_radius

n = int(sys.argv[1]) if len(sys.argv) > 1 else 512
dtype = np.float64 if (len(sys.argv) <= 2 or sys.argv[2] == "f64") else np.float32
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 20
dd = sb.DistributedDomain(n, n, n)
dd.set_gpus([0])
dd.set_radius(jacobi_radius())
h = dd.add_data(dtype)
dd.realize()
jac = Jacobi3D(dd, h)
jac.init(0.5)
s = jac.streams[0]
es = np.dtype(dtype).itemsize


def timeit(fn, cells):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record(s)
        fn()
        b.record(s)
        s.synchronize()
        ts.append(a.elapsed_time(b))
    ms = float(np.median(ts))
    return ms, 2 * es * cells / (ms * 1e-3) / 1e9


cfg = f"{np.dtype(dtype).name} {n}^3"
ms, gbs = timeit(jac.launch_interior, jac.interior_cells)
print(f"{cfg} interior {ms:.4f} ms {gbs:.0f} GB/s", flush=True)
ms, gbs = timeit(jac.launch_whole, n**3)
print(f"{cfg} whole    {ms:.4f} ms {gbs:.0f} GB/s", flush=True)
ext_cells = n**3 - jac.interior_cells
ms, gbs = timeit(jac.launch_exterior, ext_cells)
print(f"{cfg} exterior {ms:.4f} ms ({ext_cells} cells)", flush=True)
ms, _ = timeit(lambda: dd._plans[0][0].launch(s), 1)
print(f"{cfg} exchange kernel {ms:.4f} ms for {dd._plans[0][0].bytes} B -> {dd._plans[0][0].bytes/ms/1e6:.0f} GB/s payload", flush=True)
dd.close()
