"""Time the astaroth substep kernels and the full iteration.  usage: time_astaroth.py [n] [f64|f32] [reps]"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stencil_b200 as sb
from stencil_b200 import astaroth as ac

n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
dtype = np.float64 if (len(sys.argv) <= 2 or sys.argv[2] == "f64") else np.float32
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 5
es = np.dtype(dtype).itemsize
peak = 3350.0  # H100 SXM data sheet HBM3 GB/s (not measured)

dd = sb.DistributedDomain(n, n, n)
dd.set_gpus([0])
dd.set_radius(3)
handles = [dd.add_data(dtype, nm) for nm in ac.FIELDS]
dd.realize()
d = dd.domains()[0]
rng = np.random.default_rng(0)
raw = d.raw_size()
for q in range(8):
    for which in ("curr", "next"):
        d.quantity_from_host(q, (0.1 * rng.standard_normal(raw[::-1])).astype(dtype), which)
params = ac.conf_params(1e-8)
m = n + 6
cur = [d.pitched(h.id, "curr").ptr for h in handles]
nxt = [d.pitched(h.id, "next").ptr for h in handles]
stream = torch.cuda.Stream()
cells = n**3


def timeit(fn, reps=reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


tag = os.environ.get("SB_AC_SHAPE", "0") + "/" + os.environ.get("SB_AC_ZCHUNK", "auto")
for variant, name in ((ac.TEAM3_TMA, "team3-tma"), (ac.TEAM_TMA, "team2-tma"), (ac.TEAM, "team"), (ac.TILE, "tile"), (ac.CELL, "cell")):
    if variant in (ac.TEAM3_TMA, ac.TEAM_TMA) and dtype != np.float64:
        continue
    if variant == ac.CELL and os.environ.get("SKIP_CELL"):
        continue
    for step in range(3):
        ms = timeit(lambda: ac.substep(step, cur, nxt, es, (m, m, m), (3, 3, 3), (m - 3, m - 3, m - 3), params, variant, stream), reps if variant != ac.CELL else 2)
        alg = (16 if step == 0 else 24) * es * cells
        print(f"[{np.dtype(dtype).name} n={n} shape/zc={tag}] {name} substep {step}: {ms:.4f} ms  {cells/ms/1e6:.1f} Gcell/s  {alg/ms/1e6:.0f} GB/s algorithmic = {alg/ms/1e6/peak*100:.1f}% of HBM peak", flush=True)
if not os.environ.get("SKIP_ITER"):
    for overlap in (True, False):
        sim = ac.Astaroth(dd, handles, params, overlap=overlap)
        sim.step()
        torch.cuda.synchronize()
        import time

        t0 = time.perf_counter()
        for _ in range(reps):
            sim.step()
        torch.cuda.synchronize()
        dt = (time.perf_counter() - t0) / reps
        print(f"[{np.dtype(dtype).name} n={n}] iteration (3 substeps + 3 exchanges + swap) overlap={overlap}: {dt*1e3:.3f} ms  = {cells/dt/1e9:.2f} Gcell/s", flush=True)
dd.close()
