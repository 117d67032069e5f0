"""Reductions across processes.  Two modes over the same seeded fields and the same partition into N subdomains:
    python tests/mp_reduce_check.py --single N OUT.json                 one process, N subdomains: writes the result bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29561 \\
        tests/mp_reduce_check.py --expect OUT.json                      one subdomain per rank: every rank checks that its
                                                                        bits equal the file's and every other rank's
Ranks share GPUs when there are fewer GPUs than ranks.  torch.distributed (gloo) is only the rendezvous and the gather."""
import json
import os
import struct
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import stencil_b200 as sb  # noqa: E402
from stencil_b200.jacobi import Jacobi3D, jacobi_radius  # noqa: E402


def bits(r: sb.Reduction) -> str:
    return struct.pack("<4dq", r.min, r.max, r.sum, r.sumsq, r.count).hex()


def run(gpus) -> dict:
    out = {}
    for dtype, size, radius in ((np.float64, (40, 36, 28), 2), (np.float32, (33, 30, 26), 1)):
        dd = sb.DistributedDomain(*size)
        dd.set_gpus(gpus)
        dd.set_radius(radius)
        hs = [dd.add_data(dtype) for _ in range(3)]
        dd.realize()
        rng = np.random.default_rng(17)
        glob = [rng.standard_normal(tuple(reversed(size))).astype(dtype) for _ in range(4)]
        for d in dd.domains():
            o, sz, p = d.origin(), d.size(), d.halo_pos((0, 0, 0), True)
            for q, which, g in ((0, "curr", glob[0]), (1, "curr", glob[1]), (2, "curr", glob[2]), (0, "next", glob[3])):
                host = np.full(tuple(reversed(d.raw_size())), np.nan, dtype=dtype)
                host[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]] = g[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]]
                d.quantity_from_host(q, host, which)
        res = dd.reduce_many([("scalar", hs[0]), ("diff", hs[0]), ("norm", hs[0], hs[1], hs[2]), ("scalar", hs[1], "next")])
        out[np.dtype(dtype).name] = [bits(r) for r in res]
        dd.close()
    n = 48
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus(gpus)
    dd.set_radius(jacobi_radius())
    h = dd.add_data(np.float64)
    dd.realize()
    jac = Jacobi3D(dd, h)
    jac.init(0.5)
    for _ in range(5):
        jac.step()
    out["jacobi_residual"] = struct.pack("<d", jac.residual()).hex()
    jac.close()
    dd.close()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n), f)
        print("mp_reduce_check single OK", flush=True)
        return
    import torch.distributed as td

    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = local % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    td.init_process_group("gloo")
    rank, world = td.get_rank(), td.get_world_size()
    got = run([dev])
    with open(sys.argv[2]) as f:
        want = json.load(f)
    everyone = [None] * world
    td.all_gather_object(everyone, got)
    assert all(e == got for e in everyone), f"rank {rank}: ranks disagree"
    assert got == want, f"rank {rank}: {got} != one-process {want}"
    td.barrier()
    if rank == 0:
        print(f"mp_reduce_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
