"""Exact reductions across processes.  Two modes over the same seeded fields:
    python tests/mp_reduce_exact_check.py --single N OUT.json           one process, N subdomains: checks the sums
                                                                        against the oracle, writes the result bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node R --master-addr 127.0.0.1 --master-port 29571 \\
        tests/mp_reduce_exact_check.py --expect OUT.json                one subdomain per rank: every rank checks that its
                                                                        bits equal the file's and every other rank's
The file may come from a run with a different number of subdomains: exact sums do not depend on the partition.  The
fields spread over 80 binades, so ordered sums would.  Ranks share GPUs when there are fewer GPUs than ranks;
torch.distributed (gloo) is only the rendezvous and the gather."""
import json
import math
import os
import struct
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import stencil_b200 as sb  # noqa: E402

SHAPES = ((np.float64, (40, 36, 28), 2), (np.float32, (33, 30, 26), 1))


def bits(r: sb.Reduction) -> str:
    return struct.pack("<4dq", r.min, r.max, r.sum, r.sumsq, r.count).hex()


def fields(dtype, size):
    rng = np.random.default_rng(23)
    shape = tuple(reversed(size))
    span = 40 if dtype == np.float64 else 20
    return [(rng.standard_normal(shape) * np.ldexp(1.0, rng.integers(-span, span, shape))).astype(dtype) for _ in range(4)]


def run(gpus, oracle: bool) -> dict:
    out = {}
    for dtype, size, radius in SHAPES:
        dd = sb.DistributedDomain(*size)
        dd.set_gpus(gpus)
        dd.set_radius(radius)
        hs = [dd.add_data(dtype) for _ in range(3)]
        dd.realize()
        glob = fields(dtype, size)
        for d in dd.domains():
            o, sz, p = d.origin(), d.size(), d.halo_pos((0, 0, 0), True)
            for q, which, g in ((0, "curr", glob[0]), (1, "curr", glob[1]), (2, "curr", glob[2]), (0, "next", glob[3])):
                host = np.full(tuple(reversed(d.raw_size())), np.nan, dtype=dtype)
                host[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]] = g[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]]
                d.quantity_from_host(q, host, which)
        res = dd.reduce_many([("scalar", hs[0]), ("diff", hs[0]), ("norm", hs[0], hs[1], hs[2]), ("scalar", hs[0], "next")], exact=True)
        assert dd.reduce(hs[0], exact=True) == res[0] and dd.reduce_diff(hs[0], exact=True) == res[1]
        assert dd.reduce_norm(hs[0], hs[1], hs[2], exact=True) == res[2]
        if oracle:
            import exact_sum_oracle as xo
            import reduce_oracle as ro

            want = [xo.reduce_cells(ro.SCALAR, glob[0]), xo.reduce_cells(ro.DIFF, glob[0], glob[3]), xo.reduce_cells(ro.NORM3, *glob[:3]),
                    xo.reduce_cells(ro.SCALAR, glob[3])]  # fmt: skip
            for r, w in zip(res, want):
                assert struct.pack("<dd", r.sum, r.sumsq) == struct.pack("<dd", w["sum"], w["sumsq"]) and r.count == w["count"], (r, w)
                assert r.min == w["min"] and r.max == w["max"] and not math.isnan(r.sum)
        out[np.dtype(dtype).name] = [bits(r) for r in res]
        dd.close()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n, oracle=True), f)
        print("mp_reduce_exact_check single OK", flush=True)
        return
    import torch.distributed as td

    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = local % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    td.init_process_group("gloo")
    rank, world = td.get_rank(), td.get_world_size()
    got = run([dev], oracle=False)
    with open(sys.argv[2]) as f:
        want = json.load(f)
    everyone = [None] * world
    td.all_gather_object(everyone, got)
    assert all(e == got for e in everyone), f"rank {rank}: ranks disagree"
    assert got == want, f"rank {rank}: {got} != one-process {want}"
    td.barrier()
    if rank == 0:
        print(f"mp_reduce_exact_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
