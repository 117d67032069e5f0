"""Multigrid V-cycles (tests/mg_gpu.py) across processes.  Two modes over the same seeded right-hand side and the same
partition of every level into N subdomains:
    python tests/mp_mg_check.py --single N OUT.json                     one process, N subdomains: checks the result against
                                                                        the numpy cycle and writes its bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29601 \\
        tests/mp_mg_check.py --expect OUT.json                          one subdomain per rank: the gathered global result
                                                                        must equal the file's bits on every rank
Runs three V(2,2) cycles over 4 levels (32^3 .. 4^3) of -lap u = f with ODD(0) walls, in float and double.  Ranks share
GPUs when there are fewer GPUs than ranks."""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import mg_gpu  # noqa: E402
import transfer_oracle as to  # noqa: E402
from mp_stencil_check import load  # noqa: E402

SIZE = (32, 32, 32)


def gather(dd, q, world):
    """The global [z, y, x] compute array of quantity q, assembled from every rank's subdomains."""
    mine = []
    for d in dd.domains():
        o, sz, p = d.origin(), d.size(), d.halo_pos((0, 0, 0), True)
        a = d.quantity_to_host(q)
        mine.append((o, sz, a[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]].copy()))
    if world > 1:
        import torch.distributed as td

        parts = [None] * world
        td.all_gather_object(parts, mine)
        mine = [x for part in parts for x in part]
    out = np.full(dd.size()[::-1], np.nan, mine[0][2].dtype)
    for o, sz, a in mine:
        out[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]] = a
    return out


def run(gpus, world, check_oracle):
    out = {}
    for dtype in (np.float64, np.float32):
        lv = mg_gpu.hierarchy(SIZE, 4, 0.0, dtype, (mg_gpu.F,) * 3, gpus)
        f = np.random.default_rng(32).uniform(-1, 1, SIZE[::-1]).astype(dtype)
        load(lv[0].dd, lv[0].f.id, "curr", f)
        for L in lv:
            load(L.dd, L.u.id, "curr", np.zeros(L.size[::-1], dtype))
        if check_oracle:
            ref = to.hierarchy(SIZE, 4, 0.0, dtype, (False,) * 3)
            ref[0].interior(ref[0].f)[...] = f
        for cyc in range(3):
            mg_gpu.vcycle(lv)
            got = gather(lv[0].dd, lv[0].u.id, world)
            if check_oracle:
                to.vcycle(ref)
                want = ref[0].interior(ref[0].u)
                assert np.array_equal(got.view(np.uint8), np.ascontiguousarray(want).view(np.uint8)), f"{np.dtype(dtype).name} cycle {cyc}: bits differ from the oracle"
            out[f"cycle{cyc}_{np.dtype(dtype).name}"] = hashlib.sha256(got.tobytes()).hexdigest()
        mg_gpu.close(lv)
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n, 1, True), f)
        print("mp_mg_check single OK", flush=True)
        return
    import torch.distributed as td

    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = local % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    td.init_process_group("gloo")
    rank, world = td.get_rank(), td.get_world_size()
    got = run([dev], world, False)
    with open(sys.argv[2]) as f:
        want = json.load(f)
    assert got == want, f"rank {rank}: {got} != one-process {want}"
    td.barrier()
    if rank == 0:
        print(f"mp_mg_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
