"""DistributedDomain.apply_system across processes.  Two modes over the same seeded fields and the same partition into N
subdomains:
    python tests/mp_system_check.py --single N OUT.json                one process, N subdomains: checks the result against
                                                                       the numpy rule and writes its bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29591 \\
        tests/mp_system_check.py --expect OUT.json                     one subdomain per rank: the gathered global fields
                                                                       must equal the file's bits on every rank
Runs 6 leapfrog steps of Maxwell's equations on a periodic Yee grid (E = E + dt curl- H, then H = H - dt curl+ E, both in
place in the curr buffers, overlapped with the exchange), in float and double.  Ranks share GPUs when there are fewer GPUs
than ranks."""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import stencil_b200 as sb  # noqa: E402
import system_oracle as yo  # noqa: E402
from mp_stencil_check import SIZE, gather, load  # noqa: E402

H = (1.0, 0.5, 0.75)
IDENT = [(j, 3 + j, (0, 0, 0), 1.0) for j in range(3)]


def run(gpus, world, check_oracle):
    out = {}
    et, ht = IDENT + yo.scaled(yo.curl(-1, H), 0.2), IDENT + yo.scaled(yo.curl(1, H), -0.2)
    for dtype in (np.float64, np.float32):
        rng = np.random.default_rng(43)
        f = [rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(6)]
        dd = sb.DistributedDomain(*SIZE)
        dd.set_gpus(gpus)
        dd.set_radius(sb.Radius.face_edge_corner(1, 0, 0))
        hs = [dd.add_data(dtype) for _ in range(6)]
        dd.realize()
        for q, a in zip(hs, f):
            load(dd, q.id, "curr", a)
        e_sys, h_sys = sb.StencilSystem(et, dtype), sb.StencilSystem(ht, dtype)
        E, Hf = hs[:3], hs[3:]
        for _ in range(6):
            dd.apply_system(e_sys, [(q, "curr") for q in E], list(Hf) + [(q, "curr") for q in E])
            dd.apply_system(h_sys, [(q, "curr") for q in Hf], list(E) + [(q, "curr") for q in Hf])
            if check_oracle:
                f[:3] = yo.apply_periodic(et, f[3:] + f[:3])
                f[3:] = yo.apply_periodic(ht, f[:3] + f[3:])
        for k, q in enumerate(hs):
            got = gather(dd, q.id, world)
            if check_oracle:
                assert np.array_equal(got.view(np.uint8), f[k].view(np.uint8)), f"field {k} {np.dtype(dtype).name}: bits differ from the oracle"
            out[f"yee{k}_{np.dtype(dtype).name}"] = hashlib.sha256(got.tobytes()).hexdigest()
        dd.close()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n, 1, True), f)
        print("mp_system_check single OK", flush=True)
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
        print(f"mp_system_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
