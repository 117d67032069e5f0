"""Coloured DistributedDomain.apply across processes.  Two modes over the same seeded fields and the same partition into
N subdomains:
    python tests/mp_colour_check.py --single N OUT.json                 one process, N subdomains: checks the result against
                                                                        the numpy rule and writes its bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29591 \\
        tests/mp_colour_check.py --expect OUT.json                      one subdomain per rank: the gathered global result
                                                                        must equal the file's bits on every rank
Runs, in float and double, 4 red-black SOR sweeps of a periodic Helmholtz problem in place (f on aux, overlapped
exchange) and one 8-colour sweep of a 27-point relaxation.  Ranks share GPUs when there are fewer GPUs than ranks."""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import colour_oracle as co  # noqa: E402
import stencil_b200 as sb  # noqa: E402
from mp_stencil_check import SIZE, gather, load  # noqa: E402


def box27_relax():
    rng = np.random.default_rng(27)
    A = [(0, (x, y, z), float(rng.uniform(-1, 0))) for z in (-1, 0, 1) for y in (-1, 0, 1) for x in (-1, 0, 1) if (x, y, z) != (0, 0, 0)]
    return co.relax(A + [(0, (0, 0, 0), 30.0)], 1.2)


def run(gpus, world, check_oracle):
    out = {}
    for dtype in (np.float64, np.float32):
        rng = np.random.default_rng(51)
        u0, f = (rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(2))
        sor = co.relax(co.helmholtz(1.0, 0.3), 1.6)
        for name, terms, m, sweeps, radius in (("sor", sor, 2, 4, sb.Radius.face_edge_corner(1, 0, 0)),
                                               ("box27", box27_relax(), 8, 1, sb.Radius.face_edge_corner(1, 1, 1))):
            dd = sb.DistributedDomain(*SIZE)
            dd.set_gpus(gpus)
            dd.set_radius(radius)
            h, hf = dd.add_data(dtype), dd.add_data(dtype)
            dd.realize()
            load(dd, h.id, "curr", u0)
            load(dd, hf.id, "curr", f)
            op = sb.StencilOp(terms, dtype)
            u = u0
            for _ in range(sweeps):
                for c in range(m):
                    dd.apply(op, (h, "curr"), h, hf, colour=(m, c))
                    if check_oracle:
                        u = co.apply_periodic(terms, u, f, [], u, m, c)
            got = gather(dd, h.id, world)
            dd.close()
            if check_oracle:
                assert np.array_equal(got.view(np.uint8), u.view(np.uint8)), f"{name} {np.dtype(dtype).name}: bits differ from the oracle"
            out[f"{name}_{np.dtype(dtype).name}"] = hashlib.sha256(got.tobytes()).hexdigest()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n, 1, True), f)
        print("mp_colour_check single OK", flush=True)
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
        print(f"mp_colour_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
