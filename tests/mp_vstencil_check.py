"""DistributedDomain.apply with coefficient fields across processes.  Two modes over the same seeded fields and the same
partition into N subdomains:
    python tests/mp_vstencil_check.py --single N OUT.json               one process, N subdomains: checks the result against
                                                                        the numpy rule and writes its bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29581 \\
        tests/mp_vstencil_check.py --expect OUT.json                    one subdomain per rank: the gathered global result
                                                                        must equal the file's bits on every rank
Runs a periodic heterogeneous heat equation u + dt div(kappa grad u) (kappa on the faces in three quantities, overlapped
exchange) and a variable-speed wave equation 2u - u_prev + c^2 lap(u) written over u_prev, in float and double.  The
coefficient quantities hold the same cells in curr and next, so they survive every swap.  Ranks share GPUs when there
are fewer GPUs than ranks."""
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
import stencil_op_oracle as so  # noqa: E402
import vstencil_oracle as vo  # noqa: E402
from mp_stencil_check import SIZE, gather, load  # noqa: E402


def run(gpus, world, check_oracle):
    out = {}
    for dtype in (np.float64, np.float32):
        rng = np.random.default_rng(41)
        u0, p0 = (rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(2))
        ks = [rng.uniform(0.2, 2.0, SIZE[::-1]).astype(dtype) for _ in range(3)]
        heat = [(s, o, 0.05 * w, k, c) for s, o, w, k, c in vo.div_grad((0.9, 1.0, 1.1))] + [(0, (0, 0, 0), 1.0)]
        wave = [(0, (0, 0, 0), 2.0), (1, (0, 0, 0), -1.0)] + [(s, o, 0.1 * w, 0, (0, 0, 0)) for s, o, w in so.laplacian(2, (1.0, 1.0, 1.0))]
        for name, terms, nk in (("heat", heat, 3), ("wave", wave, 1)):
            dd = sb.DistributedDomain(*SIZE)
            dd.set_gpus(gpus)
            dd.set_radius(sb.Radius.face_edge_corner(1, 0, 0))
            h = dd.add_data(dtype)
            kh = [dd.add_data(dtype) for _ in range(nk)]
            dd.realize()
            load(dd, h.id, "curr", u0)
            load(dd, h.id, "next", p0)
            for q, k in zip(kh, ks):
                load(dd, q.id, "curr", k)
                load(dd, q.id, "next", k)
            op = sb.StencilOp(terms, dtype)
            u, prev = u0, p0
            for _ in range(6):
                if name == "heat":
                    dd.apply(op, h, h, coefs=kh)
                    u = vo.apply_periodic(terms, u, None, ks) if check_oracle else u
                else:
                    dd.apply(op, (h, "next"), h, (h, "next"), coefs=kh)
                    if check_oracle:
                        u, prev = vo.apply_periodic(terms, u, prev, ks[:1]), u
                dd.swap()
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
        print("mp_vstencil_check single OK", flush=True)
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
        print(f"mp_vstencil_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
