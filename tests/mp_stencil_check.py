"""DistributedDomain.apply across processes.  Two modes over the same seeded fields and the same partition into N
subdomains:
    python tests/mp_stencil_check.py --single N OUT.json                one process, N subdomains: checks the result against
                                                                        the numpy rule and writes its bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29571 \\
        tests/mp_stencil_check.py --expect OUT.json                     one subdomain per rank: the gathered global result
                                                                        must equal the file's bits on every rank
Runs a periodic heat equation (order-4 Laplacian, overlapped exchange) and a wave equation written over u_prev
(dst == aux == next), in float and double.  Ranks share GPUs when there are fewer GPUs than ranks."""
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

SIZE = (34, 22, 18)


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
    out = np.full(SIZE[::-1], np.nan, mine[0][2].dtype)
    for o, sz, a in mine:
        out[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]] = a
    return out


def load(dd, q, which, glob):
    for d in dd.domains():
        o, sz, p = d.origin(), d.size(), d.halo_pos((0, 0, 0), True)
        host = np.full(d.raw_size()[::-1], np.nan, glob.dtype)
        host[p[2] : p[2] + sz[2], p[1] : p[1] + sz[1], p[0] : p[0] + sz[0]] = glob[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]]
        d.quantity_from_host(q, host, which)


def run(gpus, world, check_oracle):
    out = {}
    for dtype in (np.float64, np.float32):
        rng = np.random.default_rng(31)
        u0, p0 = (rng.uniform(-1, 1, SIZE[::-1]).astype(dtype) for _ in range(2))
        heat = [(0, (0, 0, 0), 1.0)] + [(s, o, 0.02 * w) for s, o, w in so.laplacian(4, (1.0, 0.9, 1.1))]
        wave = [(0, (0, 0, 0), 2.0), (1, (0, 0, 0), -1.0)] + [(s, o, 0.15 * w) for s, o, w in so.laplacian(2, (1.0, 1.0, 1.0))]
        for name, terms, radius in (("heat", heat, sb.Radius.face_edge_corner(2, 0, 0)), ("wave", wave, sb.Radius.constant(1))):
            dd = sb.DistributedDomain(*SIZE)
            dd.set_gpus(gpus)
            dd.set_radius(radius)
            h = dd.add_data(dtype)
            dd.realize()
            load(dd, h.id, "curr", u0)
            load(dd, h.id, "next", p0)
            op = sb.StencilOp(terms, dtype)
            u, prev = u0, p0
            for _ in range(6):
                if name == "heat":
                    dd.apply(op, h, h)
                    u = so.apply_periodic(terms, u, None) if check_oracle else u
                else:
                    dd.apply(op, (h, "next"), h, (h, "next"))
                    if check_oracle:
                        u, prev = so.apply_periodic(terms, u, prev), u
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
        print("mp_stencil_check single OK", flush=True)
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
        print(f"mp_stencil_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
