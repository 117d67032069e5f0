"""DistributedDomain.exchange(only=...) and a PCG solve across processes (DESIGN.md section 2.15).  Two modes over the same
grids, fills and partition into N subdomains:
    python tests/mp_exchange_subset_check.py --single N OUT.json     one process, N subdomains: writes the bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29661 \\
        tests/mp_exchange_subset_check.py --expect OUT.json          one subdomain per rank (CUDA IPC, or the NCCL
                                                                     fallback with SB_FORCE_NCCL=1): every rank's
                                                                     subdomains must hold the file's bits
The exchange part poisons every ghost cell, exchanges subsets of four quantities (float32, int8, float64, float32) on a
walled grid with boundary conditions, before and after swap(), and records the whole allocation of every quantity of
every subdomain after each; the solver part is tests/mp_krylov_check.py's PCG, whose internal exchanges are subsets.
Ranks share GPUs when there are fewer GPUs than ranks."""
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
from mp_krylov_check import run as pcg_run  # noqa: E402
from oracle import np_oracle as no  # noqa: E402

DTYPES = [np.float32, np.int8, np.float64, np.float32]
SUBSETS = [(0,), (1, 2), (3,), (0, 1, 2, 3)]


def poisoned(d, q, seed):
    dt = np.dtype(DTYPES[q])
    raw, sz, r, org = d.raw_size(), d.size(), d.radius(), d.origin()
    lo = (r.x(-1), r.y(-1), r.z(-1))
    a = np.full(raw[::-1], np.nan if dt.kind == "f" else 0x5A, dt)
    zz, yy, xx = np.meshgrid(*[np.arange(org[k], org[k] + sz[k]) for k in (2, 1, 0)], indexing="ij")
    a[lo[2] : lo[2] + sz[2], lo[1] : lo[1] + sz[1], lo[0] : lo[0] + sz[0]] = (no.hash_field(q, xx, yy, zz) % 101 + seed).astype(dt)
    return a


def exchange_bits(gpus):
    """{"<subset>/<round>/<subdomain index>/<quantity>": sha256 of the whole allocation after the subset exchange}."""
    dd = sb.DistributedDomain(24, 18, 20)
    dd.set_gpus(gpus)
    dd.set_radius(sb.Radius.face_edge_corner(2, 1, 1))
    hs = [dd.add_data(dt, f"q{i}") for i, dt in enumerate(DTYPES)]
    dd.set_boundary(sb.Boundary.FIXED, sb.Boundary.PERIODIC, sb.Boundary.FIXED)
    for q, h in enumerate(hs):
        for f in (0, 1, 4, 5):
            if np.dtype(DTYPES[q]).kind == "f":
                bc = [sb.BC.ODD(0.25 * q), sb.BC.EVEN(), sb.BC.VALUE(-1.5), sb.BC.ODD(0.0)][(q + f) % 4]
            else:
                bc = sb.BC.EVEN()
            dd.set_boundary_condition(h, sb.FACES[f], bc)
    dd.realize()
    out = {}
    for rnd in range(2):
        for sub in SUBSETS:
            for d in dd.domains():
                for q in range(len(DTYPES)):
                    d.quantity_from_host(q, poisoned(d, q, rnd))
            dd.exchange(only=[hs[q] for q in sub])
            for idx, d in zip(dd.domain_idx_, dd.domains()):
                for q in range(len(DTYPES)):
                    out["/".join(map(str, (sub, rnd, idx, q)))] = hashlib.sha256(d.quantity_to_host(q).tobytes()).hexdigest()
        dd.swap()
    dd.close()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump({"exchange": exchange_bits([0] * n), "pcg": pcg_run([0] * n, 1, False)}, f)
        print("mp_exchange_subset_check single OK", flush=True)
        return
    import torch.distributed as td

    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = local % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    if os.environ.get("SB_FORCE_NCCL") == "1":  # the exchange's fallback sends device buffers through the process group
        td.init_process_group("nccl", device_id=torch.device("cuda", dev))
    else:
        td.init_process_group("gloo")
    rank, world = td.get_rank(), td.get_world_size()
    with open(sys.argv[2]) as f:
        want = json.load(f)
    got = exchange_bits([dev])
    assert got and all(want["exchange"][k] == v for k, v in got.items()), f"rank {rank}: subset exchange bits differ from one process"
    assert pcg_run([dev], world, False) == want["pcg"], f"rank {rank}: PCG bits differ from one process"
    td.barrier()
    if rank == 0:
        print(f"mp_exchange_subset_check OK: world={world} nccl={os.environ.get('SB_FORCE_NCCL', '0')}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
