"""Run under torchrun (one rank per process; ranks share GPUs when there are fewer GPUs than ranks): boundary
conditions on non-periodic grids through the one-process-per-GPU exchange (CUDA-IPC direct writes + device-side flags)
vs the oracle (tests/bc_oracle.py), whole allocations, three exchange/swap rounds per case.
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29541 tests/mp_boundary_check.py
torch.distributed is only the rendezvous (gloo): the data path is the library's."""
import os
import sys

import numpy as np
import torch
import torch.distributed as td

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bc_oracle as bo  # noqa: E402
import stencil_b200 as sb  # noqa: E402
from gpu_util import oracle_radius  # noqa: E402
from oracle import np_oracle as no  # noqa: E402

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED


def main():
    local = int(os.environ.get("LOCAL_RANK", 0))
    dev = local % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    td.init_process_group("gloo")
    rank, world = td.get_rank(), td.get_world_size()
    kinds = [(bo.VALUE, 1.5), (bo.EVEN, 0.0), (bo.ODD, 0.5), (bo.NONE, 0.0), (bo.ODD, -2.25), (bo.VALUE, -0.75)]
    cases = [
        ((24, 20, 16), sb.Radius.constant(2), (F, F, F)),
        ((16, 18, 20), sb.Radius.face_edge_corner(3, 2, 1), (P, P, F)),
        ((20, 12, 12), sb.Radius.constant(1), (F, P, P)),
    ]
    for size, radius, boundary in cases:
        dtypes = [np.float32, np.float64, np.int8]
        bcs = {}
        for q, dt in enumerate(dtypes):
            for f in range(6):
                if boundary[f // 2] == F:
                    bcs[(q, f)] = kinds[(f + 2 * q) % len(kinds)] if dt != np.int8 else ((bo.EVEN, 0.0) if f % 2 else (bo.NONE, 0.0))
        dd = sb.DistributedDomain(*size)
        dd.set_gpus([dev])
        dd.set_radius(radius)
        hs = [dd.add_data(dt) for dt in dtypes]
        dd.set_boundary(*boundary)
        for (q, f), (kind, c) in bcs.items():
            dd.set_boundary_condition(hs[q], sb.FACES[f], sb.BC(kind, c))
        dd.realize()
        od = bo.Domains(size, oracle_radius(radius), dtypes, n_subdomains=world, periodic=[b == P for b in boundary])
        for rep in range(3):
            fld = lambda q, x, y, z, rep=rep: no.hash_field(q, x, y, z) + rep  # noqa: E731
            od.fill(fld)
            for di, d in enumerate(dd.domains()):
                for q in range(len(dtypes)):
                    d.quantity_from_host(q, od.arrays[dd.domain_idx_[di]][q])
            td.barrier()
            dd.exchange()
            od.exchange()
            bo.apply_boundary(od, bcs)
            for di, d in enumerate(dd.domains()):
                for q in range(len(dtypes)):
                    got, want = d.quantity_to_host(q), od.arrays[dd.domain_idx_[di]][q]
                    assert np.array_equal(got, want), (rank, size, boundary, rep, q, int(np.count_nonzero(got != want)))
            td.barrier()
            dd.swap()
        dd.close()
    td.barrier()
    if rank == 0:
        print(f"mp_boundary_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
