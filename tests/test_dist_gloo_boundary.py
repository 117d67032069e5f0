"""world_size-2 and -4 `gloo` tests (CPU) of the one-process-per-GPU planning on non-periodic grids: rank -> subdomain
ownership, each rank's send plan equals the oracle's wall-aware plan (tests/bc_oracle.py) restricted to that rank, no
message crosses a wall, executing every rank's plan gives the oracle's exchange, and the neighbour-rank relation stays
symmetric.  Data is moved by numpy; the planning under test is the product's (DistributedDomain.plan_messages and
dist.messages_from over the C ABI)."""
import os
import socket
import sys

import numpy as np
import pytest
import torch.distributed as td
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, size, rname, walls, out_q):
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
        td.init_process_group("gloo", rank=rank, world_size=world)
        import bc_oracle as bo
        import stencil_b200 as sb
        from gpu_util import oracle_radius
        from oracle import np_oracle as no
        from stencil_b200 import dist

        P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
        boundary = tuple(F if c == "F" else P for c in walls)
        periodic = [b == P for b in boundary]
        radius = {"c1": sb.Radius.constant(1), "c2": sb.Radius.constant(2), "f2e1": sb.Radius.face_edge_corner(2, 1, 0)}[rname]
        dtypes = [np.float32, np.float64]
        dd = sb.DistributedDomain(*size)
        dd.set_gpus([0])  # one subdomain per rank
        dd.set_radius(radius)
        for dt in dtypes:
            dd.add_data(dt)
        dd.set_boundary(*boundary)
        dd.do_placement()  # no GPU needed: partition + ownership only
        msgs = dd.plan_messages()
        od = bo.Domains(size, oracle_radius(radius), dtypes, n_subdomains=world, periodic=periodic)
        mine = [i for i in od.indices if dd._owner[i][0] == rank]
        assert len(mine) == 1 and all(m["src_idx"] == mine[0] for m in msgs)
        keys = ("src_idx", "dst_idx", "dir", "src_pos", "dst_pos", "ext")
        want = [m for m in bo.plan_sends(od.dim, od.sizes, od.radius, periodic) if m["src_idx"] == mine[0]]
        key = lambda m: m["dir"]  # noqa: E731
        assert sorted(({k: m[k] for k in keys} for m in msgs), key=key) == sorted(want, key=key)
        assert sorted(({k: m[k] for k in keys} for m in dist.messages_from(dd, rank)), key=key) == sorted(want, key=key)
        od.fill(no.hash_field)
        outbox = []
        for m in msgs:
            for q in range(len(dtypes)):
                outbox.append((m["dst_idx"], m["dst_rank"], q, m["dst_pos"], m["ext"], no.pack(od.arrays[mine[0]][q], m["src_pos"], m["ext"])))
        everyone = [None] * world
        td.all_gather_object(everyone, outbox)
        for box in everyone:
            for dst_idx, dst_rank, q, dst_pos, ext, payload in box:
                if dst_rank == rank:
                    no.unpack(od.arrays[mine[0]][q], payload, dst_pos, ext)
        for q in range(len(dtypes)):
            assert np.array_equal(od.arrays[mine[0]][q], od.expected_after_exchange(no.hash_field, mine[0], q)), (rank, q)
        nb = sorted({m["dst_rank"] for m in msgs} - {rank})
        allnb = [None] * world
        td.all_gather_object(allnb, nb)
        for r, lst in enumerate(allnb):
            for o in lst:
                assert r in allnb[o]
        td.barrier()
        td.destroy_process_group()
        out_q.put((rank, "ok"))
    except Exception:  # pragma: no cover
        import traceback

        out_q.put((rank, "FAIL: " + traceback.format_exc()))


@pytest.mark.parametrize(
    "world,size,rname,walls",
    [(2, (10, 10, 10), "c1", "FFF"), (2, (13, 9, 8), "c2", "PPF"), (4, (12, 10, 14), "f2e1", "FPP"), (4, (16, 16, 16), "c2", "FPF")],
)
def test_multi_process_plans_with_walls_over_gloo(world, size, rname, walls):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, size, rname, walls, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(results) == [(r, "ok") for r in range(world)], results
