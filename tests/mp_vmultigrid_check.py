"""stencil_b200.Multigrid with coefficient fields across processes.  Two modes over the same seeded right-hand side,
kappa and partition of the grid into N subdomains:
    python tests/mp_vmultigrid_check.py --single N OUT.json             one process, N subdomains: checks every cycle
                                                                        against the numpy cycle (tests/vmg_oracle.py)
                                                                        and writes the bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29631 \\
        tests/mp_vmultigrid_check.py --expect OUT.json                  one subdomain per rank: the gathered global result
                                                                        must equal the file's bits on every rank
Runs three queued V(2,2) cycles over 4 levels (32^3 .. 4^3) of -div(kappa grad u) + sigma u = f, kappa smooth on faces
(EVEN walls), sigma a cell field (VALUE walls), u with ODD(c) walls (a different c on each face), in float and double,
then update_coefficients() after kappa is scaled and solve() to 1e-6 (double) or 1e-3 (float).  Ranks share GPUs when
there are fewer GPUs than ranks."""
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
import vmg_oracle as vm  # noqa: E402
from mp_mg_check import gather  # noqa: E402
from mp_stencil_check import load  # noqa: E402

SIZE = (32, 32, 32)
WALLS = {0: ("odd", 0.0), 1: ("odd", 0.25), 2: ("odd", -0.5), 3: ("odd", 1.0), 4: ("odd", 0.125), 5: ("odd", -1.0)}
KWALLS = [{f: ("even", 0.0) for f in range(6)} for _ in range(3)] + [{f: ("value", 2.0) for f in range(6)}]
KINDS = ("x", "y", "z", "cell")


def A_at(l):
    return vm.helmholtz_div_grad(2.0 ** l / SIZE[0], sigma_field=True)


def run(gpus, world, check_oracle):
    out = {}
    for dtype in (np.float64, np.float32):
        dtype = np.dtype(dtype)
        dd = sb.DistributedDomain(*SIZE)
        dd.set_gpus(gpus)
        dd.set_radius(sb.Radius.constant(1))
        u, f, r = (dd.add_data(dtype, n) for n in ("u", "f", "r"))
        ks = [dd.add_data(dtype, n) for n in ("kx", "ky", "kz", "sigma")]
        dd.set_boundary(sb.Boundary.FIXED)
        for fc, (_, c) in WALLS.items():
            dd.set_boundary_condition(u, sb.FACES[fc], sb.BC.ODD(c))
        for k, w in zip(ks, KWALLS):
            for fc, (kind, c) in w.items():
                dd.set_boundary_condition(k, sb.FACES[fc], sb.BC.EVEN() if kind == "even" else sb.BC.VALUE(c))
        dd.realize()
        kp = vm.kappa_faces(SIZE, 1.0 / SIZE[0], "smooth", dtype)
        kp.append(np.random.default_rng(3).uniform(0.5, 2.0, tuple(n + 2 for n in SIZE[::-1])).astype(dtype))
        for q, a in zip(ks, kp):
            load(dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1]))
        fh = np.random.default_rng(32).uniform(-1, 1, SIZE[::-1]).astype(dtype)
        load(dd, f.id, "curr", fh)
        load(dd, u.id, "curr", np.zeros(SIZE[::-1], dtype))
        mg = sb.Multigrid(dd, u, f, r, lambda l: sb.StencilOp(A_at(l), dtype), levels=4, coefs=ks, coef_kinds=KINDS)
        if check_oracle:
            ref = vm.hierarchy(SIZE, 4, A_at, dtype, (False,) * 3, WALLS, [dict(w) for w in KWALLS])
            ref[0].interior(ref[0].f)[...] = fh
            for a, b in zip(ref[0].k, kp):
                a[...] = b
            vm.update_coefficients(ref, KINDS)
        for cyc in range(3):
            mg.cycle()
            got = gather(dd, u.id, world)
            if check_oracle:
                vm.vcycle(ref)
                want = np.ascontiguousarray(ref[0].interior(ref[0].u))
                assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), f"{dtype.name} cycle {cyc}: bits differ from the oracle"
            out[f"cycle{cyc}_{dtype.name}"] = hashlib.sha256(got.tobytes()).hexdigest()
        for q, a in zip(ks[:3], kp[:3]):
            load(dd, q.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1] * dtype.type(1.5)))
        mg.update_coefficients()
        rtol = 1e-6 if dtype == np.float64 else 1e-3
        hist = mg.solve(rtol, 25)
        assert hist[-1] <= rtol * dd.reduce(f, "curr", exact=True).l2(), hist
        out[f"solve_{dtype.name}"] = [float(h).hex() for h in hist]
        mg.close()
        dd.close()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n, 1, True), f)
        print("mp_vmultigrid_check single OK", flush=True)
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
        print(f"mp_vmultigrid_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
