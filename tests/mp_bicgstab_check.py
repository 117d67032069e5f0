"""stencil_b200.BiCGStab across processes.  Two modes over the same seeded right-hand side, kappa and partition of the
grid into N subdomains:
    python tests/mp_bicgstab_check.py --single N OUT.json               one process, N subdomains: checks every iteration
                                                                        against the numpy solver (tests/bicgstab_oracle.py)
                                                                        and writes the bits
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29661 \\
        tests/mp_bicgstab_check.py --expect OUT.json                    one subdomain per rank: the gathered global result
                                                                        must equal the file's bits on every rank
Runs 1, 2 and 3 iterations of multigrid-preconditioned BiCGStab over 4 levels (32^3 .. 4^3) of -div(kappa grad x) +
b . grad x + sigma x = f, kappa smooth on faces (EVEN walls), sigma a cell field (VALUE walls), x with ODD(c) walls (a
different c on each face), in float and double, then solve() to 1e-8 (double) or 1e-4 (float).  Ranks share GPUs when
there are fewer GPUs than ranks."""
import hashlib
import json
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bicgstab_oracle as bo  # noqa: E402
import krylov_oracle as ko  # noqa: E402
import stencil_b200 as sb  # noqa: E402
import vmg_oracle as vm  # noqa: E402
from mp_mg_check import gather  # noqa: E402
from mp_stencil_check import load  # noqa: E402

SIZE = (32, 32, 32)
WALLS = {0: ("odd", 0.0), 1: ("odd", 0.25), 2: ("odd", -0.5), 3: ("odd", 1.0), 4: ("odd", 0.125), 5: ("odd", -1.0)}
KWALLS = [{f: ("even", 0.0) for f in range(6)} for _ in range(3)] + [{f: ("value", 2.0) for f in range(6)}]
KINDS = ("x", "y", "z", "cell")


B = (4.0, 2.4, 1.2)


def A_at(l):
    h = 2.0**l / SIZE[0]
    conv = [(0, tuple(s * (a == j) for j in range(3)), s * B[a] / (2 * h)) for a in range(3) for s in (1, -1)]
    return vm.helmholtz_div_grad(h, sigma_field=True) + conv


def run(gpus, world, check_oracle):
    out = {}
    for dtype in (np.float64, np.float32):
        dtype = np.dtype(dtype)
        dd = sb.DistributedDomain(*SIZE)
        dd.set_gpus(gpus)
        dd.set_radius(sb.Radius.constant(1))
        V = {n: dd.add_data(dtype, n) for n in sb.BiCGStab.NAMES}
        x, f = V["x"], V["f"]
        ks = [dd.add_data(dtype, n) for n in ("kx", "ky", "kz", "sigma")]
        dd.set_boundary(sb.Boundary.FIXED)
        for fc, (_, c) in WALLS.items():
            dd.set_boundary_condition(x, sb.FACES[fc], sb.BC.ODD(c))
            dd.set_boundary_condition(V["phat"], sb.FACES[fc], sb.BC.ODD(0.0))
            dd.set_boundary_condition(V["shat"], sb.FACES[fc], sb.BC.ODD(0.0))
        for k, w in zip(ks, KWALLS):
            for fc, (kind, c) in w.items():
                dd.set_boundary_condition(k, sb.FACES[fc], sb.BC.EVEN() if kind == "even" else sb.BC.VALUE(c))
        dd.realize()
        kp = vm.kappa_faces(SIZE, 1.0 / SIZE[0], "smooth", dtype)
        kp.append(np.random.default_rng(3).uniform(0.5, 2.0, tuple(n + 2 for n in SIZE[::-1])).astype(dtype))
        for h, a in zip(ks, kp):
            load(dd, h.id, "curr", np.ascontiguousarray(a[1:-1, 1:-1, 1:-1]))
        fh = np.random.default_rng(41).uniform(-1, 1, SIZE[::-1]).astype(dtype)
        load(dd, f.id, "curr", fh)
        cg = sb.BiCGStab(dd, *(V[n] for n in sb.BiCGStab.NAMES), lambda l: sb.StencilOp(A_at(l), dtype), levels=4, coefs=ks, coef_kinds=KINDS)
        if check_oracle:
            lv = vm.hierarchy(SIZE, 4, A_at, dtype, (False,) * 3, ko.homogeneous(WALLS), [dict(w) for w in KWALLS])
            for a, b in zip(lv[0].k, kp):
                a[...] = b
            vm.update_coefficients(lv, KINDS)
            ref = bo.BiCGStab(lv, WALLS)
            ref.I(ref.f)[...] = fh
            hist_ref = [math.sqrt(ref.start())]
        for it in range(1, 4):
            load(dd, x.id, "curr", np.zeros(SIZE[::-1], dtype))
            hist = cg.solve(0.0, it)
            got = gather(dd, x.id, world)
            if check_oracle:
                assert ref.iterate(it - 1, 0.0, hist_ref)
                assert hist == hist_ref, f"{dtype.name} {it} iterations: history {hist} != oracle {hist_ref}"
                want = np.ascontiguousarray(ref.I(ref.x))
                assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), f"{dtype.name} {it} iterations: bits differ from the oracle"
            out[f"iter{it}_{dtype.name}"] = [hashlib.sha256(got.tobytes()).hexdigest()] + [float(h).hex() for h in hist]
        load(dd, x.id, "curr", np.zeros(SIZE[::-1], dtype))
        rtol = 1e-8 if dtype == np.float64 else 1e-4
        hist = cg.solve(rtol, 30)
        assert hist[-1] <= rtol * math.sqrt(dd.dot(f, f)) and cg.breakdown is None, hist
        out[f"solve_{dtype.name}"] = [float(h).hex() for h in hist]
        cg.close()
        dd.close()
    return out


def main():
    if sys.argv[1] == "--single":
        n = int(sys.argv[2])
        with open(sys.argv[3], "w") as f:
            json.dump(run([0] * n, 1, True), f)
        print("mp_bicgstab_check single OK", flush=True)
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
        print(f"mp_bicgstab_check OK: world={world}", flush=True)
    td.destroy_process_group()


if __name__ == "__main__":
    main()
