"""GPU parity of DistributedDomain.restrict_to / prolong_from: both transfers on 1, 2, 3 (96 x 32 x 32 cut along x), 4
and 8 subdomains of one GPU, periodic and walled (ODD and EVEN faces on the coarse grid), under SB_ALLOC_ALIGN=0 and 1,
bit-identical to tests/transfer_oracle.py; three V(2,2) cycles over 4 levels bit for bit against the numpy V-cycle
after every cycle on every partition; the h-independent convergence of the cycle on 64^3 .. 256^3 FP64 ODD(0) Poisson;
every pairing error; and the plan cache across swap()."""
import numpy as np
import pytest

import bc_oracle as bo
import mg_gpu
import stencil_b200 as sb
import stencil_op_oracle as so
import transfer_oracle as to
from gpu_util import oracle_radius
from test_gpu_stencil_domain import gather, lo_of, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
PARTS = [1, 2, 3, 4, 8]


def fine_size(ndom):
    return (96, 32, 32) if ndom == 3 else (32, 32, 32)


def pair(ndom, dtype, boundary=(P, P, P), bcs=None, size=None):
    """A fine domain (quantities u, v) and its coarsening (quantities e, w), radius 1 in all 26 directions; bcs apply to
    the coarse e."""
    size = size or fine_size(ndom)
    out = []
    for lvl, sz in enumerate((size, tuple(n // 2 for n in size))):
        dd = sb.DistributedDomain(*sz)
        dd.set_gpus([0] * ndom)
        dd.set_radius(sb.Radius.constant(1))
        hs = [dd.add_data(dtype), dd.add_data(dtype)]
        dd.set_boundary(*boundary)
        if lvl == 1:
            for fc, (kind, c) in (bcs or {}).items():
                dd.set_boundary_condition(hs[0], sb.FACES[fc], sb.BC(kind, c))
        dd.realize()
        out.append((dd, hs))
    return out


WALLS = {0: (bo.ODD, 0.0), 1: (bo.ODD, 0.25), 2: (bo.EVEN, 0.0), 3: (bo.EVEN, 0.0), 4: (bo.ODD, -0.5), 5: (bo.EVEN, 0.0)}


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("boundary", [(P, P, P), (F, F, F), (F, P, F)])
@pytest.mark.parametrize("align", ["1", "0"])
def test_transfers(ndom, dtype, boundary, align, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    dtype = np.dtype(dtype)
    size = fine_size(ndom)
    csize = tuple(n // 2 for n in size)
    bcs = {fc: v for fc, v in WALLS.items() if boundary[fc // 2] == F}
    (fd, (u, v)), (cd, (e, w)) = pair(ndom, dtype, boundary, bcs)
    try:
        rng = np.random.default_rng(ndom)
        fine = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        coarse = rng.uniform(-1, 1, csize[::-1]).astype(dtype)
        # restriction from curr and from next
        load(fd, u.id, "curr", fine)
        load(fd, v.id, "next", fine[::-1].copy())
        fd.restrict_to(cd, (w, "curr"), (u, "curr"))
        want = np.empty(csize[::-1], dtype)
        to.restrict_box(want, (0, 0, 0), fine, (0, 0, 0), (0, 0, 0), csize)
        assert same(gather(cd, w.id), want)
        fd.restrict_to(cd, w, (v, "next"))  # a bare dst handle is next
        to.restrict_box(want, (0, 0, 0), fine[::-1].copy(), (0, 0, 0), (0, 0, 0), csize)
        assert same(gather(cd, w.id, "next"), want)
        # prolongation: the coarse ghost cells from the exchange and the coarse BCs
        load(cd, e.id, "curr", coarse)
        od = bo.Domains(csize, oracle_radius(cd.radius_), [dtype], n_subdomains=1, periodic=[b == P for b in boundary])
        rl = lo_of(cd.radius_)
        so._view(od.arrays[(0, 0, 0)][0], rl, csize, (0, 0, 0))[...] = coarse
        od.exchange()
        bo.apply_boundary(od, {(0, fc): kv for fc, kv in bcs.items()})
        E, eo = od.arrays[(0, 0, 0)][0], tuple(-r for r in rl)
        base = rng.uniform(-1, 1, size[::-1]).astype(dtype)
        load(fd, u.id, "curr", base)
        fd.prolong_from(cd, (u, "curr"), (e, "curr"), aux=(u, "curr"))  # in place
        want = base.copy()
        to.prolong_box(want, (0, 0, 0), E, eo, (0, 0, 0), size, aux=want)
        assert same(gather(fd, u.id), want)
        fd.prolong_from(cd, v, e)  # no aux, into next
        want = np.empty(size[::-1], dtype)
        to.prolong_box(want, (0, 0, 0), E, eo, (0, 0, 0), size)
        assert same(gather(fd, v.id, "next"), want)
        cd.exchange()  # the caller guarantees the ghost cells
        fd.prolong_from(cd, (v, "curr"), (e, "curr"), aux=(u, "next"), exchange=False)
        aux = np.asarray(gather(fd, u.id, "next"))
        to.prolong_box(want, (0, 0, 0), E, eo, (0, 0, 0), size, aux=aux)
        assert same(gather(fd, v.id), want)
    finally:
        fd.close()
        cd.close()


def vcycle_case(ndom, dtype, walls):
    size = fine_size(ndom)
    periodic, sigma = ((False,) * 3, 0.0) if walls == "odd" else ((True,) * 3, 1.0)
    boundary = tuple(P if p else F for p in periodic)
    lv = mg_gpu.hierarchy(size, 4, sigma, dtype, boundary, [0] * ndom)
    ref = to.hierarchy(size, 4, sigma, dtype, periodic)
    try:
        f = np.random.default_rng(7).uniform(-1, 1, size[::-1]).astype(dtype)
        load(lv[0].dd, lv[0].f.id, "curr", f)
        ref[0].interior(ref[0].f)[...] = f
        for L in lv:
            load(L.dd, L.u.id, "curr", np.zeros(L.size[::-1], dtype))
        for cyc in range(3):
            mg_gpu.vcycle(lv)
            to.vcycle(ref)
            assert same(gather(lv[0].dd, lv[0].u.id), ref[0].interior(ref[0].u).copy()), cyc
    finally:
        mg_gpu.close(lv)


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("dtype,walls", [(np.float64, "odd"), (np.float32, "odd"), (np.float64, "periodic")])
def test_vcycle_bits(ndom, dtype, walls):
    """Three V(2,2) cycles over 4 levels (32^3 .. 4^3, or 96 x 32 x 32 .. 12 x 4 x 4), 30 coarsest sweeps: every
    component is partition-independent, so the whole cycle is, bit for bit against the numpy cycle."""
    vcycle_case(ndom, np.dtype(dtype), walls)


def test_vcycle_bits_reference_placement(monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", "0")
    vcycle_case(4, np.dtype(np.float64), "odd")


def test_vcycle_convergence_is_h_independent():
    """FP64 -lap u = f with ODD(0) walls, f uniform(-1, 1): V(2,2) cycles down to 4^3 on 64^3, 128^3 and 256^3.  After
    the first cycle each factor is <= 0.15, and the factor of each cycle differs by < 0.02 between the sizes."""
    fs = {}
    for n in (64, 128, 256):
        lv = mg_gpu.hierarchy((n, n, n), int(np.log2(n)) - 1, 0.0, np.float64, (F, F, F), [0])
        try:
            load(lv[0].dd, lv[0].f.id, "curr", np.random.default_rng(n).uniform(-1, 1, (n, n, n)))
            for L in lv:
                load(L.dd, L.u.id, "curr", np.zeros(L.size[::-1]))
            r = [lv[0].residual_norm()]
            for _ in range(5):
                mg_gpu.vcycle(lv)
                r.append(lv[0].residual_norm())
            fs[n] = [r[k + 1] / r[k] for k in range(5)]
        finally:
            mg_gpu.close(lv)
    for n, f in fs.items():
        assert max(f[1:]) <= 0.15, (n, f)
    for k in range(1, 5):
        vals = [fs[n][k] for n in fs]
        assert max(vals) - min(vals) < 0.02, (k, fs)


def test_pairing_errors():
    import torch

    def dom(size, ndom, radius=1, dtype=np.float64, gpus=None):
        dd = sb.DistributedDomain(*size)
        dd.set_gpus(gpus or [0] * ndom)
        dd.set_radius(sb.Radius.constant(radius) if isinstance(radius, int) else radius)
        h = dd.add_data(dtype)
        dd.realize()
        return dd, h

    made = []
    try:
        fine, u = dom((32, 32, 32), 2)
        made.append(fine)
        odd, e = dom((17, 16, 16), 2)  # an uneven cut: not twice as coarse everywhere
        made.append(odd)
        with pytest.raises(sb.StencilError, match="not twice the coarse|must be the same"):
            fine.restrict_to(odd, e, u)
        other_dim, e2 = dom((16, 16, 16), 4)
        made.append(other_dim)
        with pytest.raises(sb.StencilError, match="the coarse one"):
            fine.restrict_to(other_dim, e2, u)
        thin = sb.Radius.face_edge_corner(1, 1, 0)
        nocorner, e3 = dom((16, 16, 16), 2, thin)
        made.append(nocorner)
        fine.restrict_to(nocorner, e3, u)  # restriction reads no ghost cells
        with pytest.raises(sb.StencilError, match=r"coarse radius in direction \(-1, -1, -1\) is 0"):
            fine.prolong_from(nocorner, u, (e3, "curr"))
        f32, e4 = dom((16, 16, 16), 2, dtype=np.float32)
        made.append(f32)
        with pytest.raises(sb.StencilError, match="float32 or all float64"):
            fine.restrict_to(f32, e4, u)
        good, e5 = dom((16, 16, 16), 2)
        made.append(good)
        with pytest.raises(sb.StencilError, match="src must be a curr buffer"):
            fine.prolong_from(good, u, (e5, "next"))
        with pytest.raises(sb.StencilError, match="coarse must be another DistributedDomain"):
            fine.restrict_to(fine, u, u)
        with pytest.raises(sb.StencilError, match="must be a DataHandle"):
            fine.restrict_to(good, (e5, "both"), u)
        if torch.cuda.device_count() > 1:
            moved, e6 = dom((16, 16, 16), 2, gpus=[0, 1])
            made.append(moved)
            with pytest.raises(sb.StencilError, match="on GPU 0 on the fine level and GPU 1"):
                fine.restrict_to(moved, e6, u)
        else:
            pytest.skip("the mismatched-GPU case needs two GPUs; every other pairing error passed")
    finally:
        for d in made:
            d.close()


def test_plan_cache_across_swap():
    (fd, (u, v)), (cd, (e, w)) = pair(2, np.float64)
    try:
        rng = np.random.default_rng(3)
        size, csize = (32, 32, 32), (16, 16, 16)
        fine = [rng.uniform(-1, 1, size[::-1]) for _ in range(2)]
        load(fd, u.id, "curr", fine[0])
        load(fd, u.id, "next", fine[1])
        for k in range(4):
            fd.restrict_to(cd, (e, "curr"), (u, "curr"))
            want = np.empty(csize[::-1])
            to.restrict_box(want, (0, 0, 0), fine[k % 2], (0, 0, 0), (0, 0, 0), csize)
            assert same(gather(cd, e.id), want), k
            assert len(fd._transfer_plans) == min(k + 1, 2)
            fd.swap()
        assert len(fd._transfer_plans) == 2  # one per fine parity
        cd.swap()
        fd.restrict_to(cd, (e, "curr"), (u, "curr"))
        assert len(fd._transfer_plans) == 3  # the coarse parity is part of the key
        fd.restrict_to(cd, (e, "curr"), (u, "curr"))
        assert len(fd._transfer_plans) == 3
        fd.close()
        assert fd._transfer_plans == {} and fd._paired == set()
    finally:
        fd.close()
        cd.close()
