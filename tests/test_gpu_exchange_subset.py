"""GPU tests of exchange(only=...) and of exchange="reads" (DESIGN.md section 2.15).  With every ghost cell poisoned
(NaN, or 0x5A for integer quantities), a subset exchange gives each quantity of the subset the bits the full exchange
gives it, walls and boundary conditions included, and leaves every byte of the other quantities, ghost cells included,
as it was: on 1, 2, 3, 4 and 8 subdomains, float32, int8 and float64, radius 0, 1, 2, face-edge-corner and
asymmetric, after swap(), under SB_ALLOC_ALIGN=0 and 1, and on two GPUs where the machine has them.  apply, relax,
apply_system, the fused residual-restriction and prolong_from give the same outputs with exchange="reads" as with
exchange=True; the solvers' internal exchanges are subsets."""
import numpy as np
import pytest
import torch

import stencil_b200 as sb
from oracle import np_oracle as no
from stencil_b200.multigrid import residual_op
from test_gpu_stencil_domain import gather, load, same

pytestmark = pytest.mark.gpu

P, F = sb.Boundary.PERIODIC, sb.Boundary.FIXED
PARTS = [1, 2, 3, 4, 8]
DTYPES = [np.float32, np.int8, np.float64, np.float32]


def radius(name):
    if name.startswith("c"):
        return sb.Radius.constant(int(name[1:]))
    if name == "f2e1c1":
        return sb.Radius.face_edge_corner(2, 1, 1)
    r = sb.Radius.constant(0)  # asymmetric: 2 cells towards +x, 1 towards -x and +y
    r.set_dir((1, 0, 0), 2)
    r.set_dir((-1, 0, 0), 1)
    r.set_dir((0, 1, 0), 1)
    return r


def make(ndom, rname, walls, gpus=None):
    dd = sb.DistributedDomain(24, 18, 20)
    dd.set_gpus(gpus or [0] * ndom)
    dd.set_radius(radius(rname))
    hs = [dd.add_data(dt, f"q{i}") for i, dt in enumerate(DTYPES)]
    if walls:
        dd.set_boundary(F, P, F)
        for q, h in enumerate(hs):
            for f in (0, 1, 4, 5):
                if np.dtype(DTYPES[q]).kind == "f":
                    bc = [sb.BC.ODD(0.25 * q), sb.BC.EVEN(), sb.BC.VALUE(-1.5), sb.BC.ODD(0.0)][(q + f) % 4]
                else:
                    bc = sb.BC.EVEN()
                dd.set_boundary_condition(h, sb.FACES[f], bc)
    dd.realize()
    return dd, hs


def poisoned(d, q, seed):
    """Quantity q of local subdomain d: hashed compute cells, every ghost cell poisoned."""
    dt = np.dtype(DTYPES[q])
    raw, sz, r = d.raw_size(), d.size(), d.radius()
    lo = (r.x(-1), r.y(-1), r.z(-1))
    a = np.full(raw[::-1], np.nan if dt.kind == "f" else 0x5A, dt)
    org = d.origin()
    zz, yy, xx = np.meshgrid(*[np.arange(org[k], org[k] + sz[k]) for k in (2, 1, 0)], indexing="ij")
    a[lo[2] : lo[2] + sz[2], lo[1] : lo[1] + sz[1], lo[0] : lo[0] + sz[0]] = (no.hash_field(q, xx, yy, zz) % 101 + seed).astype(dt)
    return a


def load_all(dd, seed):
    for d in dd.domains():
        for q in range(len(DTYPES)):
            d.quantity_from_host(q, poisoned(d, q, seed))


def snapshot(dd):
    return [[d.quantity_to_host(q).view(np.uint8).copy() for q in range(len(DTYPES))] for d in dd.domains()]


def check_subsets(dd, hs, subsets, seed=0):
    load_all(dd, seed)
    dd.exchange()
    full = snapshot(dd)
    for sub in subsets:
        load_all(dd, seed)
        before = snapshot(dd)
        dd.exchange(only=[hs[q] for q in sub])
        got = snapshot(dd)
        for di in range(len(dd.domains())):
            for q in range(len(DTYPES)):
                want = full[di][q] if q in sub else before[di][q]
                assert np.array_equal(got[di][q], want), (sub, dd.domain_idx_[di], q)


SUBSETS = [(0,), (1,), (2,), (0, 2), (1, 3), (0, 1, 2, 3)]


@pytest.mark.parametrize("walls", [False, True])
@pytest.mark.parametrize("rname", ["c0", "c1", "c2", "f2e1c1", "asym"])
@pytest.mark.parametrize("ndom", PARTS)
def test_subset_exchange_moves_only_the_subset(ndom, rname, walls):
    dd, hs = make(ndom, rname, walls)
    try:
        check_subsets(dd, hs, SUBSETS)
        dd.swap()  # the other parity's plans
        check_subsets(dd, hs, [(0,), (1, 2)], seed=3)
    finally:
        dd.close()


@pytest.mark.parametrize("align", ["0", "1"])
def test_subset_exchange_alloc_align(align, monkeypatch):
    monkeypatch.setenv("SB_ALLOC_ALIGN", align)
    dd, hs = make(4, "c2", True)
    try:
        check_subsets(dd, hs, SUBSETS)
    finally:
        dd.close()


def test_subset_exchange_two_gpus_if_available():
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    for gpus in ([0, 1], [0, 1, 0, 1]):
        dd, hs = make(len(gpus), "c2", True, gpus)
        try:
            check_subsets(dd, hs, SUBSETS)  # staged thin rows: the subset's entries at the full layout's offsets
        finally:
            dd.close()


def test_subset_plans_are_cached_and_the_full_set_is_the_full_plan():
    dd, hs = make(4, "c1", True)
    try:
        dd.exchange(only=[hs[1], hs[0]])
        assert set(dd._subset_plans) == {(0, (0, 1))}
        dd.exchange(only=[hs[0], hs[1]])
        assert set(dd._subset_plans) == {(0, (0, 1))}
        dd.exchange(only=hs)
        assert set(dd._subset_plans) == {(0, (0, 1))}  # every quantity: the full plan
        assert dd.exchange_bytes([hs[0]]) < dd.exchange_bytes()
        assert dd.exchange_bytes(hs) == dd.exchange_bytes()
        with pytest.raises(sb.StencilError, match="names no quantity"):
            dd.exchange(only=[])
        with pytest.raises(sb.StencilError, match="named twice"):
            dd.exchange(only=[hs[0], hs[0]])
        other, ohs = make(1, "c1", False)
        try:
            with pytest.raises(sb.StencilError, match="not a DataHandle of this domain"):
                dd.exchange(only=[ohs[0]])
        finally:
            other.close()
    finally:
        dd.close()


# ------------------------------------------------------------------------------------------- exchange="reads"
def op_domain(ndom, nq, boundary=(P, P, P), wall_bc=None, size=(24, 20, 18)):
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([0] * ndom)
    dd.set_radius(sb.Radius.constant(1))
    hs = [dd.add_data(np.float64, f"q{i}") for i in range(nq)]
    dd.set_boundary(*boundary)
    if wall_bc is not None:
        for h in hs:
            for f in range(6):
                if boundary[f // 2] == F:
                    dd.set_boundary_condition(h, sb.FACES[f], wall_bc)
    dd.realize()
    return dd, hs


def fields(dd, nq, seed):
    rng = np.random.default_rng(seed)
    return [rng.uniform(0.5, 1.5, dd.size()[::-1]) for _ in range(nq)]


def both_ways(dd, hs, glob, call, outs):
    """call(exchange) on inputs reloaded with NaN ghost cells, once with True and once with "reads": same outputs."""
    res = []
    for ex in (True, "reads"):
        for q, g in enumerate(glob):
            load(dd, q, "curr", g)
            load(dd, q, "next", g)
        call(ex)
        res.append([gather(dd, q, w) for q, w in outs])
    for a, b in zip(*res):
        assert same(a, b)
        assert not np.isnan(a).any()


@pytest.mark.parametrize("ndom", PARTS)
@pytest.mark.parametrize("boundary", [(P, P, P), (F, P, F)])
def test_reads_matches_true(ndom, boundary):
    dd, hs = op_domain(ndom, 7, boundary, sb.BC.ODD(0.5))
    glob = fields(dd, 7, ndom)
    u, f, kx, ky, kz, out, w = hs
    try:
        lap = sb.StencilOp.laplacian(2, (1.0, 1.0, 1.0), np.float64)
        dg = sb.StencilOp.div_grad((1.0, 1.0, 1.0), np.float64).scaled(-1.0)
        # the read sets exchange="reads" moves
        assert dd._exchange_sel("apply", "reads", [u.id] + sb.domain.op_moved_coefs(dg, [kx.id, ky.id, kz.id])) == (0, 2, 3, 4)
        both_ways(dd, hs, glob, lambda ex: dd.apply(lap, out, u, exchange=ex), [(out.id, "next")])
        both_ways(dd, hs, glob, lambda ex: dd.apply(dg, out, u, coefs=[kx, ky, kz], exchange=ex), [(out.id, "next")])
        both_ways(dd, hs, glob, lambda ex: [dd.relax(dg, (u, "curr"), u, f, coefs=[kx, ky, kz], colour=(2, c), exchange=ex) for c in range(2)],
                  [(u.id, "curr")])
        both_ways(dd, hs, glob, lambda ex: dd.relax(lap.scaled(-1.0), out, u, f, exchange=ex), [(out.id, "next")])
        sysop = sb.StencilSystem.grad(1, (1.0, 1.0, 1.0), np.float64)
        assert sysop.moved_inputs() == {0}
        both_ways(dd, hs, glob, lambda ex: dd.apply_system(sysop, [out, w, (kx, "next")], [u], exchange=ex),
                  [(out.id, "next"), (w.id, "next"), (kx.id, "next")])
    finally:
        dd.close()


@pytest.mark.parametrize("ndom", [1, 2, 4, 8])
def test_reads_matches_true_for_transfers(ndom):
    fine, fhs = op_domain(ndom, 6, (F, F, F), sb.BC.ODD(0.0), (24, 20, 16))
    coarse = sb.DistributedDomain(12, 10, 8)
    coarse.set_gpus([0] * ndom)
    coarse.set_radius(sb.Radius.constant(1))
    chs = [coarse.add_data(np.float64, f"c{i}") for i in range(3)]
    coarse.set_boundary(F, F, F)
    for h in chs:
        for fc in range(6):
            coarse.set_boundary_condition(h, sb.FACES[fc], sb.BC.ODD(0.0))
    coarse.realize()
    try:
        u, f, kx, ky, kz, _ = fhs
        res = residual_op(sb.StencilOp.div_grad((1.0, 1.0, 1.0), np.float64).scaled(-1.0))
        gf, gc = fields(fine, 6, 1), fields(coarse, 3, 2)

        def restrict(ex):
            for q, g in enumerate(gc):
                load(coarse, q, "curr", g)
            fine.restrict_to(coarse, (chs[0], "curr"), (u, "curr"), op=res, aux=(f, "curr"), coefs=[kx, ky, kz], exchange=ex)

        outs = {}
        for ex in (True, "reads"):
            for q, g in enumerate(gf):
                load(fine, q, "curr", g)
            restrict(ex)
            outs[ex] = gather(coarse, chs[0].id)
        assert same(outs[True], outs["reads"]) and not np.isnan(outs[True]).any()
        for ex in (True, "reads"):
            for q, g in enumerate(gf):
                load(fine, q, "curr", g)
            for q, g in enumerate(gc):
                load(coarse, q, "curr", g)
            fine.prolong_from(coarse, (u, "curr"), (chs[1], "curr"), aux=(u, "curr"), exchange=ex)
            outs[ex] = gather(fine, u.id)
        assert same(outs[True], outs["reads"]) and not np.isnan(outs[True]).any()
    finally:
        coarse.close()
        fine.close()


@pytest.mark.parametrize("ndom", [1, 4])
def test_pcg_exchanges_subsets_and_keeps_its_bits(ndom):
    """The jump-kappa PCG of test_gpu_krylov gives the oracle's bits, and its exchanges are subsets: x, the vector A is
    applied to, u on every level and the coefficient fields; no cycle exchanges every quantity."""
    import test_gpu_krylov as tk

    s = tk.Setup(tk.fine_size(ndom), [0] * ndom, "jump-kvalue-f64")
    try:
        tk.run_bits(s, iters=2)
        fine = {qs for _, qs in s.dd._subset_plans}
        assert fine == {(s.x.id,), (s.p.id,), (s.z.id,), tuple(k.id for k in s.ks)}, fine
        for L in s.cg.mg.levels[1:]:
            assert {qs for _, qs in L.dd._subset_plans} == {(L.u.id,), tuple(k.id for k in L.coefs)}
    finally:
        s.close()
