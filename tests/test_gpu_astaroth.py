"""GPU parity of the astaroth solve<step> kernels (stencil_b200/csrc/astaroth.cu) against the CPU oracle
(oracle/astaroth_oracle.c), against golden vectors produced by the REFERENCE's own kernels
(tests/golden/astaroth_solve_ref.npz), and through DistributedDomain (interior || exchange -> exterior, 3 substeps,
swap) against the oracle's single-address-space exchange.  Floating point: every result is compared with the long double
oracle under the rounding budget of astaroth_util (K times the error of the same-precision oracle, plus a few ulps)."""
import os

import numpy as np
import pytest

import stencil_b200 as sb
from astaroth_util import GOLDEN, assert_within, budgets, cached_reference, make_fields, reference_substeps
from gpu_util import DevArray
from oracle import c_oracle as co
from oracle import geometry as g
from oracle import np_oracle as no
from stencil_b200 import astaroth as ac

pytestmark = pytest.mark.gpu


def tma_applies(dtype, raw) -> bool:
    """The TMA-fed team kernel needs FP64 and rows that are a multiple of 16 bytes (an even number of doubles)."""
    return np.dtype(dtype) == np.float64 and raw[0] % 2 == 0


def run_gpu(step, fin, fout, lo, hi, params, variant, lead=0):
    """fin / fout: lists of 8 host arrays; returns the 8 updated `out` arrays.  lead: byte offset of every field from
    the start of its (256-byte aligned) device block."""
    if variant in (ac.TEAM_TMA, ac.TEAM3_TMA) and not tma_applies(fin[0].dtype, fin[0].shape[::-1]):
        pytest.skip("TMA-fed kernel: FP64 with an even row length only")
    din = [DevArray(a, lead=lead) for a in fin]
    dout = [DevArray(a, lead=lead) for a in fout]
    mz, my, mx = fin[0].shape
    ac.substep(step, [d.ptr for d in din], [d.ptr for d in dout], fin[0].dtype.itemsize, (mx, my, mz), lo, hi, params, variant)
    res = [d.get() for d in dout]
    for d in din + dout:
        d.free()
    return res


def run_substeps(fields, ref, lo, hi, params, variant, lead=0):
    """Three substeps into the same `out` (like the driver: no swap in between), each checked against the long double
    oracle under its budget; then nothing outside the box may have changed."""
    fin, fout = fields[:8], fields[8:]
    cur = [a.copy() for a in fout]
    for step in range(3):
        cur = run_gpu(step, fin, cur, lo, hi, params, variant, lead)
        ext, budget = ref[step]
        assert_within(cur, ext, budget, f"step {step}", ac.FIELDS)
    for a, b in zip(cur, fout):
        m = np.ones(a.shape, dtype=bool)
        m[lo[2] : hi[2], lo[1] : hi[1], lo[0] : hi[0]] = False
        assert np.array_equal(a[m], b[m])
    return cur


BOXES = [
    # raw size (x,y,z), lo, hi
    ((38, 34, 30), (3, 3, 3), (35, 31, 27)),  # the whole compute region, partial tiles in x and y
    ((70, 26, 41), (3, 3, 3), (67, 23, 38)),
    ((40, 40, 40), (6, 6, 6), (34, 34, 34)),  # an interior region
    ((40, 40, 40), (3, 3, 3), (6, 37, 37)),  # x-face exterior slab (thin -> cell kernel under AUTO)
    ((40, 40, 40), (6, 34, 3), (34, 37, 37)),  # y-face slab
    ((40, 40, 40), (6, 6, 34), (34, 34, 37)),  # z-face slab
    ((23, 22, 21), (5, 4, 3), (16, 17, 18)),
]


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("variant", [ac.AUTO, ac.CELL, ac.TILE, ac.TEAM, ac.TEAM_TMA, ac.TEAM3_TMA])
@pytest.mark.parametrize("box", BOXES, ids=[f"{b[0]}-{b[1]}-{b[2]}" for b in BOXES])
def test_substeps_match_oracle(dtype, variant, box):
    raw, lo, hi = box
    fields, ref = cached_reference(raw, lo, hi, 7, np.dtype(dtype).name, "conf")
    run_substeps(fields, ref, lo, hi, ac.conf_params(dt=1e-3), variant)


@pytest.mark.parametrize("variant", [ac.CELL, ac.TILE, ac.TEAM, ac.TEAM_TMA, ac.TEAM3_TMA])
@pytest.mark.parametrize("shape", [0, 1])
def test_tile_shapes_and_zchunks(variant, shape, monkeypatch):
    """Both tile shapes per precision (SB_AC_SHAPE) and a forced short z chunk (ring warm-up at every chunk start)."""
    monkeypatch.setenv("SB_AC_SHAPE", str(shape))
    monkeypatch.setenv("SB_AC_ZCHUNK", "5")
    for dtype in (np.float64, np.float32):
        if variant in (ac.TEAM_TMA, ac.TEAM3_TMA) and dtype == np.float32:
            continue
        raw, lo, hi = (50, 45, 29), (3, 3, 3), (47, 42, 26)
        fields, ref = cached_reference(raw, lo, hi, 11, np.dtype(dtype).name, "conf")
        run_substeps(fields, ref, lo, hi, ac.conf_params(dt=1e-3), variant)


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="golden vectors not generated yet (oracle/ref/make_astaroth_golden.py)")
@pytest.mark.parametrize("variant", [ac.CELL, ac.TILE, ac.TEAM, ac.TEAM_TMA, ac.TEAM3_TMA])
def test_matches_reference_kernel_golden(variant):
    """The reference's own solve<0,1,2> (astaroth/kernels.cu, compiled unmodified) produced these."""
    z = np.load(GOLDEN)
    n, dt = int(z["n"]), float(z["dt"])
    check_golden(z["inputs"], z["outputs"], (n + 6,) * 3, co.astaroth_conf_params(dt), ac.conf_params(dt=dt), variant)


def check_golden(inputs, outputs, raw, op, params, variant):
    """The kernel and the reference's kernel each within the FP64 budget of the long double oracle, so within twice it
    of each other."""
    fin = [np.ascontiguousarray(inputs[f]) for f in range(8)]
    cur = [np.ascontiguousarray(inputs[8 + f]) for f in range(8)]
    lo, hi = (3, 3, 3), tuple(r - 3 for r in raw)
    ref = reference_substeps(fin, cur, lo, hi, op)
    c = (slice(3, -3),) * 3
    for step in range(3):
        cur = run_gpu(step, fin, cur, lo, hi, params, variant)
        ext, budget = ref[step]
        assert_within(cur, ext, budget, f"golden step {step}", ac.FIELDS)
        assert_within([a[c] for a in cur], [outputs[step, f] for f in range(8)], [2 * b for b in budget], f"golden step {step}", ac.FIELDS)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("ndom", [1, 2])
@pytest.mark.parametrize("overlap", [True, False])
@pytest.mark.parametrize("variant", [ac.AUTO, ac.TEAM])
def test_iteration_through_distributed_domain(dtype, ndom, overlap, variant):
    """astaroth/astaroth.cu:551-640: per substep interior || exchange -> exterior; swap after the third.  Two
    iterations on 24x20x28 split over `ndom` subdomains, against oracle exchange + oracle solve."""
    import torch

    size = (24, 20, 28)
    ng = torch.cuda.device_count()
    dd = sb.DistributedDomain(*size)
    dd.set_gpus([i % ng for i in range(ndom)])
    dd.set_radius(3)
    handles = [dd.add_data(dtype, name) for name in ac.FIELDS]
    dd.realize()
    try:
        glob = make_fields(size, seed=3, dtype=dtype)
        # (LocalDomain places FP64 r=3 allocations 8 bytes into their block: the TMA-fed kernel's shifted tensor base)
        sim = ac.Astaroth(dd, handles, ac.conf_params(dt=1e-3), overlap=overlap, variant=variant)
        check_iterations(dd, sim, glob, co.astaroth_conf_params(1e-3), ndom)
    finally:
        dd.close()


def check_iterations(dd, sim, glob, op, ndom, iterations=2):
    """Seeds `dd` with `glob` (16 arrays over the GLOBAL compute region: curr then next), runs `iterations` of `sim`,
    and compares every subdomain with the oracle's exchange + substeps run in long double and in the fields' precision
    (which sets the budget)."""
    size = tuple(glob[0].shape[::-1])
    dtype = glob[0].dtype
    ro = g.Radius.constant(3)
    sides = {}
    for t in (dtype, np.longdouble):
        od = no.Domains(size, ro, [t] * 8, n_subdomains=ndom)
        sides[t] = (od, {i: [np.zeros_like(a) for a in od.arrays[i]] for i in od.indices})
    for di, d in enumerate(dd.domains()):
        i = dd.domain_idx_[di]
        o, sz = sides[dtype][0].origins[i], sides[dtype][0].sizes[i]
        for q in range(8):
            for which, src in (("curr", glob[q]), ("next", glob[8 + q])):
                host = np.zeros(tuple(reversed(d.raw_size())), dtype=dtype)
                no.box(host, (3, 3, 3), sz)[...] = src[o[2] : o[2] + sz[2], o[1] : o[1] + sz[1], o[0] : o[0] + sz[0]]
                d.quantity_from_host(q, host, which)
                for t, (od, nxt) in sides.items():
                    (od.arrays[i] if which == "curr" else nxt[i])[q][...] = host
    for it in range(iterations):
        sim.step()
        for od, nxt in sides.values():
            for sub in range(3):
                od.exchange()
                for i in od.indices:
                    sz = od.sizes[i]
                    co.astaroth_substep(sub, od.arrays[i], nxt[i], (3, 3, 3), (3 + sz[0], 3 + sz[1], 3 + sz[2]), op)
            for i in od.indices:
                od.arrays[i], nxt[i] = nxt[i], od.arrays[i]
    od, odx = sides[dtype][0], sides[np.longdouble][0]
    for di, d in enumerate(dd.domains()):
        i = dd.domain_idx_[di]
        sz = od.sizes[i]
        got = [no.box(d.quantity_to_host(q), (3, 3, 3), sz) for q in range(8)]
        same = [no.box(od.arrays[i][q], (3, 3, 3), sz) for q in range(8)]
        ext = [no.box(odx.arrays[i][q], (3, 3, 3), sz) for q in range(8)]
        assert_within(got, ext, budgets(same, ext, dtype), f"domain {i}", ac.FIELDS)
