"""GPU parity of the jacobi kernels against the CPU oracle.  Bit-exact in FP32 and FP64: the kernel
uses the oracle's summation order and an exact IEEE division (stencil_b200/csrc/jacobi.cu), so the
tolerance is 0 ulp -- tighter than the 1e-6 relative BASELINE.json allows for the FP64 residual."""
import ctypes as C

import numpy as np
import pytest

import stencil_b200 as sb
from oracle import c_oracle as co
from oracle import geometry as g
from oracle import np_oracle as no
from stencil_b200._lib import check, i3, lib
from gpu_util import DevArray

pytestmark = pytest.mark.gpu


def gpu_jacobi(dst: DevArray, src: DevArray, acc_origin, lo, hi, clo, chi):
    check(lib().sb_jacobi3d(dst.pitched(), src.pitched(), src.dtype.itemsize, i3(acc_origin), i3(lo), i3(hi), i3(clo), i3(chi), None))


SHAPES = [
    # compute size (x,y,z), radius per side
    ((48, 48, 48), 1),
    ((64, 64, 64), 1),  # BASELINE config 0 size
    ((37, 29, 41), 1),  # odd everything: FP32 rows not 16B-aligned, masks on every edge
    ((130, 66, 34), 2),  # wider ghost: allocation offset 2
    ((200, 20, 20), 3),
    ((16, 16, 70), 1),
    ((5, 300, 9), 1),  # thin x -> cell kernel
]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape", SHAPES, ids=[str(s) for s in SHAPES])
def test_jacobi_full_region_bit_exact(dtype, shape):
    (nx, ny, nz), r = shape
    raw = (nz + 2 * r, ny + 2 * r, nx + 2 * r)
    rng = np.random.default_rng(3)
    a = rng.random(raw).astype(dtype)
    src, dst = DevArray(a), DevArray(np.full(raw, 7, dtype=dtype))
    args = ((-r, -r, -r), (0, 0, 0), (nx, ny, nz), (0, 0, 0), (nx, ny, nz))
    gpu_jacobi(dst, src, *args)
    want = np.full(raw, 7, dtype=dtype)
    co.jacobi_region(want, a, *args)
    got = dst.get()
    assert np.array_equal(got, want), float(np.abs(got.astype(np.float64) - want).max())
    if min(nx, ny, nz) >= 30:
        core = got[r:-r, r:-r, r:-r]
        assert (core == 1).sum() > 0 and (core == 0).sum() > 0  # both spheres present


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_jacobi_subregions_interior_and_exterior(dtype):
    """interior + the <=6 exterior slabs (src/stencil.cu:878-977) tile the compute region; a subdomain
    that is a piece of a larger global region, so the spheres are cut by the subdomain boundary."""
    n = (40, 36, 44)
    origin = (40, 0, 44)  # this subdomain's origin inside a (120, 36, 132) global region
    clo, chi = (0, 0, 0), (120, 36, 132)
    ro = g.Radius.face_edge_corner(1, 0, 0)
    raw = g.raw_size(n, ro)
    rng = np.random.default_rng(9)
    a = rng.random(raw[::-1]).astype(dtype)
    src, dst = DevArray(a), DevArray(np.full(raw[::-1], 7, dtype=dtype))
    acc = g.accessor_origin(origin, ro)
    lo, hi = origin, tuple(origin[i] + n[i] for i in range(3))
    want = np.full(raw[::-1], 7, dtype=dtype)
    regions = [g.get_interior(lo, hi, ro)] + g.get_exterior(lo, hi, ro)
    assert len(regions) == 7
    for rlo, rhi in regions:
        gpu_jacobi(dst, src, acc, rlo, rhi, clo, chi)
        co.jacobi_region(want, a, acc, rlo, rhi, clo, chi)
    got = dst.get()
    assert np.array_equal(got, want)
    assert (got == 7).sum() == got.size - n[0] * n[1] * n[2]  # exactly the compute region was written


def test_division_by_six_is_ieee_exact():
    """The fma-corrected multiply must equal IEEE division for every input pattern we can throw at it:
    feed values so that the 6-term sum lands on a dense set of floats (FP32: sweep exponents/mantissas)."""
    rng = np.random.default_rng(0)
    for dtype, bits in ((np.float32, np.uint32), (np.float64, np.uint64)):
        n = 96
        raw = (n + 2, n + 2, n + 2)
        # random bit patterns in a moderate exponent range -> arbitrary mantissas
        if dtype == np.float32:
            a = (rng.random(raw).astype(np.float32) * np.float32(2.0) ** rng.integers(-20, 20, size=raw).astype(np.float32)).astype(np.float32)
        else:
            a = rng.random(raw) * 2.0 ** rng.integers(-200, 200, size=raw)
        src, dst = DevArray(a), DevArray(np.zeros(raw, dtype=dtype))
        # compute region far away from the spheres: put the global region elsewhere
        args = ((-1, -1, -1), (0, 0, 0), (n, n, n), (10**6, 10**6, 10**6), (10**6 + 10, 10**6 + 10, 10**6 + 10))
        gpu_jacobi(dst, src, *args)
        want = np.zeros(raw, dtype=dtype)
        co.jacobi_region(want, a, *args)
        assert np.array_equal(dst.get(), want), dtype


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2])
def test_jacobi_iterations_through_distributed_domain(dtype, ndom):
    """The full loop of bin/jacobi3d.cu:296-368 (interior -> exchange -> exterior -> swap), 10
    iterations on 64^3 (BASELINE config 0), GPU vs oracle: fields bit-exact, residual within 1e-6 rel."""
    n = 64
    radius = sb.Radius.face_edge_corner(1, 0, 0)
    dd = sb.DistributedDomain(n, n, n)
    dd.set_gpus([0] * ndom)
    dd.set_radius(radius)
    h = dd.add_data(dtype, "d")
    dd.realize()
    creg = dd.get_compute_region()
    ro = g.Radius.face_edge_corner(1, 0, 0)
    od = no.Domains((n, n, n), ro, [dtype], n_subdomains=ndom)
    nxt = {i: [np.zeros_like(od.arrays[i][0])] for i in od.indices}
    try:
        for d in dd.domains():
            sb.fill(d, h, d.get_compute_region(), 0.5)
        for i in od.indices:
            od.arrays[i][0][...] = 0
            no.box(od.arrays[i][0], (1, 1, 1), od.sizes[i])[...] = 0.5
        interiors, exteriors = dd.get_interior(), dd.get_exterior()
        for it in range(10):
            for d, reg in zip(dd.domains(), interiors):
                sb.jacobi3d(d, h, reg, creg)
            dd.exchange()
            for d, regs in zip(dd.domains(), exteriors):
                for reg in regs:
                    sb.jacobi3d(d, h, reg, creg)
            for d in dd.domains():
                check(lib().sb_device_sync(d.gpu()))
            dd.swap()
            # oracle
            for i in od.indices:
                lo = od.origins[i]
                hi = tuple(lo[a] + od.sizes[i][a] for a in range(3))
                acc = g.accessor_origin(lo, ro)
                co.jacobi_region(nxt[i][0], od.arrays[i][0], acc, *g.get_interior(lo, hi, ro), *creg)
            od.exchange()
            for i in od.indices:
                lo = od.origins[i]
                hi = tuple(lo[a] + od.sizes[i][a] for a in range(3))
                acc = g.accessor_origin(lo, ro)
                for elo, ehi in g.get_exterior(lo, hi, ro):
                    co.jacobi_region(nxt[i][0], od.arrays[i][0], acc, elo, ehi, *creg)
            for i in od.indices:
                od.arrays[i][0], nxt[i][0] = nxt[i][0], od.arrays[i][0]
        for di, d in enumerate(dd.domains()):
            i = dd.domain_idx_[di]
            got = d.quantity_to_host(0)
            sz = od.sizes[i]
            assert np.array_equal(no.box(got, (1, 1, 1), sz), no.box(od.arrays[i][0], (1, 1, 1), sz)), it
            # residual ||u_{n+1}-u_n||_2 on the GPU vs the oracle (curr vs next after the last swap)
            out = DevArray(np.zeros((1, 1, 1), dtype=np.float64))
            lo, hi = d.get_compute_region()
            check(lib().sb_sqdiff(d.curr_data(0), d.next_data(0), d.elem_size(0), i3(d.accessor_origin()), i3(lo), i3(hi), C.c_void_p(out.ptr), None))
            res_gpu = float(np.sqrt(out.get()[0, 0, 0]))
            res_cpu = float(np.sqrt(co.sqdiff(od.arrays[i][0], nxt[i][0], (1, 1, 1), sz)))
            assert res_cpu > 0 and abs(res_gpu - res_cpu) <= 1e-6 * res_cpu  # BASELINE.json: 1e-6 rel for the FP64 residual
    finally:
        dd.close()


def test_jacobi_full_size_512_fp64_one_step():
    """BASELINE config 1 size: one full-region step on 512^3 FP64 vs the OpenMP oracle, bit-exact."""
    n = 512
    raw = (n + 2, n + 2, n + 2)
    rng = np.random.default_rng(1)
    a = rng.random(raw)
    src, dst = DevArray(a), DevArray(np.zeros((1, 1, 1)), extra=a.nbytes)
    dst.shape, dst.nbytes = raw, a.nbytes
    args = ((-1, -1, -1), (0, 0, 0), (n, n, n), (0, 0, 0), (n, n, n))
    gpu_jacobi(dst, src, *args)
    got = dst.get()
    want = np.zeros(raw)
    co.jacobi_region(want, a, *args)
    assert np.array_equal(got[1:-1, 1:-1, 1:-1], want[1:-1, 1:-1, 1:-1])


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fused_exterior_launch_matches_per_slab_launches(dtype):
    """sb_jacobi3d_regions (all exterior slabs in one launch) == six sb_jacobi3d launches == oracle."""
    n = (40, 36, 44)
    origin = (40, 0, 44)
    clo, chi = (0, 0, 0), (120, 36, 132)
    ro = g.Radius.face_edge_corner(1, 0, 0)
    raw = g.raw_size(n, ro)
    rng = np.random.default_rng(19)
    a = rng.random(raw[::-1]).astype(dtype)
    src, dst = DevArray(a), DevArray(np.full(raw[::-1], 7, dtype=dtype))
    acc = g.accessor_origin(origin, ro)
    lo, hi = origin, tuple(origin[i] + n[i] for i in range(3))
    slabs = g.get_exterior(lo, hi, ro)
    elo = (C.c_int64 * 18)(*[v for s in slabs for v in s[0]])
    ehi = (C.c_int64 * 18)(*[v for s in slabs for v in s[1]])
    check(lib().sb_jacobi3d_regions(dst.pitched(), src.pitched(), a.dtype.itemsize, i3(acc), len(slabs), elo, ehi, i3(clo), i3(chi), None))
    want = np.full(raw[::-1], 7, dtype=dtype)
    for rlo, rhi in slabs:
        co.jacobi_region(want, a, acc, rlo, rhi, clo, chi)
    assert np.array_equal(dst.get(), want)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ndom", [1, 2, 4])
def test_step_async_is_bitwise_step(dtype, ndom):
    """Jacobi3D.step_fused (whole region + halo push in one kernel) and
    Jacobi3D.step_async (iterations queued back to back, dependencies as CUDA events) against Jacobi3D.step (host
    synchronisation after the exchange and after the exterior kernels, bin/jacobi3d.cu:337-365): identical fields
    after 25 iterations, also when the two are mixed.  With several GPUs the subdomains are spread over them."""
    import torch

    from stencil_b200.jacobi import Jacobi3D, jacobi_radius

    n = 128  # 64 cells along x per subdomain when split: whole FP64 warp strips -> dense x staging between GPUs
    ng = torch.cuda.device_count()
    gpus = [i % ng for i in range(ndom)]
    fields = []
    for mode in ("sync", "async", "mixed", "fused", "mixed_fused"):
        dd = sb.DistributedDomain(n, n, n)
        dd.set_gpus(gpus)
        dd.set_radius(jacobi_radius())
        h = dd.add_data(dtype, "d")
        dd.realize()
        try:
            jac = Jacobi3D(dd, h)
            jac.init(0.5)
            for it in range(25):
                if mode == "sync" or (mode == "mixed" and it % 7 == 3) or (mode == "mixed_fused" and it % 9 == 4):
                    jac.step()
                elif mode in ("fused", "mixed_fused") and not (mode == "mixed_fused" and it % 5 == 1):
                    jac.step_fused()  # one kernel per subdomain: update + halo push into the neighbours' ghost cells
                else:
                    jac.step_async()
            jac.synchronize()
            fields.append([d.interior_to_host(0) for d in dd.domains()])
        finally:
            dd.close()
    for other in fields[1:]:
        for a, b in zip(fields[0], other):
            assert np.array_equal(a, b)
    assert float(np.ptp(fields[0][0])) > 0  # the hot/cold spheres made the field non-trivial


@pytest.mark.parametrize("rotate", [0, 1])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_fused_kernel_tile_walks(monkeypatch, rotate, dtype):
    """jacobi_fused_kernel walks its tiles from a rotated origin on every axis (SB_FUSED_ROTATE, default on) so that the
    walk does not end with tiles that push; inner tiles take the plain loop, boundary tiles the variant their faces need.
    Either walk, on shapes with 1..N tiles per axis (also fewer than the two boundary tiles, partial tiles, one-plane
    chunks, and subdomains 768 cells tall in y and z, whose 16-plane chunks would exceed the face-group limit), must
    reproduce Jacobi3D.step bit for bit."""
    from stencil_b200.jacobi import Jacobi3D, jacobi_radius

    monkeypatch.setenv("SB_FUSED_ROTATE", str(rotate))
    for size, ndom in [((40, 24, 70), 1), ((200, 20, 40), 1), ((256, 40, 100), 1), ((384, 30, 66), 2), ((130, 17, 33), 1), ((64, 40, 65), 2), ((128, 7, 1), 1),
                       ((128, 300, 40), 2), ((129, 40, 300), 2), ((256, 600, 9), 2),  # FP32: tail-column tiles that push y / z faces
                       ((64, 768, 768), 1), ((64, 768, 1536), 2)]:
        fields = []
        for mode in ("sync", "fused"):
            dd = sb.DistributedDomain(*size)
            dd.set_gpus([0] * ndom)
            dd.set_radius(jacobi_radius())
            h = dd.add_data(dtype, "d")
            dd.realize()
            try:
                jac = Jacobi3D(dd, h)
                jac.init(0.5)
                for it in range(7):
                    jac.step() if mode == "sync" else jac.step_fused()
                jac.synchronize()
                if mode == "fused":
                    assert jac.fused_supported
                fields.append([d.interior_to_host(0) for d in dd.domains()])
            finally:
                dd.close()
        for a, b in zip(*fields):
            assert np.array_equal(a, b), (size, ndom)


@pytest.mark.parametrize("schedule", ["host-sync", "queued", "fused"])
def test_jacobi_vs_reference_kernel_golden(schedule):
    """The CUDA kernels (all three schedules, FP32 = the reference's dtype) against the reference's own stencil_kernel run
    on a GPU (tests/golden/jacobi_ref.npz): bit for bit against its IEEE build, one ulp per iteration against its
    --use_fast_math build (approximate divide, bin/CMakeLists.txt:56)."""
    import os

    from stencil_b200.jacobi import Jacobi3D, jacobi_radius

    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jacobi_ref.npz"))
    iters = [int(i) for i in gold["iters"]]
    for si, shape in enumerate(gold["shapes"]):
        shape = tuple(int(v) for v in shape)
        dd = sb.DistributedDomain(*shape)
        dd.set_gpus([0])
        dd.set_radius(jacobi_radius())
        h = dd.add_data(np.float32, "d")
        dd.realize()
        try:
            jac = Jacobi3D(dd, h)
            jac.init(0.5)
            done = 0
            for k, target in enumerate(iters):
                while done < target:
                    {"host-sync": jac.step, "queued": jac.step_async, "fused": jac.step_fused}[schedule]()
                    done += 1
                jac.synchronize()
                got = dd.domains()[0].interior_to_host(0)
                ieee, fast = gold[f"ieee_{si}"][k], gold[f"fast_{si}"][k]
                assert np.array_equal(got, ieee), (shape, target, int(np.count_nonzero(got != ieee)))
                assert float(np.abs(got.astype(np.float64) - fast).max()) <= 6e-8 * target + 1e-12  # <= 1 ulp per iteration (fast divide)
        finally:
            dd.close()


@pytest.mark.parametrize("ndom", [1, 2])
def test_fused_iterations_as_a_cuda_graph(ndom):
    """Jacobi3D.capture_fused: 4 fused iterations captured into one CUDA graph; 3 replays (+ the 2 warm-up iterations the
    capture runs) must equal 14 iterations of Jacobi3D.step bit for bit, and fused steps may follow a replay."""
    from stencil_b200.jacobi import Jacobi3D, jacobi_radius

    fields = []
    for mode in ("sync", "graph"):
        dd = sb.DistributedDomain(128, 64, 64)
        dd.set_gpus([0] * ndom)
        dd.set_radius(jacobi_radius())
        h = dd.add_data(np.float64, "d")
        dd.realize()
        try:
            jac = Jacobi3D(dd, h)
            jac.init(0.5)
            if mode == "sync":
                for _ in range(16):
                    jac.step()
            else:
                g = jac.capture_fused(4)  # runs 2 iterations itself
                for _ in range(3):
                    g.replay()
                jac.synchronize()
                jac.step_fused()
                jac.step_fused()
            jac.synchronize()
            fields.append([d.interior_to_host(0) for d in dd.domains()])
        finally:
            dd.close()
    for a, b in zip(*fields):
        assert np.array_equal(a, b)
