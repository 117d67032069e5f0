"""The C++ API (include/stencil/*.hpp + lib/libstencil.a) on a GPU, through the programs `make` builds into bin/: our
jacobi3d_b200 driver (the reference's jacobi3d loop over stencil::FusedJacobi3d) compared with the reference's own kernel
(tests/golden/jacobi_ref.npz), as one and as two ranks, and a multi-rank exchange check.
Match: test/test_cuda_mpi_exchange.cu:193-245, bin/jacobi3d.cu."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "bin")
pytestmark = pytest.mark.gpu


def need(*names):
    missing = [n for n in names if not os.path.exists(os.path.join(ROOT, n))]
    if missing:
        pytest.fail("C++ programs not built: " + ", ".join(missing) + " missing -- run `make`")


@pytest.mark.parametrize(
    "shape,align",
    [
        pytest.param((64, 64, 64), "1", id="shape0"),
        pytest.param((96, 80, 72), "1", id="shape1"),
        # allocations at the start of their blocks, as the reference places them.  FP32 rows of 66 / 98 floats are not
        # 16-byte multiples, so LocalDomain::lead_bytes gives no lead under either setting: this pins that the switch
        # changes nothing there (the layouts it does change are swept in test_gpu_jacobi_layouts.py)
        pytest.param((64, 64, 64), "0", id="shape0-align0"),
        pytest.param((96, 80, 72), "0", id="shape1-align0"),
    ],
)
def test_jacobi3d_b200_matches_the_reference_kernel(tmp_path, shape, align):
    """Our C++ fast path (FusedJacobi3d: fused kernel; and its reference-schedule fallback) against the reference's own
    stencil_kernel built with IEEE division (tests/golden/jacobi_ref.npz, ieee_*), bit for bit after 10 iterations, with
    SB_ALLOC_ALIGN = 1 (first compute cell 16-byte aligned) and 0."""
    need("bin/jacobi3d_b200")
    gold = np.load(os.path.join(ROOT, "tests", "golden", "jacobi_ref.npz"))
    si = [tuple(int(v) for v in s) for s in gold["shapes"]].index(shape)
    want = gold[f"ieee_{si}"][[int(i) for i in gold["iters"]].index(10)].reshape(-1)
    n = [str(v) for v in shape]
    # the driver scales the size by the prime factors of the GPU count (bin/jacobi3d.cu:189-199): pin it to one GPU
    env = dict(os.environ, CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0], SB_ALLOC_ALIGN=align)
    for extra in ([], ["--reference-schedule"]):
        got_f = tmp_path / "got.bin"
        out = subprocess.run([os.path.join(BIN, "jacobi3d_b200"), *n, "-n", "5", "--dump", str(got_f)] + extra, cwd=tmp_path, env=env, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-3000:]
        got = np.fromfile(got_f, dtype=np.float32)  # 5 timed + 5 queued iterations = 10
        assert got.shape == want.shape and np.array_equal(got, want), (shape, extra, int(np.count_nonzero(got != want)))
        assert float(np.ptp(got)) > 0


def mpirun_env():
    return {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}


@pytest.mark.parametrize("ranks", [2, 4])
def test_cpp_multi_rank_exchange(tmp_path, ranks):
    """One process per rank through the C++ API (bin/sb_mpirun = this repo's node-local MPI stand-in): allocations, staging
    buffers and flag mailboxes are shared through CUDA IPC handles sent over MPI, the exchange is the fused direct write +
    device-side ready/done flags.  Every rank checks the WHOLE allocation of its subdomains (ghost cells included) against
    the periodically wrapped field, 5 radius shapes x 3 quantities x 3 rounds with swaps.  With fewer GPUs than ranks the
    ranks share GPUs (the reference's rule, src/stencil.cu:76-85), so this runs on a 1-GPU machine as well.
    Match: test/test_cuda_mpi_exchange.cu:193-245, include/stencil/tx_cuda.cuh:185-492, src/tx_colocated.cu."""
    need("bin/sb_mpirun", "bin/test_exchange_multigpu")
    out = subprocess.run([os.path.join(BIN, "sb_mpirun"), "-n", str(ranks), os.path.join(BIN, "test_exchange_multigpu")], cwd=tmp_path, env=mpirun_env(),
                         capture_output=True, text=True, timeout=900)  # fmt: skip
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    assert f"on {ranks} rank(s)" in out.stdout


def test_jacobi3d_b200_driver_one_rank_per_gpu(tmp_path):
    """The jacobi3d_b200 driver as 2 ranks (what `mpirun -n 2 jacobi3d_b200` is on a machine with MPI)."""
    need("bin/sb_mpirun", "bin/jacobi3d_b200")
    out = subprocess.run([os.path.join(BIN, "sb_mpirun"), "-n", "2", os.path.join(BIN, "jacobi3d_b200"), "64", "64", "64", "-n", "5"], cwd=tmp_path, env=mpirun_env(),
                         capture_output=True, text=True, timeout=600)  # fmt: skip
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("jacobi3d_b200,")]
    assert line and line[-1].split(",")[2] == "2", out.stdout[-2000:]  # world size 2
