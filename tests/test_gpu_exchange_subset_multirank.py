"""Subset exchanges across processes (DESIGN.md section 2.15): the Python host under torchrun with 2 and 4 ranks, over
CUDA IPC and over the NCCL fallback, gives the one-process bits of subset exchanges and of a PCG solve
(tests/mp_exchange_subset_check.py); the C++ DistributedDomain::exchange(quantities) under bin/sb_mpirun with 1, 2
and 4 ranks gives each subset the full exchange's bytes and leaves the other quantities untouched
(tests/cpp/test_exchange_subset_multigpu.cu).  With fewer GPUs than ranks the ranks share GPUs."""
import os
import subprocess
import sys

import pytest

from test_gpu_colour_multirank import BIN, ROOT, mpirun_env

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["ipc", "nccl"])
@pytest.mark.parametrize("ranks", [2, 4])
def test_python_subset_exchange_one_process_per_rank(tmp_path, ranks, mode):
    import torch

    if mode == "nccl" and torch.cuda.device_count() < ranks:
        pytest.skip("the NCCL fallback needs one GPU per rank")
    script = os.path.join(ROOT, "tests", "mp_exchange_subset_check.py")
    expect = str(tmp_path / "single.json")
    out = subprocess.run([sys.executable, script, "--single", str(ranks), expect], env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "single OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
    env = dict(mpirun_env(), SB_FORCE_NCCL="1" if mode == "nccl" else "0")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ranks}", "--master-addr", "127.0.0.1",
           "--master-port", str(29660 + 2 * ranks + (mode == "nccl")), script, "--expect", expect]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "mp_exchange_subset_check OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.parametrize("ranks", [1, 2, 4])
def test_cpp_subset_exchange_under_sb_mpirun(tmp_path, ranks):
    exe = os.path.join(BIN, "test_exchange_subset_multigpu")
    if not os.path.exists(exe):
        pytest.fail("bin/test_exchange_subset_multigpu not built -- run `make`")
    cmd = [exe] if ranks == 1 else [os.path.join(BIN, "sb_mpirun"), "-n", str(ranks), exe]
    out = subprocess.run(cmd, cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    assert f"on {ranks} rank(s)" in out.stdout
