"""stencil_b200.Multigrid and stencil::Multigrid<T> across processes give the bits of a one-process run of the same
partition: the Python solver under torchrun (tests/mp_multigrid_check.py; peer mappings and, with SB_FORCE_NCCL=1, the
NCCL fallback) and the C++ solver under bin/sb_mpirun (tests/cpp/test_multigrid_multigpu.cu).  With fewer GPUs than
ranks the ranks share GPUs, so this runs on a one-GPU machine."""
import os
import subprocess
import sys

import pytest

from test_gpu_colour_multirank import BIN, ROOT, mpirun_env

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ranks,nccl", [(2, False), (4, False), (2, True)])
def test_python_multigrid_one_process_per_rank(tmp_path, ranks, nccl):
    import torch

    if nccl and torch.cuda.device_count() < ranks:
        pytest.skip("the NCCL fallback needs one GPU per rank")
    script = os.path.join(ROOT, "tests", "mp_multigrid_check.py")
    expect = str(tmp_path / "single.json")
    out = subprocess.run([sys.executable, script, "--single", str(ranks), expect], env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "single OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
    env = mpirun_env()
    if nccl:
        env["SB_FORCE_NCCL"] = "1"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ranks}", "--master-addr", "127.0.0.1",
           "--master-port", str(29610 + ranks + (5 if nccl else 0)), script, "--expect", expect]
    out = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "mp_multigrid_check OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.parametrize("ranks", [1, 2, 4])
def test_cpp_multigrid_under_sb_mpirun(tmp_path, ranks):
    exe = os.path.join(BIN, "test_multigrid_multigpu")
    if not os.path.exists(exe):
        pytest.fail("bin/test_multigrid_multigpu not built -- run `make`")
    expect = str(tmp_path / "single.txt")
    out = subprocess.run([exe, "--single", str(ranks), expect], cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    cmd = [exe] if ranks == 1 else [os.path.join(BIN, "sb_mpirun"), "-n", str(ranks), exe]
    out = subprocess.run(cmd + ["--expect", expect], cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    assert f"on {ranks} rank(s)" in out.stdout
