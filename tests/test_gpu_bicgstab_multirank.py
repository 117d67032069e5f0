"""stencil_b200.BiCGStab and stencil::BiCGStab<T> across processes give the bits of a one-process run of the same
partition: the Python solver under torchrun (tests/mp_bicgstab_check.py) and the C++ solver under bin/sb_mpirun
(tests/cpp/test_bicgstab_multigpu.cu, which also checks the C++ solver against the same iterations written from public
C++ calls).  With fewer GPUs than ranks the ranks share GPUs, so this runs on a one-GPU machine."""
import os
import subprocess
import sys

import pytest

from test_gpu_colour_multirank import BIN, ROOT, mpirun_env

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("ranks", [2, 4])
def test_python_bicgstab_one_process_per_rank(tmp_path, ranks):
    script = os.path.join(ROOT, "tests", "mp_bicgstab_check.py")
    expect = str(tmp_path / "single.json")
    out = subprocess.run([sys.executable, script, "--single", str(ranks), expect], env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "single OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ranks}", "--master-addr", "127.0.0.1",
           "--master-port", str(29660 + ranks), script, "--expect", expect]
    out = subprocess.run(cmd, env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "mp_bicgstab_check OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.parametrize("ranks", [1, 2, 4])
def test_cpp_bicgstab_under_sb_mpirun(tmp_path, ranks):
    exe = os.path.join(BIN, "test_bicgstab_multigpu")
    if not os.path.exists(exe):
        pytest.fail("bin/test_bicgstab_multigpu not built -- run `make`")
    expect = str(tmp_path / "single.txt")
    out = subprocess.run([exe, "--single", str(ranks), expect], cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    cmd = [exe] if ranks == 1 else [os.path.join(BIN, "sb_mpirun"), "-n", str(ranks), exe]
    out = subprocess.run(cmd + ["--expect", expect], cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
    assert f"on {ranks} rank(s)" in out.stdout
