"""Exact reductions across processes give the bits of a one-process run of a DIFFERENT partition: the Python layer
under torchrun (tests/mp_reduce_exact_check.py, 2 and 4 ranks) and the C++ API under bin/sb_mpirun
(tests/cpp/test_reduce_exact_multigpu.cu, 1, 2 and 4 ranks), each against one-process runs on 1 and on 3 subdomains,
which must themselves agree.  With fewer GPUs than ranks the ranks share GPUs, so this runs on a one-GPU machine."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "bin")
pytestmark = pytest.mark.gpu


def mpirun_env():
    return {k: v for k, v in os.environ.items() if k not in ("WORLD_SIZE", "RANK", "LOCAL_RANK")}


def singles(cmd, tmp_path, ok):
    """the one-process files of 1 and 3 subdomains, which must be identical"""
    files = []
    for n in (1, 3):
        path = str(tmp_path / f"single{n}.out")
        out = subprocess.run(cmd + ["--single", str(n), path], cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
        assert out.returncode == 0 and ok in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]
        files.append(path)
    with open(files[0]) as a, open(files[1]) as b:
        assert a.read() == b.read(), "1 and 3 subdomains give different exact bits"
    return files


@pytest.mark.parametrize("ranks", [2, 4])
def test_python_exact_reductions_one_process_per_rank(tmp_path, ranks):
    script = os.path.join(ROOT, "tests", "mp_reduce_exact_check.py")
    for i, expect in enumerate(singles([sys.executable, script], tmp_path, "single OK")):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={ranks}", "--master-addr", "127.0.0.1",
               "--master-port", str(29570 + ranks + 10 * i), script, "--expect", expect]
        out = subprocess.run(cmd, env=mpirun_env(), capture_output=True, text=True, timeout=900)
        assert out.returncode == 0 and "mp_reduce_exact_check OK" in out.stdout, out.stdout[-2000:] + out.stderr[-4000:]


@pytest.mark.parametrize("ranks", [1, 2, 4])
def test_cpp_exact_reductions_under_sb_mpirun(tmp_path, ranks):
    exe = os.path.join(BIN, "test_reduce_exact_multigpu")
    if not os.path.exists(exe):
        pytest.fail("bin/test_reduce_exact_multigpu not built -- run `make`")
    for expect in singles([exe], tmp_path, "ALL OK"):
        cmd = [exe] if ranks == 1 else [os.path.join(BIN, "sb_mpirun"), "-n", str(ranks), exe]
        out = subprocess.run(cmd + ["--expect", expect], cwd=tmp_path, env=mpirun_env(), capture_output=True, text=True, timeout=900)
        assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
        assert f"on {ranks} rank(s)" in out.stdout
