"""The resident tensor-core kernel's schedule (two producer warps, one x ring per consumer warpgroup, ordered MMA turns,
the shared y block) replayed on the host as a state machine: nothing ever waits forever, and every wait sees the load
it is meant to see (tests/cpp/tc_turn_schedule_test.cu).  No GPU needed."""
import os
import shutil
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_resident_turn_schedule_never_sticks(tmp_path):
    # built outside the source tree, which need not be writable
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path / "tc_turn_schedule_test")
    cmd = [nvcc, "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
           os.path.join(ROOT, "tests", "cpp", "tc_turn_schedule_test.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
