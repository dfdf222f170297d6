"""The resident tensor-core kernel's schedule (two producer warps, one x ring per consumer warpgroup, ordered MMA turns,
the shared y block) replayed on the host as a state machine: nothing ever waits forever, and every wait sees the load
it is meant to see (tests/cpp/tc_turn_schedule_test.cu).  No GPU needed."""
import subprocess

import cpp_build


def test_resident_turn_schedule_never_sticks(tmp_path):
    exe = cpp_build.build("tc_turn_schedule_test.cu", str(tmp_path / "tc_turn_schedule_test"), standalone=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
