"""The output staging ring of the tensor-core kernel's EPI_STORE epilogue (tc_stage_store: two boxes per consumer
warpgroup, written in pairs between two named barriers and read by TMA stores) replayed on the host as a state machine
under random interleavings: nothing ever waits forever, and no box is rewritten before its store has read it
(tests/cpp/tc_stage_ring_test.cu).  No GPU needed."""
import subprocess

import cpp_build


def test_stage_ring_never_sticks_or_overwrites(tmp_path):
    exe = cpp_build.build("tc_stage_ring_test.cu", str(tmp_path / "tc_stage_ring_test"), standalone=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr
