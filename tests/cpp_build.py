"""Builds the C++ test programs of tests/cpp with nvcc.  Callers put the executables outside the source tree, which need
not be writable."""
import os
import shutil
import subprocess

from raft_b200 import _build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def build(source, exe, mock_raft=False, libs=(), standalone=False):
    """Compiles tests/cpp/<source> into exe and returns exe.

    By default the program includes the public headers and links against the library (built first if stale).
    mock_raft: compile with RAFT_B200_USE_REAL_RAFT against tests/cpp/mock_raft, a header tree with the reference's
    signatures only (raft::resources has no workspace() / stream() members).  libs: further libraries to link.
    standalone: a host program that includes the kernel headers itself, compiled for sm_90a like the library, unlinked.
    """
    cmd = [NVCC, "-std=c++17", "-O1"]
    if standalone:
        cmd += ["--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a"]
    else:
        _build.build()
        cmd += ["-I", os.path.join(ROOT, "include")]
    if mock_raft:
        cmd += ["-DRAFT_B200_USE_REAL_RAFT", "-I", os.path.join(ROOT, "tests", "cpp", "mock_raft")]
    cmd += ["-o", exe, os.path.join(ROOT, "tests", "cpp", source)]
    if not standalone:
        lib_dir = os.path.dirname(_build.SO_PATH)
        cmd += ["-L", lib_dir, "-lraft_b200", *libs, "-Xlinker", "-rpath", "-Xlinker", lib_dir]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return exe
