"""The header-only C++ shim (include/raft/distance/*.cuh) compiles against the C ABI everywhere and
passes its self-check on the GPU box."""
import os
import subprocess

import pytest

import cpp_build


@pytest.fixture(scope="module")
def build_dir(tmp_path_factory):
    """The test programs are built outside the source tree, which need not be writable."""
    return str(tmp_path_factory.mktemp("cpp"))


def compile_shim(build_dir, mock_raft=False):
    """mock_raft: the shim's scratch must come from raft::resource::get_workspace_resource_ref through
    rmm::device_uvector, since the mock raft::resources has no workspace() member."""
    exe = os.path.join(build_dir, "shim_test_mockraft" if mock_raft else "shim_test")
    return cpp_build.build("shim_test.cu", exe, mock_raft)


def test_shim_compiles_against_raft_resources_without_workspace_member(build_dir):
    assert os.path.exists(compile_shim(build_dir, mock_raft=True))


@pytest.mark.gpu
def test_shim_runs_on_gpu_with_mock_raft_resources(build_dir):
    exe = os.path.join(build_dir, "shim_test_mockraft")
    if not os.path.exists(exe):
        compile_shim(build_dir, mock_raft=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr


def test_shim_compiles_and_links(build_dir):
    assert os.path.exists(compile_shim(build_dir))


@pytest.mark.gpu
def test_shim_runs_on_gpu(build_dir):
    exe = os.path.join(build_dir, "shim_test")
    if not os.path.exists(exe):
        compile_shim(build_dir)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr


def test_block_selection_helpers_partition_the_blocks(build_dir):
    """sel_to_blk / sel_count (shared by the kernels and the launch code) on the host: the exact sample
    pass, the trial screen and the main screen visit every y block exactly once, in ascending order."""
    exe = cpp_build.build("host_logic_test.cu", os.path.join(build_dir, "host_logic_test"), standalone=True)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert res.returncode == 0 and "PASS" in res.stdout, res.stdout + res.stderr


def compile_multi(build_dir):
    return cpp_build.build("multi_test.cu", os.path.join(build_dir, "multi_test"), libs=["-lnccl"])


def test_multi_gpu_c_entry_compiles_and_links(build_dir):
    """b2d_fused_l2_nn_multi (single process, one ncclComm_t per device): the SNMG form a C++ caller uses."""
    assert os.path.exists(compile_multi(build_dir))


@pytest.mark.gpu
def test_multi_gpu_c_entry_runs(build_dir):
    """Runs with every visible device (1 on the single-GPU box: the exchange-free path; N under `gpurun --gpus N`:
    grouped ncclAllReduce(int64, min) between sub-chunks) and compares with the single-device entry point."""
    exe = os.path.join(build_dir, "multi_test")
    if not os.path.exists(exe):
        compile_multi(build_dir)
    res = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and ("PASS" in res.stdout or "SKIP" in res.stdout), res.stdout + res.stderr
