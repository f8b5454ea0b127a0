"""The packed weight-image layout of the wgmma TD kernel is written by two different kernels
(dqn_tc_pack_kernel and the Adam kernel) and read by a third; this host-only program checks
that their index maps agree (tests/csrc/tc_layout_check.cu, compiled with nvcc, run on the CPU)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_weight_image_layout_is_consistent(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = tmp_path / "tc_layout_check"
    src = os.path.join(ROOT, "tests", "csrc", "tc_layout_check.cu")
    subprocess.run([nvcc, "-std=c++17", "-O1", "-o", str(exe), src], check=True, cwd=ROOT)
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 0 and out.stdout.strip() == "ok", (out.returncode, out.stdout, out.stderr)
