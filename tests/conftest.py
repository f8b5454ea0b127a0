import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device")
    # The CPU oracle is torch fp32 on the host.  On the many-core GPU boxes torch's default (one
    # thread per core) is pathological for these small GEMMs -- bench.py's sweep measured 0.3
    # updates/s at 128 threads against ~60 at 16 -- and gets worse when the host is shared, so
    # pin a moderate count: the parity tests then take seconds wherever they run.
    import torch

    torch.set_num_threads(max(1, min(16, os.cpu_count() or 1)))


def pytest_sessionstart(session):
    """The tests need the in-tree library; build it when it is missing and nvcc is here (the
    product path never does this: `_lib.lib()` fails loudly without the extension)."""
    import shutil
    import subprocess

    so = os.path.join(ROOT, "reagent_b200", "libreagent_b200.so")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(so) and os.path.exists(nvcc):
        subprocess.run(["bash", os.path.join(ROOT, "reagent_b200", "csrc", "build.sh")], check=True)


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        # a protocol bug in a kernel must fail one test, not eat the GPU box's time budget
        for item in items:
            if "gpu" in item.keywords and item.get_closest_marker("timeout") is None:
                item.add_marker(pytest.mark.timeout(300))
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
