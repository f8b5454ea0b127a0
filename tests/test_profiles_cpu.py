"""The profile scripts without a GPU: --help works, and a measurement stops with the one
"no CUDA device" message before it builds anything or writes a result."""
import glob
import os
import runpy
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPTS = sorted(glob.glob(os.path.join(ROOT, "profiles", "time_*.py")))

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="with a GPU the scripts would start measuring")


def _run(monkeypatch, script, *args):
    monkeypatch.setattr(sys, "argv", [script, *args])
    with pytest.raises(SystemExit) as e:
        runpy.run_path(script, run_name="__main__")
    return e.value.code


def test_there_are_profile_scripts():
    assert len(SCRIPTS) >= 10


@pytest.mark.parametrize("script", SCRIPTS, ids=os.path.basename)
def test_help_exits_zero(monkeypatch, capsys, script):
    assert _run(monkeypatch, script, "--help") == 0
    assert "--out" in capsys.readouterr().out


@pytest.mark.parametrize("script", SCRIPTS, ids=os.path.basename)
def test_no_gpu_exits_before_building(monkeypatch, tmp_path, script):
    out = tmp_path / "out"
    code = _run(monkeypatch, script, "--out", str(out))
    assert code == f"{os.path.basename(script)} measures on the GPU; no CUDA device is visible"
    assert not out.exists()
