"""The measurement scripts under tools/: every one compiles, none times anything or reads the card except through
tools/measure.py, and without a CUDA device each stops with measure.require_cuda's one line rather than a traceback."""
import glob
import os
import py_compile
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = sorted(glob.glob(os.path.join(ROOT, "tools", "*.py")))
# every measurement script but the two that need torchrun and two or more GPUs (run_sharded_ba, profile_sharded)
MEASURED = [p for p in TOOLS if os.path.basename(p).startswith("time_") or os.path.basename(p) == "profile_step.py"]


@pytest.mark.parametrize("path", TOOLS, ids=os.path.basename)
def test_tool_compiles(path, tmp_path):
    py_compile.compile(path, cfile=str(tmp_path / "tool.pyc"), doraise=True)


def test_only_measure_times():
    found = []
    for path in glob.glob(os.path.join(ROOT, "tools", "*.py")) + glob.glob(os.path.join(ROOT, "tests", "tools", "*.py")):
        if path == os.path.join(ROOT, "tools", "measure.py"):
            continue
        text = open(path).read()
        found += ["%s: %s" % (os.path.relpath(path, ROOT), s) for s in ("torch.cuda.Event(", "nvidia-smi", "torch.profiler")
                  if s in text]
    assert not found, found


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the exit on a machine without a CUDA device")
@pytest.mark.parametrize("path", MEASURED, ids=os.path.basename)
def test_tool_needs_cuda(path, tmp_path):
    r = subprocess.run([sys.executable, path], cwd=tmp_path, capture_output=True, text=True, timeout=600)
    assert r.returncode != 0
    assert r.stderr.strip() == "%s: needs a CUDA device" % os.path.basename(path), r.stderr
