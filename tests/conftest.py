"""pytest configuration.

Everything that needs a GPU is marked ``@pytest.mark.gpu``; the rest runs on CPU
with multi-process SPMD jobs started through ``mpi4torch_b200.launch``.
"""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs at least one CUDA device (run on an H100 box)")


def run_spmd(nprocs, script_args, *, device="cpu", timeout=600, extra_env=None):
    """Launch an SPMD job with the repo's own launcher; returns CompletedProcess."""
    env = dict(os.environ)
    env["PYTHONPATH"] = str(ROOT) + os.pathsep + env.get("PYTHONPATH", "")
    env["M4T_TEST_DEVICE"] = device
    env.setdefault("M4T_TIMEOUT_S", "120")
    env.setdefault("M4T_DEVICE_TIMEOUT_S", "20")
    if device == "cpu":
        env["M4T_CUDA"] = "0"
    if extra_env:
        env.update(extra_env)
    cmd = [sys.executable, "-m", "mpi4torch_b200.launch", "-np", str(nprocs), "--timeout", str(timeout)] + list(script_args)
    return subprocess.run(cmd, env=env, cwd=str(ROOT), capture_output=True, text=True, timeout=timeout + 60)


@pytest.fixture
def spmd():
    return run_spmd
