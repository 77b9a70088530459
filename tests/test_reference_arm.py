"""The reference arm of bench.py (baseline/): the shared-memory MPI shim on its own, and a cross-check of this
library's CPU backend against results of the UNMODIFIED reference built against the shim (stored in
tests/golden/reference_cross_np3.json)."""
import json
import os
import shutil
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SHIM = ROOT / "baseline" / "mpi_shim"
MPIRUN = SHIM / "bin" / "mpirun"
GOLDEN = ROOT / "tests" / "golden" / "reference_cross_np3.json"


def _run(cmd, timeout=600, env=None):
    e = dict(os.environ)
    e.pop("RANK", None)
    e.pop("WORLD_SIZE", None)
    if env:
        e.update(env)
    return subprocess.run([str(c) for c in cmd], capture_output=True, text=True, timeout=timeout, env=e, cwd=str(ROOT))


@pytest.fixture(scope="module")
def shim():
    res = _run(["make", "-C", SHIM])
    assert res.returncode == 0, res.stdout + res.stderr
    assert (SHIM / "lib" / "libmpi.so").exists()
    return SHIM


@pytest.mark.parametrize("np_", [1, 2, 3, 5])
def test_mpi_shim_selftest(shim, np_, tmp_path):
    exe = tmp_path / "selftest"
    res = _run([SHIM / "bin" / "mpicxx", "-O2", "-std=c++17", "-o", exe, SHIM / "test" / "selftest.cpp"])
    assert res.returncode == 0, res.stderr
    res = _run([MPIRUN, "-np", np_, exe], timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    assert f"mpishim selftest np={np_}: ok" in res.stdout


CROSS = r'''
import json, sys, time, torch
which = sys.argv[1]
if which == "ours":
    sys.path.insert(0, sys.argv[2]); import mpi4torch_b200 as m
else:
    sys.path.insert(0, sys.argv[2] + "/baseline/_ref"); import mpi4torch as m
comm = m.COMM_WORLD
g = torch.Generator().manual_seed(7 + comm.rank)
out = {}
x = torch.randn(1 << 16, generator=g, dtype=torch.float64).requires_grad_()
y = comm.Allreduce(x, m.MPI_SUM)
(y * (comm.rank + 1)).sum().backward()
out["fwd"] = float(y.detach().double().sum()); out["fwd_abs"] = float(y.detach().abs().sum())
out["bwd"] = float(x.grad.sum())
a = torch.randn(3, comm.rank + 2, 4, generator=g, dtype=torch.float64)
out["allgather"] = float((comm.Allgather(a, 1) * torch.arange(4.0, dtype=torch.float64)).sum())
big = torch.randn(1 << 22, generator=g)   # 16 MiB fp32
for _ in range(2): comm.Allreduce(big, m.MPI_SUM)
t0 = time.perf_counter()
for _ in range(5): comm.Allreduce(big, m.MPI_SUM)
out["allreduce_16MiB_ms"] = (time.perf_counter() - t0) / 5 * 1e3
if comm.rank == 0: print(json.dumps(out))
'''


def test_reference_over_the_shim_agrees_with_this_library(tmp_path):
    """Same program as the reference ran (over the shim, np=3, results stored as golden data): identical Allreduce
    forward/backward and Allgather results through this library."""
    script = tmp_path / "cross.py"
    script.write_text(CROSS)
    ours = _run([sys.executable, "-m", "mpi4torch_b200.launch", "-np", "3", script, "ours", ROOT], timeout=600,
                env={"M4T_CUDA": "0", "PYTHONPATH": str(ROOT)})
    assert ours.returncode == 0, ours.stderr[-3000:]
    r = json.loads(GOLDEN.read_text())
    o = json.loads([ln for ln in ours.stdout.splitlines() if ln.startswith("{")][-1])
    for key in ("fwd", "fwd_abs", "bwd", "allgather"):
        assert abs(r[key] - o[key]) <= 1e-9 * max(1.0, abs(o[key])), (key, r[key], o[key])


def test_bench_reference_arm_prints_one_json_line_without_a_gpu():
    """On a box without CUDA the reference arm must say so in one JSON line and exit 0 (driver contract)."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("needs a CPU-only box")
    res = _run([sys.executable, "bench.py", "--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "1"], timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("{")][-1]
    d = json.loads(line)
    assert d["impl"] == "reference" and "unavailable" in d
