"""Dropless expert-parallel MoE over several ranks: tests/spmd/grouped_moe_steps.py on the CPU backend in float64, and
on CUDA at every world size the box offers."""
import pytest
import torch

from conftest import run_spmd


@pytest.mark.parametrize("nprocs", [1, 2, 3])
def test_grouped_moe_steps_cpu(nprocs):
    res = run_spmd(nprocs, ["tests/spmd/grouped_moe_steps.py"], device="cpu", timeout=600)
    assert res.returncode == 0, f"np={nprocs}\nSTDOUT:\n{res.stdout[-4000:]}\nSTDERR:\n{res.stderr[-8000:]}"
    assert f"grouped_moe_steps np={nprocs} device=cpu ok=True" in res.stdout


def _world_sizes():
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    return [s for s in (1, 2, 4, 8) if s <= n] or [1]


@pytest.mark.gpu
@pytest.mark.parametrize("nprocs", _world_sizes())
def test_grouped_moe_steps_cuda(nprocs):
    res = run_spmd(nprocs, ["tests/spmd/grouped_moe_steps.py"], device="cuda", timeout=900)
    assert res.returncode == 0, f"np={nprocs}\nSTDOUT:\n{res.stdout[-4000:]}\nSTDERR:\n{res.stderr[-12000:]}"
    assert f"grouped_moe_steps np={nprocs} device=cuda ok=True" in res.stdout
