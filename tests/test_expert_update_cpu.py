"""Training the expert parameters inside backward, the parts that run without a GPU: ``expert_mlp`` and
``grouped_expert_mlp`` with an ``AccumulatedSGD`` on the composition path in float64, the accumulator's owned
parameters, the errors of the update modes, ``ExpertParallelMLP`` with an accumulator at two and three ranks
(tests/spmd/expert_update_steps.py) and the MoE example with micro-batches."""
import re

import pytest
import torch

from conftest import run_spmd

from mpi4torch_b200.ops import AccumulatedSGD, InBackwardSGD, expert_mlp, grouped_expert_mlp
from mpi4torch_b200.ops.expert_mlp import grouped_rows

LR = 0.125


def _params(E, D, H, O, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    return [r(E, H, D) / D ** 0.5, r(E, H), r(E, O, H) / H ** 0.5, r(E, O)]


def _grouped_batch(counts, D, O, seed):
    """x [R, D] in the grouped layout of counts (padding rows random too: they must not matter), r [R, O], counts."""
    g = torch.Generator().manual_seed(seed)
    cnt = torch.tensor(counts, dtype=torch.int32)
    R = grouped_rows(sum(counts), len(counts))
    return torch.randn(R, D, generator=g, dtype=torch.float64), torch.randn(R, O, generator=g, dtype=torch.float64), cnt


def _micro_batches(kind, K, E, D, O):
    """K micro-batches as (forward(params, **update) -> y, weight r of the loss sum(y * r))."""
    g = torch.Generator().manual_seed(100 + K)
    if kind == "batched":
        x = torch.randn(E, 8 * K, D, generator=g, dtype=torch.float64)
        r = torch.randn(E, 8 * K, O, generator=g, dtype=torch.float64)
        return [((lambda ps, xk=xk, **u: expert_mlp(xk, *ps, **u)), rk) for xk, rk in zip(x.chunk(K, 1), r.chunk(K, 1))]
    out = []
    for k in range(K):
        counts = [(3 * k + 5 * e) % 7 for e in range(E)]  # empty experts included
        xk, rk, cnt = _grouped_batch(counts, D, O, 200 + k)
        out.append(((lambda ps, xk=xk, cnt=cnt, **u: grouped_expert_mlp(xk, cnt, *ps, **u)), rk))
    return out


@pytest.mark.parametrize("kind", ["batched", "grouped"])
@pytest.mark.parametrize("K", [1, 2, 4])
def test_accumulator_equals_plain_gradients_and_sgd(kind, K):
    """K micro-batches through the accumulator, then step(): the parameters of one SGD step on the plain gradients of
    the whole batch."""
    E, D, H, O = 3, 8, 12, 6
    init = _params(E, D, H, O, 1)
    batches = _micro_batches(kind, K, E, D, O)
    plain = [p.clone().requires_grad_() for p in init]
    sum((fwd(plain) * r).sum() for fwd, r in batches).backward()
    want = [(p - LR * p.grad).detach() for p in plain]

    ps = [p.clone().requires_grad_() for p in init]
    acc = AccumulatedSGD(LR)
    for fwd, r in batches:
        (fwd(ps, accumulator=acc) * r).sum().backward()
    assert all(p.grad is None for p in ps), "the accumulator's parameters got a .grad"
    assert len(acc.buffers()) == 4
    acc.step()
    for got, ref, name in zip(ps, want, ("w1", "b1", "w2", "b2")):
        err = float((got.detach() - ref).abs().max())
        assert err <= 1e-12 * max(1.0, float(ref.abs().max())), f"{kind} K={K} {name} off by {err}"
    assert all(bool((b == 0).all()) for _, b in acc.buffers()), "step() left a buffer non-zero"


class _CountingComm:
    """A stand-in communicator of two identical ranks that counts its collectives."""
    size = 2

    def __init__(self):
        self.calls = 0

    def AllreduceFused(self, t, op, scale, _):
        self.calls += 1
        return t * (scale * self.size)


def test_owned_buffers_step_without_a_collective():
    acc = AccumulatedSGD(LR)
    p = torch.ones(4, dtype=torch.float64)
    acc.buffer(p, None).add_(torch.arange(4.0, dtype=torch.float64))
    acc.step()
    assert torch.equal(p, 1 - LR * torch.arange(4.0, dtype=torch.float64))
    assert bool((acc.buffers()[0][1] == 0).all())


def test_replicated_and_owned_buffers_in_one_accumulator():
    comm = _CountingComm()
    acc = AccumulatedSGD(LR)
    rep, own = torch.ones(3, dtype=torch.float64), torch.ones(5, dtype=torch.float64)
    acc.buffer(rep, comm).fill_(2.0)
    acc.buffer(own, None).fill_(4.0)
    acc.step()
    assert comm.calls == 1, "exactly the replicated buffer is all-reduced"
    assert torch.equal(rep, torch.full_like(rep, 1 - LR / 2 * (2.0 + 2.0)))  # -lr / P times both ranks' buffers
    assert torch.equal(own, torch.full_like(own, 1 - LR * 4.0))


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_frozen_parameters_get_no_buffer(kind):
    E, D, H, O = 2, 8, 12, 6
    ps = [p.clone().requires_grad_(i != 0) for i, p in enumerate(_params(E, D, H, O, 2))]  # w1 frozen
    w1 = ps[0].clone()
    (fwd, r), = _micro_batches(kind, 1, E, D, O)
    acc = AccumulatedSGD(LR)
    (fwd(ps, accumulator=acc) * r).sum().backward()
    assert not any(p is ps[0] for p, _ in acc.buffers()) and len(acc.buffers()) == 3
    acc.step()
    assert torch.equal(ps[0], w1)


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_backward_after_step_raises(kind):
    E, D, H, O = 2, 8, 12, 6
    ps = [p.clone().requires_grad_() for p in _params(E, D, H, O, 3)]
    (fwd, r), = _micro_batches(kind, 1, E, D, O)
    acc = AccumulatedSGD(LR)
    loss = (fwd(ps, accumulator=acc) * r).sum()
    acc.step()
    with pytest.raises(RuntimeError, match="step\\(\\) ran between"):
        loss.backward()


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_update_mode_errors(kind):
    E, D, H, O = 2, 8, 12, 6
    ps = _params(E, D, H, O, 4)
    (fwd, _), = _micro_batches(kind, 1, E, D, O)
    with pytest.raises(ValueError, match="not both"):
        fwd(ps, optimizer=InBackwardSGD(LR), accumulator=AccumulatedSGD(LR))
    with pytest.raises(RuntimeError, match="CUDA kernel path"):
        fwd(ps, optimizer=InBackwardSGD(LR))


@pytest.mark.parametrize("nprocs", [2, 3])
def test_layer_accumulator_steps_cpu(nprocs):
    res = run_spmd(nprocs, ["tests/spmd/expert_update_steps.py"], device="cpu", timeout=600)
    assert res.returncode == 0, f"np={nprocs}\nSTDOUT:\n{res.stdout[-4000:]}\nSTDERR:\n{res.stderr[-8000:]}"
    assert f"expert_update_steps np={nprocs} device=cpu ok=True" in res.stdout


def test_moe_example_micro_batches_cpu():
    res = run_spmd(2, ["examples/moe_layer.py", "--device", "cpu", "--steps", "20", "--micro-batches", "2"],
                   device="cpu", timeout=300)
    assert res.returncode == 0, res.stderr[-4000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", res.stdout)]
    assert len(losses) == 20 and losses[-1] < losses[0], losses
