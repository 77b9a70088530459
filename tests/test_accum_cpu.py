"""Gradient accumulation (AccumulatedSGD, ``train_step(..., micro_batches=K)``) on the CPU composition path in float64
at one rank: K accumulated micro-batches give the full-batch step, and the accumulator's rules hold."""
import pytest
import torch

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPLinearModel, DPMLPClassifier, DPMLPModel
from mpi4torch_b200.ops import AccumulatedSGD, dp_linear_mse, dp_mlp_cross_entropy, dp_mlp_mse

B, D, H, O, C = 32, 12, 16, 6, 5
LR = 0.1


def _model(kind, **kw):
    comm = m4t.COMM_WORLD
    if kind == "linear":
        return DPLinearModel(D, O, comm, device="cpu", dtype=torch.float64, lr=LR, seed=1, **kw)
    if kind == "mlp":
        return DPMLPModel(D, H, O, comm, device="cpu", dtype=torch.float64, lr=LR, seed=1, **kw)
    return DPMLPClassifier(D, H, C, comm, device="cpu", dtype=torch.float64, lr=LR, seed=1, **kw)


def _params(model):
    return [model.weight] if isinstance(model, DPLinearModel) else model.parameters()


def _batch(kind, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, generator=g, dtype=torch.float64)
    if kind == "classifier":
        return x, torch.randint(0, C, (B,), generator=g)
    return x, torch.randn(B, O, generator=g, dtype=torch.float64)


def _assert_close(got, want, what, rel=1e-12):
    err = float((got - want).abs().max())
    assert err <= rel * float(want.abs().max()), f"{what}: off by {err}"


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("kind", ["linear", "mlp", "classifier"])
def test_micro_batches_equal_full_batch(kind, K):
    full, accum = _model(kind), _model(kind)
    for step in range(2):
        x, t = _batch(kind, 10 + step)
        l_full = full.train_step(x, t)
        l_acc = accum.train_step(x, t, micro_batches=K)
        _assert_close(l_acc, l_full, f"{kind} K={K} step {step} loss")
        for i, (p, q) in enumerate(zip(_params(accum), _params(full))):
            _assert_close(p.detach(), q.detach(), f"{kind} K={K} step {step} param {i}")
    for p in _params(accum):
        assert p.grad is None, f"{kind}: a .grad was left behind"
    bufs = accum.accumulator.buffers()
    assert len(bufs) == len(_params(accum))
    for p, buf in bufs:
        assert buf.dtype == p.dtype and not bool(buf.any()), "a buffer is not zero after step()"
    assert accum.accumulator.updates == 2


@pytest.mark.parametrize("kind", ["linear", "mlp", "classifier"])
def test_micro_batches_must_divide_the_batch(kind):
    model = _model(kind)
    x, t = _batch(kind, 1)
    before = [p.detach().clone() for p in _params(model)]
    for K in (3, 0, -2):
        with pytest.raises(ValueError, match="micro_batches"):
            model.train_step(x, t, micro_batches=K)
    assert all(torch.equal(p.detach(), q) for p, q in zip(_params(model), before))


def _mlp_params(seed=3):
    g = torch.Generator().manual_seed(seed)
    shapes = ((H, D), (H,), (O, H), (O,))
    return [torch.randn(*s, generator=g, dtype=torch.float64).requires_grad_() for s in shapes]


def test_stacked_forwards_equal_separate_backwards():
    comm = m4t.COMM_WORLD
    (xa, ta), (xb, tb) = _batch("mlp", 4), _batch("mlp", 5)
    bufs = []
    for stacked in (True, False):
        params = _mlp_params()
        acc = AccumulatedSGD(LR)
        la = dp_mlp_mse(xa, *params, ta, comm, loss_scale=0.5, accumulator=acc)
        if stacked:
            lb = dp_mlp_mse(xb, *params, tb, comm, loss_scale=0.5, accumulator=acc)
            (la + lb).backward()
        else:
            la.backward()
            dp_mlp_mse(xb, *params, tb, comm, loss_scale=0.5, accumulator=acc).backward()
        assert all(p.grad is None for p in params)
        by_param = {id(p): b for p, b in acc.buffers()}
        bufs.append([by_param[id(p)].clone() for p in params])
    for a, b in zip(*bufs):
        assert torch.equal(a, b)
    # the buffers hold the gradient of the summed loss
    params = _mlp_params()
    (dp_mlp_mse(xa, *params, ta, comm, loss_scale=0.5) + dp_mlp_mse(xb, *params, tb, comm, loss_scale=0.5)).backward()
    for p, b in zip(params, bufs[0]):
        _assert_close(b, p.grad, "accumulated gradient")


@pytest.mark.parametrize("frozen", range(4), ids=["w1", "b1", "w2", "b2"])
def test_frozen_parameter_gets_no_buffer(frozen):
    comm = m4t.COMM_WORLD
    params = _mlp_params()
    params[frozen].requires_grad_(False)
    before = [p.detach().clone() for p in params]
    acc = AccumulatedSGD(LR)
    x, t = _batch("mlp", 6)
    dp_mlp_mse(x, *params, t, comm, loss_scale=0.5, accumulator=acc).backward()
    assert all(p is not params[frozen] for p, _ in acc.buffers()) and len(acc.buffers()) == 3
    acc.step()
    assert torch.equal(params[frozen], before[frozen])
    assert all(not torch.equal(p.detach(), q) for i, (p, q) in enumerate(zip(params, before)) if i != frozen)


@pytest.mark.parametrize("kind", ["linear", "mlp", "classifier"])
def test_forward_before_step_raises_in_backward(kind):
    comm = m4t.COMM_WORLD
    acc = AccumulatedSGD(LR)
    x, t = _batch(kind, 8)
    if kind == "linear":
        w = torch.randn(O, D, dtype=torch.float64, requires_grad=True)
        stale = dp_linear_mse(x, w, t, comm, loss_scale=0.5, accumulator=acc)
        dp_linear_mse(x, w, t, comm, loss_scale=0.5, accumulator=acc).backward()
    else:
        params = _mlp_params()
        if kind == "classifier":
            params = [params[0], params[1], torch.randn(C, H, dtype=torch.float64, requires_grad=True),
                      torch.zeros(C, dtype=torch.float64, requires_grad=True)]
        node = dp_mlp_mse if kind == "mlp" else dp_mlp_cross_entropy
        stale = node(x, *params, t, comm, loss_scale=0.5, accumulator=acc)
        node(x, *params, t, comm, loss_scale=0.5, accumulator=acc).backward()
    acc.step()
    with pytest.raises(RuntimeError, match="step\\(\\) ran between"):
        stale.backward()


def test_accumulator_and_optimizers_are_exclusive():
    from mpi4torch_b200.ops import InBackwardSGD

    comm = m4t.COMM_WORLD
    acc = AccumulatedSGD(LR)
    x, t = _batch("mlp", 9)
    params = _mlp_params()
    opts = (InBackwardSGD(LR), InBackwardSGD(LR))
    with pytest.raises(ValueError, match="not both"):
        dp_mlp_mse(x, *params, t, comm, loss_scale=1.0, optimizers=opts, accumulator=acc)
    labels = torch.zeros(B, dtype=torch.int64)
    with pytest.raises(ValueError, match="not both"):
        dp_mlp_cross_entropy(x, params[0], params[1], params[2], params[3], labels, comm, loss_scale=1.0,
                             optimizers=opts, accumulator=acc)
    w = torch.randn(O, D, dtype=torch.float64, requires_grad=True)
    with pytest.raises(ValueError, match="not both"):
        dp_linear_mse(x, w, t, comm, loss_scale=1.0, optimizer=opts[0], accumulator=acc)


def test_averages_are_computed_once_per_step():
    """The forwards of one step share the parameter averages; step() and a manual edit drop them."""
    comm = m4t.COMM_WORLD
    acc = AccumulatedSGD(LR)
    w = torch.randn(O, D, dtype=torch.float64, requires_grad=True)
    a1 = acc.average(comm, w)
    assert acc.average(comm, w) is a1
    acc.step()
    a2 = acc.average(comm, w)
    assert a2 is not a1
    with torch.no_grad():
        w.mul_(2.0)
    assert acc.cached_average(w) is None


def test_buffer_dtypes():
    acc = AccumulatedSGD(LR)
    comm = m4t.COMM_WORLD
    for dtype, want in ((torch.bfloat16, torch.float32), (torch.float16, torch.float32), (torch.float32, torch.float32),
                        (torch.float64, torch.float64)):
        p = torch.zeros(3, 4, dtype=dtype)
        assert acc.buffer(p, comm).dtype == want
