"""dp_mlp_cross_entropy and DPMLPClassifier off the kernel path (CPU tensors, world size 1): the torch composition
against F.cross_entropy, argument validation, and the shipped classifier example at np = 2 on the CPU backend."""
import re

import pytest
import torch
import torch.nn.functional as F

import mpi4torch_b200 as m4t
from conftest import run_spmd
from mpi4torch_b200.models import DPMLPClassifier
from mpi4torch_b200.ops import dp_mlp_cross_entropy, dp_mlp_cross_entropy_supported


def _params(B=12, D=8, H=16, C=5, dtype=torch.float64):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(B, D, generator=g, dtype=dtype)
    w1 = torch.randn(H, D, generator=g, dtype=dtype).requires_grad_()
    b1 = torch.randn(H, generator=g, dtype=dtype).requires_grad_()
    w2 = torch.randn(C, H, generator=g, dtype=dtype).requires_grad_()
    b2 = torch.randn(C, generator=g, dtype=dtype).requires_grad_()
    labels = torch.randint(0, C, (B,), generator=g)
    return x, w1, b1, w2, b2, labels


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
def test_composition_matches_cross_entropy(dtype):
    x, w1, b1, w2, b2, labels = _params(dtype=dtype)
    labels[2] = -100
    labels[7] = 3
    assert not dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels)
    loss = dp_mlp_cross_entropy(x, w1, b1, w2, b2, labels, loss_scale=0.25)
    assert loss.shape == (1,) and loss.dtype == dtype
    loss.sum().backward()
    got = [p.grad.clone() for p in (w1, b1, w2, b2)]
    for p in (w1, b1, w2, b2):
        p.grad = None
    y = F.linear(F.gelu(F.linear(x, w1, b1), approximate="tanh"), w2, b2)
    ref = F.cross_entropy(y, labels, reduction="sum", ignore_index=-100) * 0.25
    ref.backward()
    tol = 1e-12 if dtype == torch.float64 else 1e-5
    loss, ref = loss.detach(), ref.detach()
    assert abs(float(loss) - float(ref)) <= tol * abs(float(ref))
    for g, p in zip(got, (w1, b1, w2, b2)):
        assert torch.allclose(g, p.grad, rtol=tol, atol=tol)
    # a custom ignore_index
    labels[2] = 0
    with torch.no_grad():
        l3 = dp_mlp_cross_entropy(x, w1, b1, w2, b2, labels, loss_scale=1.0, ignore_index=3)
        want = F.cross_entropy(y, labels, reduction="sum", ignore_index=3)
    assert abs(float(l3) - float(want)) <= tol * abs(float(want))


def test_argument_validation():
    x, w1, b1, w2, b2, labels = _params()
    for bad in (labels.int(), labels.float(), labels[:-1], labels.reshape(3, 4), labels[:, None]):
        with pytest.raises(ValueError, match="labels"):
            dp_mlp_cross_entropy(x, w1, b1, w2, b2, bad, loss_scale=1.0)
        assert not dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, bad)
    from mpi4torch_b200.ops import InBackwardSGD

    with pytest.raises(RuntimeError, match="InBackwardSGD"):
        dp_mlp_cross_entropy(x, w1, b1, w2, b2, labels, loss_scale=1.0,
                             optimizers=(InBackwardSGD(0.1), InBackwardSGD(0.1)))


def test_classifier_trains_on_cpu():
    comm = m4t.COMM_WORLD
    model = DPMLPClassifier(8, 32, 3, comm, device="cpu", dtype=torch.float64, lr=0.5, seed=1)
    g = torch.Generator().manual_seed(0)
    centers = 3 * torch.randn(3, 8, generator=g, dtype=torch.float64)
    labels = torch.randint(0, 3, (64,), generator=g)
    x = centers[labels] + torch.randn(64, 8, generator=g, dtype=torch.float64)
    losses = [float(model.train_step(x, labels)) for _ in range(20)]
    assert losses[-1] < 0.5 * losses[0], losses
    assert all(p.grad is None for p in model.parameters())
    acc = float((model.logits(x).argmax(1) == labels).double().mean())
    assert acc > 0.9, acc
    # ignored rows count in the denominator B * P
    lab = labels.clone()
    lab[::2] = -100
    y = model.logits(x)
    want = F.cross_entropy(y, lab, reduction="sum") / 64
    assert abs(float(model.loss(x, lab)) - float(want)) <= 1e-12 * float(want)


def test_classifier_example_world_size_2_cpu():
    res = run_spmd(2, ["examples/dp_mlp_classifier.py", "--device", "cpu", "--steps", "12"], device="cpu", timeout=300)
    assert res.returncode == 0, res.stderr[-4000:]
    steps = re.findall(r"loss ([0-9.]+) accuracy ([0-9.]+)", res.stdout)
    assert len(steps) == 12, res.stdout[-2000:]
    losses = [float(a) for a, _ in steps]
    accs = [float(b) for _, b in steps]
    assert losses[-1] < 0.5 * losses[0], losses
    assert accs[-1] > accs[0] and accs[-1] >= 0.9, accs
