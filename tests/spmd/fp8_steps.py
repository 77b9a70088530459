"""A few fp8 steps of ``DPLinearModel(fp8=True)`` in plain-gradient mode (``.grad`` + SGD) against a single-process
emulation of the global batch: every rank quantizes its own x and dy with its own scales, and the gradient of the
global loss is the sum of the ranks' gradients.  The weights must be bit-identical on every rank.

CPU (M4T_TEST_DEVICE=cpu): float64 through the torch composition, tolerance 1e-12 relative.
CUDA: bf16 through the fp8 kernels, 2 % of the loss and a few bf16 ulps of the weights."""
import torch

from common import DEVICE, comm

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPLinearModel
from mpi4torch_b200.ops.fp8 import E4M3, E5M2, dequantize, quantize_fp8_reference

P, RANK = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"
STEPS = 3
LR = 0.25


def batches(B, D, O, step, dtype):
    g = torch.Generator().manual_seed(3000 + step)
    xs = [torch.randn(B, D, generator=g).to(dtype) for _ in range(P)]
    ts = [torch.randn(B, O, generator=g).to(dtype) for _ in range(P)]
    return xs, ts


def deq(v, fmt):
    q, inv = quantize_fp8_reference(v, fmt)
    return dequantize(q, inv, torch.float64)


def reference(w, B, D, O, dtype):
    """float64 emulation of STEPS plain-gradient steps on the global batch; the weight is rounded to its dtype."""
    losses = []
    for step in range(STEPS):
        xs, ts = batches(B, D, O, step, dtype)
        wd = deq(w, E4M3)  # the ranks' average of identical weights is the weight
        loss, grad = 0.0, torch.zeros(w.shape, dtype=torch.float64)
        for x, t in zip(xs, ts):
            xd = deq(x, E4M3)
            d = xd @ wd.t() - t.double()
            loss += float(d.square().sum()) / (B * P)
            dy = (d * (2.0 / (B * P))).to(dtype)
            grad += deq(dy, E5M2).t() @ xd
        # the loss is the sum over ranks: its gradient sums every rank's local gradient
        w = (w.double() - LR * grad.to(dtype).double()).to(dtype)
        losses.append(loss)
    return losses, w


def check(B, D, O):
    dtype = torch.bfloat16 if CUDA else torch.float64
    model = DPLinearModel(D, O, comm, device=DEVICE, dtype=dtype, lr=LR, seed=5, sgd_in_backward=False, fp8=True)
    w0 = model.weight.detach().cpu().clone()
    losses = []
    for step in range(STEPS):
        xs, ts = batches(B, D, O, step, dtype)
        losses.append(float(model.train_step(xs[RANK].to(DEVICE), ts[RANK].to(DEVICE))))
    ref_losses, ref_w = reference(w0, B, D, O, dtype)
    rel = 2e-2 if CUDA else 1e-12
    what = f"np={P} shape={(B, D, O)}"
    for got, want in zip(losses, ref_losses):
        assert abs(got - want) <= rel * abs(want), f"{what}: loss {got} vs {want} (all {losses} vs {ref_losses})"
    w = model.weight.detach().double()
    err = float((w.cpu() - ref_w.double()).abs().max())
    # CUDA: a few bf16 ulps of the largest weight (an fp8 rounding of dy can flip against the emulation's)
    assert err <= (5e-2 if CUDA else 1e-12) * float(ref_w.double().abs().max()), f"{what}: weight off by {err}"
    assert torch.equal(comm.Allreduce(w, m4t.MPI_MAX), w) and torch.equal(comm.Allreduce(w, m4t.MPI_MIN), w), \
        f"{what}: the weight differs across ranks"
    assert model.weight.grad is None
    return losses


if __name__ == "__main__":
    shapes = [(256, 256, 128)] if CUDA else [(16, 12, 8), (40, 24, 16)]
    for shape in shapes:
        losses = check(*shape)
        if RANK == 0:
            print(f"[fp8_steps] shape={shape} losses={losses}", flush=True)
    if RANK == 0:
        print(f"fp8_steps np={P} device={DEVICE.type} ok=True", flush=True)
