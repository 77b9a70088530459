"""Three gradient-accumulation steps (``train_step(..., micro_batches=K)``) of DPMLPModel and DPMLPClassifier against a
single-process fp64 torch reference of SGD on the whole global batch, plus bit-identical parameters on every rank.

CPU (M4T_TEST_DEVICE=cpu): float64 parameters through the composition path, tolerance 1e-6 relative.
CUDA: bf16 weights / fp32 biases through the kernels (``wgrad_accumulate_`` into fp32 buffers), tolerance of the
bf16 compute type."""
import torch
import torch.nn.functional as F

from common import DEVICE, comm

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPMLPClassifier, DPMLPModel

P, RANK = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"
STEPS = 3


def batches(B, D, O, step, dtype, classes):
    """Every rank's batch of one step (all ranks generate all of them: the reference needs them)."""
    g = torch.Generator().manual_seed(2000 + step)
    xs = [torch.randn(B, D, generator=g).to(dtype) for _ in range(P)]
    if classes:
        ts = [torch.randint(0, O, (B,), generator=g) for _ in range(P)]
    else:
        ts = [torch.randn(B, O, generator=g).to(dtype) for _ in range(P)]
    return xs, ts


def reference(params, B, D, O, lr, dtype, classes):
    """fp64 SGD on the global loss sum_ranks loss(x_r, t_r) / (B * P), one update per step."""
    w1, b1, w2, b2 = [p.detach().double().cpu().clone().requires_grad_() for p in params]
    losses = []
    for step in range(STEPS):
        xs, ts = batches(B, D, O, step, dtype, classes)
        x, t = torch.cat(xs).double(), torch.cat(ts)
        y = F.linear(F.gelu(F.linear(x, w1, b1), approximate="tanh"), w2, b2)
        if classes:
            loss = F.cross_entropy(y, t, reduction="sum") / (B * P)
        else:
            loss = (y - t.double()).square().sum() / (B * P)
        loss.backward()
        with torch.no_grad():
            for p in (w1, b1, w2, b2):
                p -= lr * p.grad
                p.grad = None
        losses.append(float(loss))
    return losses, [p.detach() for p in (w1, b1, w2, b2)]


def check(B, D, H, O, K, classes):
    dtype = torch.bfloat16 if CUDA else torch.float64
    lr = 0.05
    cls = DPMLPClassifier if classes else DPMLPModel
    model = cls(D, H, O, comm, device=DEVICE, dtype=dtype, lr=lr, seed=11)
    init = [p.detach().clone() for p in model.parameters()]
    losses = []
    for step in range(STEPS):
        xs, ts = batches(B, D, O, step, dtype, classes)
        losses.append(float(model.train_step(xs[RANK].to(DEVICE), ts[RANK].to(DEVICE), micro_batches=K)))
    ref_losses, ref_params = reference(init, B, D, O, lr, dtype, classes)
    loss_tol, param_tol = (1e-2, 2e-2) if CUDA else (1e-6, 1e-6)
    what = f"np={P} shape={(B, D, H, O)} K={K} {cls.__name__}"
    for got, ref in zip(losses, ref_losses):
        assert abs(got - ref) <= loss_tol * abs(ref), f"{what}: loss {got} vs {ref}"
    for name, p, ref in zip(("w1", "b1", "w2", "b2"), model.parameters(), ref_params):
        err = float((p.detach().double().cpu() - ref).abs().max())
        bound = param_tol if CUDA else param_tol * float(ref.abs().max())
        assert err <= bound, f"{what}: {name} off by {err}"
        assert p.grad is None, f"{what}: {name}.grad left behind"
        # bit-identical on every rank: the exact fp64 image of the parameter has the same max and min over ranks
        v = p.detach().double()
        assert torch.equal(comm.Allreduce(v, m4t.MPI_MAX), v) and torch.equal(comm.Allreduce(v, m4t.MPI_MIN), v), \
            f"{what}: {name} differs across ranks"
    for p, buf in model.accumulator.buffers():
        assert not bool(buf.any()), f"{what}: a buffer is not zero after step()"
    assert model.accumulator.updates == STEPS
    return losses


if __name__ == "__main__":
    shapes = [(256, 256, 256, 256)] if CUDA else [(16, 8, 12, 4), (128, 256, 256, 256)]
    for shape in shapes:
        for classes in (False, True):
            for K in (2, 4):
                losses = check(*shape, K=K, classes=classes)
                if RANK == 0:
                    print(f"[accum_steps] shape={shape} K={K} classes={classes} losses={losses}", flush=True)
    if RANK == 0:
        print(f"accum_steps np={P} device={DEVICE.type} ok=True", flush=True)
