"""Three training steps of DPMLPClassifier in both optimizer modes against a single-process fp64 torch reference of
the global loss (every rank's batch, parameters averaged over ranks), plus bit-identical parameters on every rank.

Some rows of every batch are labelled ignore_index: the global loss is sum over non-ignored rows of CE / (B * P).
CPU (M4T_TEST_DEVICE=cpu): float64 parameters through the composition path, tolerance 1e-6 relative.
CUDA: bf16 weights / fp32 biases through the kernels, tolerance of the bf16 compute type."""
import torch
import torch.nn.functional as F

from common import DEVICE, comm

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPMLPClassifier

P, RANK = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"
STEPS = 3
IGNORE = -100


def batches(B, D, C, step, dtype):
    """Every rank's batch of one step (all ranks generate all of them: the reference needs them)."""
    g = torch.Generator().manual_seed(2000 + step)
    xs = [torch.randn(B, D, generator=g).to(dtype) for _ in range(P)]
    labels = [torch.randint(0, C, (B,), generator=g) for _ in range(P)]
    for i, lab in enumerate(labels):
        lab[i::7] = IGNORE
    return xs, labels


def reference(params, B, D, C, lr, dtype):
    """fp64 SGD on the global loss sum_ranks sum_rows CE(MLP(x_r), labels_r) / (B * P)."""
    w1, b1, w2, b2 = [p.detach().double().cpu().clone().requires_grad_() for p in params]
    losses = []
    for step in range(STEPS):
        xs, labels = batches(B, D, C, step, dtype)
        x, lab = torch.cat(xs).double(), torch.cat(labels)
        y = F.linear(F.gelu(F.linear(x, w1, b1), approximate="tanh"), w2, b2)
        loss = F.cross_entropy(y, lab, reduction="sum", ignore_index=IGNORE) / (B * P)
        loss.backward()
        with torch.no_grad():
            for p in (w1, b1, w2, b2):
                p -= lr * p.grad
                p.grad = None
        losses.append(float(loss))
    return losses, [p.detach() for p in (w1, b1, w2, b2)]


def check(B, D, H, C, sgd_in_backward):
    dtype = torch.bfloat16 if CUDA else torch.float64
    lr = 0.5
    model = DPMLPClassifier(D, H, C, comm, device=DEVICE, dtype=dtype, lr=lr, seed=9, sgd_in_backward=sgd_in_backward)
    init = [p.detach().clone() for p in model.parameters()]
    losses = []
    for step in range(STEPS):
        xs, labels = batches(B, D, C, step, dtype)
        losses.append(float(model.train_step(xs[RANK].to(DEVICE), labels[RANK].to(DEVICE))))
    ref_losses, ref_params = reference(init, B, D, C, lr, dtype)
    loss_tol, param_tol = (1e-2, 2e-2) if CUDA else (1e-6, 1e-6)
    what = f"np={P} shape={(B, D, H, C)} sgd_in_backward={sgd_in_backward}"
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
    return losses


if __name__ == "__main__":
    shapes = [(128, 256, 256, 256)] if CUDA else [(16, 8, 12, 5), (128, 256, 256, 256)]
    for shape in shapes:
        for mode in (True, False):
            losses = check(*shape, sgd_in_backward=mode)
            if RANK == 0:
                print(f"[xent_steps] shape={shape} sgd_in_backward={mode} losses={losses}", flush=True)
    if RANK == 0:
        print(f"xent_steps np={P} device={DEVICE.type} ok=True", flush=True)
