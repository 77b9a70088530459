"""Dropless expert parallelism over several ranks: ExpertParallelMLP(capacity=None)'s output and all gradients against
the single-process float64 reference of the whole global batch, under a skewed router that makes capacity routing drop
pairs.

CPU (M4T_TEST_DEVICE=cpu): float64 layers through the composition path, tolerance 1e-10.
CUDA: bf16 experts on the grouped kernels, tolerance of the bf16 compute type."""
import torch

from common import DEVICE, comm
from moe_steps import reference_layer, reference_slots

import mpi4torch_b200 as m4t
from mpi4torch_b200.parallel import ExpertParallelMLP

P, RANK = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"


def check_dropless(T, d, hidden, E, k):
    dtype = torch.bfloat16 if CUDA else torch.float64
    layer = ExpertParallelMLP(d, hidden, E, None, comm, top_k=k, dtype=dtype, device=DEVICE, seed=23)
    with torch.no_grad():  # skew: global expert 0 is every token's most probable choice, most of the time
        layer.router[0] += 0.5 * layer.router[1:].abs().sum(0).sign()
    gen = torch.Generator().manual_seed(211 + k)
    xs = [(torch.randn(T, d, generator=gen).abs() + 0.1).to(dtype) for _ in range(P)]
    rs = [torch.randn(T, d, generator=gen, dtype=torch.float64) for _ in range(P)]
    x = xs[RANK].to(DEVICE).requires_grad_()
    out, info = layer(x)
    (out.double() * rs[RANK].to(DEVICE)).sum().backward()
    assert not bool(info.dropped.any()), "dropless routing dropped a pair"
    G = P * E
    fair = -(-T * k // G)  # the capacity of an even split
    skew_drops = int((reference_slots(info.expert.cpu(), G, fair) < 0).sum())
    full = [comm.Allgather(p.detach().contiguous(), 0) for p in (layer.w1, layer.b1, layer.w2, layer.b2)]
    choices = list(comm.Allgather(info.expert.contiguous(), 0).cpu().reshape(P, T, k))
    # capacity T * k: the reference drops nothing either
    ins, outs, _ = reference_layer(xs, layer.router.detach(), *full, k, E, T * k, choices)
    sum((o * r).sum() for o, r in zip(outs, rs)).backward()
    tol = 3e-2 if CUDA else 1e-10
    what = f"np={P} k={k}"

    def close(got, ref, name):
        got = got.detach().double().cpu()
        err = float((got - ref).abs().max())
        assert err <= tol * max(1.0, float(ref.abs().max())), f"{what}: {name} off by {err}"

    close(out, outs[RANK].detach(), "out")
    close(x.grad, ins[5 + RANK].grad, "x.grad")
    close(layer.router.grad, ins[0].grad, "router.grad")
    mine = slice(RANK * E, (RANK + 1) * E)
    for name, p, ref in zip(("w1", "b1", "w2", "b2"), (layer.w1, layer.b1, layer.w2, layer.b2), ins[1:5]):
        close(p.grad, ref.grad[mine], f"{name}.grad")
    return skew_drops


if __name__ == "__main__":
    shape = dict(T=256, d=128, hidden=256, E=4) if CUDA else dict(T=24, d=8, hidden=12, E=3)
    for k in (1, 2):
        drops = check_dropless(**shape, k=k)
        total = int(comm.Allreduce(torch.tensor([float(drops)], device=DEVICE), m4t.MPI_SUM).item())
        assert total > 0, "the skew is too weak: capacity routing at an even split would drop nothing"
        if RANK == 0:
            print(f"[grouped_moe_steps] k={k} {shape}: even-split capacity would drop {total} pairs, dropless none",
                  flush=True)
    if RANK == 0:
        print(f"grouped_moe_steps np={P} device={DEVICE.type} ok=True", flush=True)
