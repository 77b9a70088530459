"""ExpertParallelMLP with an AccumulatedSGD over several ranks, in capacity and dropless routing: K micro-batches
through the accumulator and one step() leave, on every rank, the parameters of one plain SGD step on the plain
gradients of the whole batch.  The experts' buffers are owned, so step() issues no collective for them.

CPU (M4T_TEST_DEVICE=cpu): float64 layers through the composition path, tolerance 1e-12.
CUDA: bf16 experts on the kernels, tolerance of the bf16 compute type."""
import torch

from common import DEVICE, comm

from mpi4torch_b200.ops import AccumulatedSGD
from mpi4torch_b200.parallel import ExpertParallelMLP

P, RANK = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"
LR = 0.25


def check(capacity, T, d, hidden, E, k, K):
    dtype = torch.bfloat16 if CUDA else torch.float64
    # capacity T * k: no pair is dropped, so the micro-batches route exactly as the whole batch
    cap = None if capacity is None else T * k
    plain, accum = (ExpertParallelMLP(d, hidden, E, cap, comm, top_k=k, dtype=dtype, device=DEVICE, seed=31)
                    for _ in range(2))
    gen = torch.Generator().manual_seed(400 + RANK)
    x = torch.randn(T, d, generator=gen).to(dtype).to(DEVICE)
    r = torch.randn(T, d, generator=gen, dtype=torch.float64).to(DEVICE)

    out, _ = plain(x)
    (out.double() * r).sum().backward()
    names = ("w1", "b1", "w2", "b2")
    want = [(getattr(plain, n) - LR * getattr(plain, n).grad).detach() for n in names]

    acc = AccumulatedSGD(LR)
    for xk, rk in zip(x.chunk(K), r.chunk(K)):
        out, info = accum(xk, accumulator=acc)
        assert not bool(info.dropped.any())
        (out.double() * rk).sum().backward()
    assert all(getattr(accum, n).grad is None for n in names), "an expert parameter got a .grad"
    acc.step()
    tol = 2e-2 if CUDA else 1e-12
    what = f"np={P} capacity={capacity} k={k} K={K}"
    for n, ref in zip(names, want):
        got = getattr(accum, n).detach()
        err = float((got.double() - ref.double()).abs().max())
        assert err <= tol * max(1.0, float(ref.double().abs().max())), f"{what}: {n} off by {err}"
    # the router keeps its plain gradient, summed over the micro-batches
    err = float((accum.router.grad - plain.router.grad).abs().max())
    assert err <= tol * max(1.0, float(plain.router.grad.abs().max())), f"{what}: router.grad off by {err}"


if __name__ == "__main__":
    shape = dict(T=256, d=128, hidden=256, E=2) if CUDA else dict(T=24, d=8, hidden=12, E=3)
    for capacity in ("capacity", None):
        for k in (1, 2):
            check(capacity, **shape, k=k, K=2)
    check(None, **shape, k=2, K=3 if not CUDA else 2)
    if RANK == 0:
        print(f"expert_update_steps np={P} device={DEVICE.type} ok=True", flush=True)
