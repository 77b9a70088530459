"""Expert parallelism over several ranks: the per-expert dispatch layout, capacity drops with top-2 priority, the
inverse exchange, and ExpertParallelMLP's output and gradients against a single-process float64 reference of the whole
global batch with all P * E experts.

CPU (M4T_TEST_DEVICE=cpu): float64 layers through the composition path, tolerance 1e-10.
CUDA: bf16 experts on the batched kernels (P * capacity % 128 == 0), tolerance of the bf16 compute type."""
import math

import torch
import torch.nn.functional as F

from common import DEVICE, comm

import mpi4torch_b200 as m4t
from mpi4torch_b200.parallel import ExpertParallelMLP, combine_from_experts, dispatch_to_experts

P, RANK = comm.size, comm.rank
CUDA = DEVICE.type == "cuda"


def reference_slots(choice, G, C):
    """[T, k] slot of every pair of one source rank, choice-major, -1 over capacity (plain loops)."""
    T, k = choice.shape
    count = [0] * G
    slot = torch.full((T, k), -1, dtype=torch.int64)
    for j in range(k):
        for t in range(T):
            g = int(choice[t, j])
            if count[g] < C:
                slot[t, j] = count[g]
            count[g] += 1
    return slot


def check_dispatch(T, d, E, C, k):
    G = P * E
    gen = torch.Generator().manual_seed(31 + 7 * k)
    # every rank's tokens and choices (all ranks generate all of them: the reference needs them)
    toks = [torch.randn(T, d, generator=gen, dtype=torch.float64) for _ in range(P)]
    choices = [torch.stack([torch.randperm(G, generator=gen)[:k] for _ in range(T)]) for _ in range(P)]
    tokens = toks[RANK].to(DEVICE).requires_grad_()
    received, routing = dispatch_to_experts(tokens, choices[RANK].to(DEVICE), E, C, comm)
    assert tuple(received.shape) == (E, P * C, d), received.shape
    want = torch.zeros(E, P * C, d, dtype=torch.float64)
    for p in range(P):
        slot = reference_slots(choices[p], G, C)
        if p == RANK:
            assert torch.equal(routing.slot.cpu(), slot), f"k={k}: slots {routing.slot} vs {slot}"
        for t in range(T):
            for j in range(k):
                g = int(choices[p][t, j])
                if slot[t, j] >= 0 and g // E == RANK:
                    want[g % E, p * C + slot[t, j]] = toks[p][t]
    assert torch.equal(received.detach().cpu(), want), f"k={k}: dispatch layout"
    # top-2 priority: no second choice holds a slot while a first choice to the same expert was dropped
    mine = reference_slots(choices[RANK], G, C)
    if k == 2:
        for g in range(G):
            first_dropped = bool(((choices[RANK][:, 0] == g) & (mine[:, 0] < 0)).any())
            second_kept = bool(((choices[RANK][:, 1] == g) & (mine[:, 1] >= 0)).any())
            assert not (first_dropped and second_kept), f"expert {g}: a second choice beat a first choice"
    # the inverse exchange returns each pair's own row (here 3 * token + expert id), zero for dropped pairs
    ids = torch.arange(E, dtype=torch.float64, device=DEVICE)[:, None, None] + RANK * E
    back = combine_from_experts(3.0 * received + ids, routing, comm)
    want_back = (3.0 * toks[RANK][:, None, :] + choices[RANK][:, :, None].double()) * (mine >= 0)[:, :, None]
    assert torch.equal(back.detach().cpu(), want_back), f"k={k}: combine"
    # backward of both exchanges: d/dtokens sum(back * w) = 3 * sum over kept choices of w
    w = torch.randn(back.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    (back * w.to(DEVICE)).sum().backward()
    assert torch.allclose(tokens.grad.cpu(), 3.0 * (w * (mine >= 0)[:, :, None]).sum(1), rtol=0, atol=1e-12)
    dropped = int((mine < 0).sum())
    return dropped


def reference_layer(xs, router, w1, b1, w2, b2, k, E, C, choices=None):
    """All P ranks' batches through all P * E experts in float64: outputs per rank, and the gradient of
    sum_p sum(out_p * R_p) with respect to every input."""
    G = P * E
    ins = [t.detach().double().cpu().clone().requires_grad_() for t in [router, w1, b1, w2, b2] + xs]
    router, w1, b1, w2, b2 = ins[:5]
    outs, picked = [], []
    for p, x in enumerate(ins[5:]):
        probs = torch.softmax(x @ router.t(), -1)
        gate, choice = probs.topk(k, -1)
        if choices is not None:
            choice = choices[p]
            gate = probs.gather(1, choice)
        picked.append(choice)
        slot = reference_slots(choice, G, C)
        out = torch.zeros_like(x)
        for j in range(k):
            g = choice[:, j]
            h = F.gelu(torch.einsum("td,thd->th", x, w1[g]) + b1[g], approximate="tanh")
            y = torch.einsum("th,toh->to", h, w2[g]) + b2[g]
            out = out + gate[:, j:j + 1] * y * (slot[:, j:j + 1] >= 0)
        outs.append(out)
    return ins, outs, picked


def check_layer(T, d, hidden, E, C, k):
    dtype = torch.bfloat16 if CUDA else torch.float64
    layer = ExpertParallelMLP(d, hidden, E, C, comm, top_k=k, dtype=dtype, device=DEVICE, seed=17)
    gen = torch.Generator().manual_seed(101 + k)
    xs = [torch.randn(T, d, generator=gen).to(dtype) for _ in range(P)]
    rs = [torch.randn(T, d, generator=gen, dtype=torch.float64) for _ in range(P)]
    x = xs[RANK].to(DEVICE).requires_grad_()
    out, info = layer(x)
    (out.double() * rs[RANK].to(DEVICE)).sum().backward()
    full = [comm.Allgather(p.detach().contiguous(), 0) for p in (layer.w1, layer.b1, layer.w2, layer.b2)]
    # the layer's choices, gathered, so that a near-tie rounded differently on the GPU cannot change the reference
    choices = list(comm.Allgather(info.expert.contiguous(), 0).cpu().reshape(P, T, k)) if CUDA else None
    ins, outs, picked = reference_layer(xs, layer.router.detach(), *full, k, E, C, choices)
    sum((o * r).sum() for o, r in zip(outs, rs)).backward()
    tol = 3e-2 if CUDA else 1e-10
    what = f"np={P} k={k} C={C}"

    def close(got, ref, name):
        got = got.detach().double().cpu()
        err = float((got - ref).abs().max())
        assert err <= tol * max(1.0, float(ref.abs().max())), f"{what}: {name} off by {err}"

    if not CUDA:
        assert torch.equal(info.expert.cpu(), picked[RANK]), f"{what}: routing differs from the reference"
    else:
        agree = float((torch.topk(ins[5 + RANK].detach() @ ins[0].detach().t(), k, -1)[1] == info.expert.cpu())
                      .double().mean())
        assert agree >= 0.98, f"{what}: only {agree} of the choices agree with the float64 router"
    assert torch.equal(info.dropped.cpu(), reference_slots(info.expert.cpu(), P * E, C) < 0)
    close(out, outs[RANK].detach(), "out")
    close(x.grad, ins[5 + RANK].grad, "x.grad")
    close(layer.router.grad, ins[0].grad, "router.grad")
    g = layer.router.grad.double()
    assert torch.equal(comm.Allreduce(g, m4t.MPI_MAX), g), f"{what}: the router gradient differs across ranks"
    mine = slice(RANK * E, (RANK + 1) * E)
    for name, p, ref in zip(("w1", "b1", "w2", "b2"), (layer.w1, layer.b1, layer.w2, layer.b2), ins[1:5]):
        close(p.grad, ref.grad[mine], f"{name}.grad")
    return int(info.dropped.sum())


if __name__ == "__main__":
    E = 2
    for k in (1, 2):
        dropped = check_dispatch(T=12, d=3, E=E, C=3, k=k)
        assert dropped > 0 or P * E * 3 >= 12 * k, "the dispatch case drops nothing"
        if RANK == 0:
            print(f"[moe_steps] dispatch k={k} dropped={dropped}", flush=True)
    if CUDA:
        shape = dict(T=256, d=128, hidden=256, E=4, C=128 // math.gcd(128, P))
    else:
        shape = dict(T=24, d=8, hidden=12, E=2, C=5)
    for k in (1, 2):
        dropped = check_layer(**shape, k=k)
        if RANK == 0:
            print(f"[moe_steps] layer k={k} {shape} dropped={dropped}", flush=True)
    if RANK == 0:
        print(f"moe_steps np={P} device={DEVICE.type} ok=True", flush=True)
