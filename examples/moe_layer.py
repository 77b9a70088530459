"""Mixture-of-experts regression: an ExpertParallelMLP (experts_per_rank experts on every rank, top-k routing with a
capacity per expert and source rank) followed by a replicated linear head, trained with plain SGD on a synthetic
target.  Every rank draws its own batch; the router and the head are replicated (their gradients are summed over
ranks), the experts are owned by their rank.  Each step prints the global loss and the share of dropped pairs.

    python -m mpi4torch_b200.launch -np 2 examples/moe_layer.py --device cpu
    python -m mpi4torch_b200.launch -np 8 examples/moe_layer.py --d-model 1024 --hidden 4096 --capacity 32
    python -m mpi4torch_b200.launch -np 2 examples/moe_layer.py --device cpu --dropless
    python -m mpi4torch_b200.launch -np 2 examples/moe_layer.py --device cpu --micro-batches 2
    python -m mpi4torch_b200.launch -np 8 examples/moe_layer.py --d-model 1024 --hidden 4096 --sgd-in-backward

On CUDA the experts run on the batched kernels when d_model and hidden are multiples of 128 and
size * capacity is a multiple of 128 (the default capacity is the smallest such one); otherwise they run the torch
composition.  With --dropless no pair is dropped: every expert takes exactly the rows routed to it, on the grouped
kernels when d_model and hidden are multiples of 128.

With --sgd-in-backward (CUDA kernel path only) the experts' SGD step runs inside backward, in their weight-gradient
kernels, and the experts get no .grad.  With --micro-batches K every step runs K forward/backward passes on slices of
the batch and the experts' gradients are summed in fp32 buffers (AccumulatedSGD) before one update.  The router and the
head keep their .grad and the plain SGD update in both modes.
"""
import argparse
import math

import torch
import torch.nn.functional as F

import mpi4torch_b200 as m4t
from mpi4torch_b200.ops import AccumulatedSGD, InBackwardSGD
from mpi4torch_b200.parallel import ExpertParallelMLP, replicated_input


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--d-model", type=int, default=128)
    ap.add_argument("--hidden", type=int, default=256)
    ap.add_argument("--experts-per-rank", type=int, default=4)
    ap.add_argument("--capacity", type=int, default=0, help="0: the smallest C with size * C % 128 == 0")
    ap.add_argument("--dropless", action="store_true", help="route without a capacity: no pair is dropped")
    ap.add_argument("--top-k", type=int, default=2)
    ap.add_argument("--lr", type=float, default=0.5)
    ap.add_argument("--device", default="cuda" if torch.cuda.is_available() else "cpu")
    ap.add_argument("--sgd-in-backward", action="store_true", help="update the experts inside backward (CUDA only)")
    ap.add_argument("--micro-batches", type=int, default=1, help="accumulate the experts' gradients over K slices")
    args = ap.parse_args()
    K = args.micro_batches
    if K < 1 or args.tokens % K:
        raise SystemExit("--micro-batches must divide --tokens")
    if args.sgd_in_backward and K > 1:
        raise SystemExit("--sgd-in-backward updates after every backward: it does not combine with --micro-batches")
    comm = m4t.COMM_WORLD
    P = comm.size
    cuda = args.device == "cuda"
    device = torch.device("cuda", torch.cuda.current_device()) if cuda else torch.device("cpu")
    dtype = torch.bfloat16 if cuda else torch.float32
    capacity = None if args.dropless else args.capacity or 128 // math.gcd(128, P)
    moe = ExpertParallelMLP(args.d_model, args.hidden, args.experts_per_rank, capacity, comm, top_k=args.top_k,
                            dtype=dtype, device=device, seed=3)
    head = (torch.randn(1, args.d_model, generator=torch.Generator().manual_seed(4)) / math.sqrt(args.d_model))
    head = head.to(device).requires_grad_()
    params = list(moe.parameters()) + [head]
    update = {}
    if args.sgd_in_backward:
        update = {"optimizer": InBackwardSGD(args.lr)}
    elif K > 1:
        update = {"accumulator": AccumulatedSGD(args.lr)}
    u = torch.randn(args.d_model, generator=torch.Generator().manual_seed(5)).to(device) / math.sqrt(args.d_model)
    g = torch.Generator().manual_seed(100 + comm.rank)  # every rank sees different data
    for step in range(args.steps):
        x = torch.randn(args.tokens, args.d_model, generator=g).to(device)
        target = torch.tanh(2.0 * (x @ u))[:, None]
        loss = dropped = 0.0
        for xk, tk in zip(x.chunk(K), target.chunk(K)):
            out, routing = moe(xk.to(dtype), **update)
            pred = F.linear(out.float(), replicated_input(head, comm))
            # the objective is the sum of every rank's loss: the mean squared error over the global batch
            part = (pred - tk).square().sum() / (args.tokens * P)
            part.backward()
            loss, dropped = loss + part.detach().double(), dropped + routing.dropped.sum().double()
        if "accumulator" in update:
            update["accumulator"].step()
        with torch.no_grad():
            for p in params:
                if p.grad is not None:  # the experts have none when they are trained in backward
                    p -= args.lr * p.grad.to(p.dtype)
                    p.grad = None
        total = comm.Allreduce(torch.stack([loss, dropped]), m4t.MPI_SUM)
        if comm.rank == 0:
            dropped = float(total[1]) / (args.tokens * args.top_k * P)
            print(f"step {step:3d}  loss {float(total[0]):.5f} dropped {dropped:.3f}", flush=True)


if __name__ == "__main__":
    main()
