"""Expert-parallel token exchange (dispatch / combine) on the single-kernel,
differentiable ``Alltoall`` (the reference would need 4*P blocking MPI
collectives per exchange, ``csrc/extension.cpp:917-987``).

Capacity-based routing: every rank may send at most ``capacity`` tokens to each
destination rank; tokens over capacity are dropped (their combined output is
zero), as in capacity-factor MoE layers.  Both directions are ONE ``Alltoall``
of a ``[P, capacity, d]`` tensor (scatter the destination axis, gather along
the slot axis); the backward pass is the same exchange in the other direction,
produced by autograd.

``dispatch_to_experts`` / ``combine_from_experts`` do the same per expert: ``experts_per_rank`` experts live on
every rank and each has ``capacity`` slots per source rank, so the exchange is ONE ``Alltoall`` of an
``[E, P, capacity, d]`` tensor.  :class:`ExpertParallelMLP` is the mixture-of-experts feed-forward layer built on
them and on :func:`mpi4torch_b200.ops.expert_mlp`, or, dropless (``capacity=None``), on
:func:`mpi4torch_b200.ops.grouped_expert_mlp`.
"""
from __future__ import annotations

import math
from typing import NamedTuple

import torch
import torch.nn.functional as F

import mpi4torch_b200 as m4t
from mpi4torch_b200.ops.expert_mlp import expert_group_starts, expert_mlp, grouped_expert_mlp, grouped_rows

from .tensor_parallel import replicated_input


class DispatchInfo(NamedTuple):
    slot: torch.Tensor      # [T] position of each local token inside its destination bucket (-1 = dropped)
    dest: torch.Tensor      # [T] destination rank of each local token
    capacity: int
    valid: torch.Tensor     # [P, capacity] bool: which received slots hold a real token (per source rank)


def _assign_slots(bucket: torch.Tensor, buckets: int, capacity: int) -> torch.Tensor:
    """Slot of each entry in its bucket: how many earlier entries chose the same bucket (stable order), or -1 when
    ``capacity`` earlier entries already did."""
    onehot = F.one_hot(bucket, buckets)                                  # [T, buckets]
    slot = (onehot.cumsum(0) - onehot).gather(1, bucket[:, None])[:, 0]  # [T]
    return torch.where(slot < capacity, slot, torch.full_like(slot, -1))


def _exchange(buckets: torch.Tensor, comm) -> torch.Tensor:
    """[P(dest), C, ...] on every rank -> [P(source), C, ...]: bucket r of every rank lands on rank r."""
    P, C = buckets.shape[0], buckets.shape[1]
    out = comm.Alltoall(buckets, 1, 0, 1)  # scatter axis 0 (one bucket each), gather the sources along the slot axis
    return out.reshape((P, C) + tuple(buckets.shape[2:]))


def dispatch_tokens(tokens: torch.Tensor, dest_rank: torch.Tensor, capacity: int, comm=None):
    """Send token ``i`` to rank ``dest_rank[i]``.

    Returns ``(received, info)``: ``received[p, s]`` is the ``s``-th token rank ``p`` sent here
    (zeros where ``info.valid[p, s]`` is False).  Differentiable with respect to ``tokens``.
    """
    c = m4t.COMM_WORLD if comm is None else comm
    P = c.size
    T = tokens.shape[0]
    dest = dest_rank.to(torch.int64)
    if T and (int(dest.min()) < 0 or int(dest.max()) >= P):
        raise ValueError("dest_rank entries must be in [0, comm.size)")
    slot = _assign_slots(dest, P, capacity)
    keep = slot >= 0
    flat = dest * capacity + slot.clamp_min(0)
    buckets = torch.zeros((P * capacity,) + tuple(tokens.shape[1:]), dtype=tokens.dtype, device=tokens.device)
    buckets = buckets.index_add(0, flat[keep], tokens[keep])           # differentiable scatter (slots are unique)
    filled = torch.zeros(P * capacity, dtype=torch.int32, device=tokens.device)
    filled[flat[keep]] = 1
    received = _exchange(buckets.reshape((P, capacity) + tuple(tokens.shape[1:])), c)
    valid = _exchange(filled.reshape(P, capacity), c) > 0
    return received, DispatchInfo(slot=slot, dest=dest, capacity=capacity, valid=valid)


def combine_tokens(processed: torch.Tensor, info: DispatchInfo, comm=None) -> torch.Tensor:
    """Inverse exchange: ``processed[p, s]`` (the expert's output for the token it received from
    rank ``p`` in slot ``s``) travels back; returns ``[T, ...]`` aligned with the original tokens
    (zeros for dropped ones)."""
    c = m4t.COMM_WORLD if comm is None else comm
    back = _exchange(processed, c)                                    # [P(dest), C, ...]: my tokens' results
    flat = back.reshape((-1,) + tuple(back.shape[2:]))
    keep = info.slot >= 0
    idx = info.dest * info.capacity + info.slot.clamp_min(0)
    out = flat[idx]
    mask = keep.reshape((-1,) + (1,) * (out.dim() - 1)).to(out.dtype)
    return out * mask


# ---------------------------------------------------------------------------------------------------------------------
# Per-expert exchange and the mixture-of-experts layer
# ---------------------------------------------------------------------------------------------------------------------
class ExpertRouting(NamedTuple):
    expert: torch.Tensor    # [T, k] global expert of each (token, choice) pair, in [0, P * experts_per_rank)
    slot: torch.Tensor      # [T, k] row of the pair among the rows this rank sends to that expert (-1 = dropped)
    experts_per_rank: int
    capacity: int


def _exchange_experts(buf: torch.Tensor, comm) -> torch.Tensor:
    """[E, P(dest), C, ...] on every rank -> [E, P(source), C, ...]: ``out[e, p] = buf_p[e, this rank]``."""
    E, P, C = buf.shape[0], buf.shape[1], buf.shape[2]
    out = comm.Alltoall(buf, 2, 1, 1)  # scatter the destination axis, gather the sources along the slot axis
    return out.reshape((E, P, C) + tuple(buf.shape[3:]))


def _send_rows(routing: ExpertRouting, P: int) -> torch.Tensor:
    """[T, k] row of each pair in the flattened [E, P, C] send buffer (the same row of the returned results)."""
    E, C = routing.experts_per_rank, routing.capacity
    dest, local = routing.expert // E, routing.expert % E
    return (local * P + dest) * C + routing.slot.clamp_min(0)


def dispatch_to_experts(tokens: torch.Tensor, expert: torch.Tensor, experts_per_rank: int, capacity: int, comm=None):
    """Send every (token, choice) pair to global expert ``g = expert[t, j]``, which lives on rank ``g // E`` as its
    local expert ``g % E`` (``E = experts_per_rank``).  ``expert`` is ``[T]`` or ``[T, k]``.

    Each expert takes at most ``capacity`` pairs from each rank, in choice-major order: every token's first choice
    claims a slot before any second choice, and within one choice earlier tokens come first.  Pairs beyond that are
    dropped (``slot == -1``).  Returns ``(received, routing)``: ``received [E, P * capacity, ...]`` holds each local
    expert's rows, contiguous per expert, ordered by source rank and then by slot, with zero rows in empty slots.
    One ``Alltoall``; differentiable with respect to ``tokens``."""
    c = m4t.COMM_WORLD if comm is None else comm
    P, E, C = c.size, int(experts_per_rank), int(capacity)
    choice = expert.to(torch.int64)
    if choice.dim() == 1:
        choice = choice[:, None]
    T, k = choice.shape
    if T and (int(choice.min()) < 0 or int(choice.max()) >= P * E):
        raise ValueError("expert entries must be in [0, comm.size * experts_per_rank)")
    slot = _assign_slots(choice.t().reshape(-1), P * E, C).reshape(k, T).t()
    routing = ExpertRouting(expert=choice, slot=slot, experts_per_rank=E, capacity=C)
    keep = slot >= 0
    token = torch.arange(T, device=tokens.device)[:, None].expand(T, k)
    rest = tuple(tokens.shape[1:])
    send = torch.zeros((E * P * C,) + rest, dtype=tokens.dtype, device=tokens.device)
    send = send.index_add(0, _send_rows(routing, P)[keep], tokens[token[keep]])  # rows are unique
    received = _exchange_experts(send.reshape((E, P, C) + rest), c)
    return received.reshape((E, P * C) + rest), routing


def combine_from_experts(processed: torch.Tensor, routing: ExpertRouting, comm=None) -> torch.Tensor:
    """Inverse of :func:`dispatch_to_experts`: ``processed [E, P * capacity, ...]`` (each local expert's output for
    the rows it received) travels back.  Returns ``[T, k, ...]``, the result of every (token, choice) pair, zero for
    dropped pairs.  One ``Alltoall``; its backward is the dispatch exchange, produced by autograd."""
    c = m4t.COMM_WORLD if comm is None else comm
    P, E, C = c.size, routing.experts_per_rank, routing.capacity
    rest = tuple(processed.shape[2:])
    back = _exchange_experts(processed.reshape((E, P, C) + rest), c)  # [E, P, C, ...]: this rank's pairs' results
    T, k = routing.slot.shape
    out = back.reshape((-1,) + rest)[_send_rows(routing, P).reshape(-1)].reshape((T, k) + rest)
    mask = (routing.slot >= 0).reshape((T, k) + (1,) * len(rest)).to(out.dtype)
    return out * mask


class MoERouting(NamedTuple):
    probs: torch.Tensor     # [T, P * E] router softmax probabilities
    expert: torch.Tensor    # [T, k] chosen global experts, most probable first
    dropped: torch.Tensor   # [T, k] bool: the pair went over its expert's capacity and contributes nothing


class ExpertParallelMLP(torch.nn.Module):
    """Mixture-of-experts feed-forward layer, expert parallel: ``P * experts_per_rank`` experts
    ``gelu_tanh(x W1^T + b1) W2^T + b2`` (``d_model -> hidden -> d_model``), ``experts_per_rank`` of them on each rank.

    ``forward(x [T, d_model])`` returns ``(out [T, d_model], MoERouting)`` with
    ``out[t] = sum over its top_k choices of gate * expert_output``, the gate being the router's softmax probability
    of the chosen expert (so the router gets a gradient) and a dropped pair contributing 0.  The routing record gives
    the probabilities, the chosen experts and the dropped mask, from which a load-balancing loss can be built.

    Parameters:
      * ``router [P * E, d_model]``: replicated, identical on every rank from ``seed``; it runs in torch in fp32 (fp64
        for fp64 layers).  Its gradient is summed over ranks (``replicated_input``): the objective is the sum of all
        ranks' losses, mpi4torch's convention.
      * ``w1 [E, hidden, d_model]``, ``b1 [E, hidden]``, ``w2 [E, d_model, hidden]``, ``b2 [E, d_model]``: this rank's
        experts, rows ``[rank * E, rank * E + E)`` of one seeded global initialisation.  They are owned, not
        replicated: their gradients arrive through the exchange's adjoint and need no collective.  Biases are fp32
        (fp64 for fp64 layers).

    ``capacity``: rows each expert takes from each rank (C).  Every expert then processes ``P * C`` rows, dropped
    slots being zero rows.  The experts run on the batched kernels (:func:`mpi4torch_b200.ops.expert_mlp`) when
    ``expert_mlp_supported`` holds: bf16 CUDA tensors, ``d_model`` and ``hidden`` multiples of 128, and
    ``P * C % 128 == 0``, i.e. ``C % 128 == 0`` at one rank and ``C % 16 == 0`` at eight.  Otherwise the same math
    runs as the torch composition.

    ``capacity=None``: dropless routing.  No pair is dropped and each expert computes exactly the rows routed to it,
    on the grouped kernels (:func:`mpi4torch_b200.ops.grouped_expert_mlp`, when ``grouped_expert_mlp_supported``
    holds: bf16 CUDA tensors, ``d_model`` and ``hidden`` multiples of 128).  At one rank the pairs go straight into
    the grouped layout with no host synchronisation.  At several ranks one ``Alltoall`` exchanges the per-expert
    pair counts and one ``Allreduce(MAX)``, read on the host, sets the exchange's capacity to the largest count; the
    exchange then moves the padded ``[E, P, C, d_model]`` buffer and the received rows are packed into the grouped
    layout.

    ``forward(x, optimizer=None, accumulator=None)`` trains the experts inside backward, in both routing modes and at
    any P (see :func:`mpi4torch_b200.ops.expert_mlp`): with an ``InBackwardSGD`` the expert weights and biases are
    updated by the backward itself (kernel path only), with an ``AccumulatedSGD`` their gradients go into its fp32
    buffers and ``step()`` applies them, with no collective either way.  The experts then get no ``.grad``.  The
    router is tiny, replicated and fp32: it keeps its ``.grad`` in both modes, for the caller's own update."""

    def __init__(self, d_model: int, hidden: int, experts_per_rank: int, capacity, comm=None, top_k: int = 1,
                 dtype=torch.bfloat16, device="cpu", seed: int = 0):
        super().__init__()
        self.comm = m4t.COMM_WORLD if comm is None else comm
        P, r = self.comm.size, self.comm.rank
        if not 1 <= top_k <= P * experts_per_rank:
            raise ValueError("top_k must be in [1, comm.size * experts_per_rank]")
        self.d_model, self.hidden, self.experts_per_rank = d_model, hidden, experts_per_rank
        self.capacity, self.top_k = capacity, top_k
        E, G = experts_per_rank, P * experts_per_rank
        fdt = torch.float64 if dtype == torch.float64 else torch.float32
        gen = torch.Generator().manual_seed(seed)  # identical on every rank, then sliced

        def uniform(shape, fan_in):
            return (torch.rand(shape, generator=gen, dtype=torch.float64) * 2 - 1) / math.sqrt(fan_in)

        router = uniform((G, d_model), d_model)
        w1, b1 = uniform((G, hidden, d_model), d_model), uniform((G, hidden), d_model)
        w2, b2 = uniform((G, d_model, hidden), hidden), uniform((G, d_model), hidden)
        mine = slice(r * E, (r + 1) * E)
        self.router = torch.nn.Parameter(router.to(fdt).to(device))
        self.w1 = torch.nn.Parameter(w1[mine].to(dtype).to(device).contiguous())
        self.b1 = torch.nn.Parameter(b1[mine].to(fdt).to(device).contiguous())
        self.w2 = torch.nn.Parameter(w2[mine].to(dtype).to(device).contiguous())
        self.b2 = torch.nn.Parameter(b2[mine].to(fdt).to(device).contiguous())

    def forward(self, x: torch.Tensor, optimizer=None, accumulator=None):
        c = self.comm
        update = {"optimizer": optimizer, "accumulator": accumulator}
        router = replicated_input(self.router, c)
        probs = torch.softmax(F.linear(x.to(router.dtype), router), dim=-1)  # [T, P * E]
        gate, choice = probs.topk(self.top_k, dim=-1)                          # [T, k]
        if self.capacity is None:
            back = self._dropless(x, choice, update)
            dropped = torch.zeros(choice.shape, dtype=torch.bool, device=choice.device)
        else:
            received, routing = dispatch_to_experts(x, choice, self.experts_per_rank, self.capacity, c)
            y = expert_mlp(received, self.w1, self.b1, self.w2, self.b2, **update)  # [E, P * C, d_model]
            back = combine_from_experts(y, routing, c)                             # [T, k, d_model]
            dropped = routing.slot < 0
        out = (gate.unsqueeze(-1) * back.to(gate.dtype)).sum(1).to(x.dtype)
        return out, MoERouting(probs=probs, expert=choice, dropped=dropped)

    def _experts(self, xg, counts, update):
        return grouped_expert_mlp(xg, counts.to(torch.int32), self.w1, self.b1, self.w2, self.b2, **update)

    def _dropless(self, x: torch.Tensor, choice: torch.Tensor, update) -> torch.Tensor:
        """[T, k, d_model]: every (token, choice) pair's expert output, no pair dropped."""
        c = self.comm
        P, E = c.size, self.experts_per_rank
        T, k = choice.shape
        d = x.shape[1]
        if P == 1:
            # pair i = j * T + t (choice-major, as the slots of dispatch_to_experts) goes to row
            # start[expert] + (pairs before it with the same expert)
            flat = choice.t().reshape(-1)
            onehot = F.one_hot(flat, E)
            rows = expert_group_starts(onehot.sum(0))[flat] + (onehot.cumsum(0) - onehot).gather(1, flat[:, None])[:, 0]
            R = grouped_rows(T * k, E)
            xg = x.new_zeros((R, d)).index_add(0, rows, x.repeat(k, 1))
            y = self._experts(xg, onehot.sum(0), update)
            return y[rows].reshape(k, T, d).transpose(0, 1)
        send = F.one_hot(choice.reshape(-1), P * E).sum(0).to(torch.int32)     # [P * E] pairs for each global expert
        recv = _exchange(send.reshape(P, 1, E), c).reshape(P, E)               # [P(source), E] pairs received
        C = max(int(c.Allreduce(send.max().reshape(1), m4t.MPI_MAX).item()), 1)  # the one host read
        received, routing = dispatch_to_experts(x, choice, E, C, c)            # [E, P * C, d], nothing dropped
        counts = recv.sum(0)                                                   # [E] rows of each local expert
        before = (torch.cumsum(recv, 0) - recv).t()                            # [E, P] rows from earlier sources
        s = torch.arange(C, device=x.device)
        dst = expert_group_starts(counts)[:, None, None] + before[:, :, None] + s  # [E, P, C] row in the grouped layout
        R = grouped_rows(E * P * C, E)
        dst = torch.where(s < recv.t()[:, :, None], dst, R).reshape(-1)       # empty slots -> a scratch row R
        xg = received.new_zeros((R + 1, d)).index_add(0, dst, received.reshape(-1, d))[:R]
        y = self._experts(xg, counts, update)
        processed = torch.cat([y, y.new_zeros((1, d))])[dst].reshape(E, P * C, d)
        return combine_from_experts(processed, routing, c)
