"""The experts of a mixture-of-experts feed-forward block as one autograd node on batched wgmma kernels.

``expert_mlp(x, w1, b1, w2, b2)``  for every expert e:  y_e = gelu_tanh(x_e W1_e^T + b1_e) W2_e^T + b2_e

All E experts have the same shapes and are stacked along dim 0: x [E, M, D], w1 [E, H, D], w2 [E, O, H] (bf16),
b1 [E, H], b2 [E, O] (fp32).  Every expert gets the same number of rows M, which is what capacity-based routing
produces.  Forward is two launches whatever E is (csrc/kernels/gemm_wgmma.cu, batched instantiations): bias + GELU
storing z and h, then bias.  Backward is the batched GELU-backward GEMM (dz with its column-sum partials), the two
batched weight-gradient GEMMs, the batched NN GEMM for dx and the batched column sum for db1; db2 is a torch sum.

Elsewhere (CPU tensors, other dtypes, shapes the kernels reject) the same math runs as the composition
``baddbmm -> F.gelu(tanh) -> baddbmm`` in fp32 (fp64 for fp64 inputs).

``grouped_expert_mlp(x, counts, w1, b1, w2, b2)`` is the dropless form: expert e takes exactly ``counts[e]`` rows of
one ``[R, D]`` tensor in the grouped layout of :func:`expert_group_starts`, and the counts stay on the device.

Both take ``optimizer=InBackwardSGD(lr)`` or ``accumulator=AccumulatedSGD(lr)`` to train the expert parameters inside
backward instead of giving them a ``.grad``.  Expert parameters are owned by their rank, not replicated, so neither
mode issues a collective:

* ``optimizer``: each weight wgrad is its SGD step, ``W <- bf16(W - lr * G)`` in the kernel's epilogue
  (``batched_wgrad_sgd_`` / ``grouped_wgrad_sgd_``), and each bias gets ``b -= lr * db`` in fp32.  Backward reads w2
  (for dz) before updating it and w1 (for dx) before updating it, so ``x.grad`` is the plain mode's.
* ``accumulator``: each weight wgrad adds its gradient into the accumulator's fp32 buffer in the kernel's epilogue
  (``batched_wgrad_accumulate_`` / ``grouped_wgrad_accumulate_``), each bias gradient is added to its buffer, and
  ``accumulator.step()`` applies ``p -= lr * buf``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

import mpi4torch_b200 as m4t

from .fused_linear import AccumulatedSGD, InBackwardSGD, _ops, owned_accumulated


def _check_shapes(x, w1, b1, w2, b2) -> None:
    if not (x.dim() == 3 and w1.dim() == 3 and w2.dim() == 3 and b1.dim() == 2 and b2.dim() == 2):
        raise ValueError("mpi4torch_b200: expert_mlp needs x [E, M, D], w1 [E, H, D], b1 [E, H], w2 [E, O, H], "
                         "b2 [E, O]")
    E, _, D = x.shape
    H, O = w1.shape[1], w2.shape[1]
    want = {"w1": (E, H, D), "b1": (E, H), "w2": (E, O, H), "b2": (E, O)}
    for name, t in (("w1", w1), ("b1", b1), ("w2", w2), ("b2", b2)):
        if tuple(t.shape) != want[name]:
            raise ValueError(f"mpi4torch_b200: expert_mlp: {name} has shape {tuple(t.shape)}, expected {want[name]} "
                             f"for x of shape {tuple(x.shape)}")


def expert_mlp_supported(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor,
                         b2: torch.Tensor) -> bool:
    """Does :func:`expert_mlp` run on the library's kernels for these tensors?  All five on one CUDA device and
    contiguous, bf16 x / w1 / w2 and fp32 b1 / b2, M, D, H and O multiples of 128, and aligned bases (see
    ``batched_gemm_tn_supported``)."""
    if not (m4t.cuda_backend_ready() and hasattr(_ops(), "batched_linear_bias_gelu_forward")):
        return False
    try:
        _check_shapes(x, w1, b1, w2, b2)
    except ValueError:
        return False
    if not all(t.is_cuda and t.device == x.device for t in (w1, b1, w2, b2)):
        return False
    ops = _ops()
    E, M, _ = x.shape
    # h is allocated by the first GEMM: only its shape matters for the second
    return bool(ops.batched_gemm_tn_supported(x, w1, b1)
                and ops.batched_gemm_tn_supported(x.new_empty((E, M, w1.shape[1])), w2, b2))


def _kernel_grad(dy: torch.Tensor) -> torch.Tensor:
    """The upstream gradient as the backward kernels read it: contiguous, with a 16-byte-aligned base.  The forward
    never sees it, so it may be e.g. the expanded gradient of a sum, or a slice of a larger buffer at an odd offset,
    which ``.contiguous()`` returns unchanged."""
    dy = dy.contiguous()
    return dy if dy.data_ptr() % 16 == 0 else dy.clone()


def _check_update(name, optimizer, accumulator) -> None:
    if optimizer is not None and accumulator is not None:
        raise ValueError(f"mpi4torch_b200: {name} takes either optimizer= or accumulator=, not both")


def _save_update(ctx, optimizer, accumulator) -> None:
    """Keep the update mode and the counts that tell backward whether its saved weights are still current."""
    ctx.opt, ctx.acc = optimizer, accumulator
    ctx.updates = optimizer.updates if optimizer is not None else accumulator.updates if accumulator is not None else 0


def _begin_backward(ctx, need) -> None:
    """Raise when the weights this node saved were updated since its forward.  Runs before the saved tensors are read:
    ``step()`` changes the parameters in place."""
    if ctx.acc is not None:
        ctx.acc.check_fresh(ctx.updates)
    if ctx.opt is not None:
        if ctx.opt.updates != ctx.updates:
            raise RuntimeError("mpi4torch_b200: the expert weights were updated in place by another backward since this "
                               "node's forward, so its saved weights are stale; with InBackwardSGD, run one backward "
                               "per forward")
        if any(need):
            ctx.opt.updates += 1


def _weight_grad(ctx, kind, w, dy, a, *counts):
    """The gradient of the expert weights ``w`` from ``dy`` and ``a`` (``kind``: ``batched`` or ``grouped``): returned
    in plain mode, applied as the SGD step with an optimizer, added into the fp32 buffer with an accumulator."""
    ops = _ops()
    if ctx.opt is not None:
        getattr(ops, f"{kind}_wgrad_sgd_")(w, dy, a, *counts, -ctx.opt.lr)
        return None
    if ctx.acc is not None:
        getattr(ops, f"{kind}_wgrad_accumulate_")(ctx.acc.buffer(w, None), dy, a, *counts)
        return None
    return getattr(ops, f"{kind}_wgrad_bf16")(dy, a, *counts)


def _bias_grad(ctx, b, db):
    """As :func:`_weight_grad` for a bias and its fp32 gradient ``db``."""
    if ctx.opt is not None:
        b.add_(db, alpha=-ctx.opt.lr)
        return None
    if ctx.acc is not None:
        ctx.acc.buffer(b, None).add_(db)
        return None
    return db


class _ExpertMLP(torch.autograd.Function):
    """Kernel path of :func:`expert_mlp`.  Backward takes the bf16 upstream gradient dy and fills plain gradients (or
    updates the parameters, see the module docstring); an input that needs no gradient gets none, and no launch is
    spent on it."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, optimizer, accumulator):
        ops = _ops()
        h, z = ops.batched_linear_bias_gelu_forward(x, w1, b1)
        ctx.save_for_backward(x, w1, w2, h, z)
        ctx.biases = (b1, b2)
        _save_update(ctx, optimizer, accumulator)
        return ops.batched_linear_bias_forward(h, w2, b2)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        need = ctx.needs_input_grad
        _begin_backward(ctx, need[1:5])
        x, w1, w2, h, z = ctx.saved_tensors
        b1, b2 = ctx.biases
        ops = _ops()
        dy = _kernel_grad(dy)
        gx = gw1 = gb1 = gw2 = gb2 = None
        # every read of a weight comes before its update: dz reads w2, dx reads w1
        if need[0] or need[1] or need[2]:
            dz, dz_part = ops.batched_gemm_nn_gelu_backward(dy, w2, z)
        if need[3]:
            gw2 = _weight_grad(ctx, "batched", w2, dy, h)
        if need[0]:
            gx = ops.batched_gemm_nn(dz, w1)
        if need[1]:
            gw1 = _weight_grad(ctx, "batched", w1, dz, x)
        if need[2]:
            gb1 = _bias_grad(ctx, b1, ops.batched_column_sum(dz_part))
        if need[4]:
            gb2 = _bias_grad(ctx, b2, dy.sum(1, dtype=torch.float32))
        return gx, gw1, gb1, gw2, gb2, None, None


def _composition(x, w1, b1, w2, b2):
    acc = torch.float64 if x.dtype == torch.float64 else torch.float32
    z = torch.baddbmm(b1.to(acc).unsqueeze(1), x.to(acc), w1.to(acc).transpose(1, 2))
    h = F.gelu(z, approximate="tanh")
    return torch.baddbmm(b2.to(acc).unsqueeze(1), h, w2.to(acc).transpose(1, 2)).to(x.dtype)


def _owned(optimizer, accumulator, params, name):
    """The parameters as the composition path reads them in the update modes."""
    if optimizer is not None:
        raise RuntimeError(f"mpi4torch_b200: InBackwardSGD for {name} is only available on the CUDA kernel path")
    if accumulator is None:
        return params
    return [owned_accumulated(accumulator, p) for p in params]


def expert_mlp(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor, *,
               optimizer: Optional[InBackwardSGD] = None,
               accumulator: Optional[AccumulatedSGD] = None) -> torch.Tensor:
    """``y [E, M, O]`` with ``y_e = gelu_tanh(x_e W1_e^T + b1_e) W2_e^T + b2_e`` for each of the E stacked experts.

    On the kernel path (:func:`expert_mlp_supported`) ``z`` and ``h`` are stored as bf16 between the two GEMMs and
    ``y`` is bf16; forward is two launches and backward at most five, whatever E is.  Otherwise the composition
    ``baddbmm -> F.gelu(approximate="tanh") -> baddbmm`` runs in fp32 (fp64 for fp64 inputs) and ``y`` has x's
    dtype.

    ``optimizer``: an :class:`InBackwardSGD`; backward applies ``p -= lr * grad`` to the four parameters that require
    a gradient (the weights in their wgrad kernels) and gives them no ``.grad``.  Only ``lr`` is used.  Kernel path
    only (``RuntimeError`` elsewhere); run one backward per forward, as a node whose weights another backward updated
    since its forward raises ``RuntimeError``.
    ``accumulator``: an :class:`AccumulatedSGD`; backward adds the gradients into its buffers of the parameters, which
    it holds as owned (no collective), on any path.  Not combinable with ``optimizer`` (``ValueError``)."""
    _check_shapes(x, w1, b1, w2, b2)
    _check_update("expert_mlp", optimizer, accumulator)
    if expert_mlp_supported(x, w1, b1, w2, b2):
        return _ExpertMLP.apply(x, w1, b1, w2, b2, optimizer, accumulator)
    return _composition(x, *_owned(optimizer, accumulator, (w1, b1, w2, b2), "expert_mlp"))


# ---------------------------------------------------------------------------------------------------------------------
# Grouped (dropless) experts
# ---------------------------------------------------------------------------------------------------------------------
GROUP_ROWS = 128  # a group's rows start on a multiple of this: no 128-row GEMM tile spans two experts


def expert_group_starts(counts: torch.Tensor) -> torch.Tensor:
    """First row of each expert in the grouped layout: ``start[e] = 128 * sum_{j<e} ceil(counts[j] / 128)``, negative
    counts counting as 0.  ``counts [E]`` is any integer tensor; the result is int64 on its device, computed without
    a host synchronisation.  A tensor of ``128 * (ceil(N / 128) + E)`` rows holds any ``N`` routed rows."""
    blocks = (counts.to(torch.int64).clamp_min(0) + GROUP_ROWS - 1) // GROUP_ROWS
    return GROUP_ROWS * (torch.cumsum(blocks, 0) - blocks)


def grouped_rows(pairs: int, experts: int) -> int:
    """Rows of a grouped tensor that holds any ``pairs`` rows routed to ``experts`` experts."""
    return GROUP_ROWS * (-(-pairs // GROUP_ROWS) + experts)


def _check_grouped(x, counts, w1, b1, w2, b2) -> None:
    if not (x.dim() == 2 and counts.dim() == 1 and w1.dim() == 3 and w2.dim() == 3 and b1.dim() == 2 and b2.dim() == 2):
        raise ValueError("mpi4torch_b200: grouped_expert_mlp needs x [R, D], counts [E], w1 [E, H, D], b1 [E, H], "
                         "w2 [E, O, H], b2 [E, O]")
    if counts.dtype.is_floating_point or counts.dtype == torch.bool:
        raise ValueError("mpi4torch_b200: grouped_expert_mlp: counts must be an integer tensor")
    E, D = counts.shape[0], x.shape[1]
    H, O = w1.shape[1], w2.shape[1]
    want = {"w1": (E, H, D), "b1": (E, H), "w2": (E, O, H), "b2": (E, O)}
    for name, t in (("w1", w1), ("b1", b1), ("w2", w2), ("b2", b2)):
        if tuple(t.shape) != want[name]:
            raise ValueError(f"mpi4torch_b200: grouped_expert_mlp: {name} has shape {tuple(t.shape)}, expected "
                             f"{want[name]} for x of shape {tuple(x.shape)} and {E} experts")


def grouped_expert_mlp_supported(x: torch.Tensor, counts: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor,
                                 w2: torch.Tensor, b2: torch.Tensor) -> bool:
    """Does :func:`grouped_expert_mlp` run on the library's kernels for these tensors?  All six on one CUDA device and
    contiguous, bf16 x / w1 / w2, fp32 b1 / b2, int32 counts, 1 <= E <= 1024, R, D, H and O multiples of 128, and
    aligned bases (see ``grouped_gemm_tn_supported``)."""
    if not (m4t.cuda_backend_ready() and hasattr(_ops(), "grouped_linear_bias_gelu_forward")):
        return False
    try:
        _check_grouped(x, counts, w1, b1, w2, b2)
    except ValueError:
        return False
    if not all(t.is_cuda and t.device == x.device for t in (counts, w1, b1, w2, b2)):
        return False
    ops = _ops()
    # h is allocated by the first GEMM: only its shape matters for the second
    return bool(ops.grouped_gemm_tn_supported(x, w1, counts, b1)
                and ops.grouped_gemm_tn_supported(x.new_empty((x.shape[0], w1.shape[1])), w2, counts, b2))


class _GroupedExpertMLP(torch.autograd.Function):
    """Kernel path of :func:`grouped_expert_mlp`.  No host synchronisation: the counts are only read by the kernels.
    Backward takes the bf16 upstream gradient and launches at most six kernels, none for an input that needs no
    gradient."""

    @staticmethod
    def forward(ctx, x, counts, w1, b1, w2, b2, optimizer, accumulator):
        ops = _ops()
        h, z = ops.grouped_linear_bias_gelu_forward(x, w1, b1, counts)
        ctx.save_for_backward(x, counts, w1, w2, h, z)
        ctx.mark_non_differentiable(counts)
        ctx.biases = (b1, b2)
        _save_update(ctx, optimizer, accumulator)
        return ops.grouped_linear_bias_forward(h, w2, b2, counts)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        need = ctx.needs_input_grad
        _begin_backward(ctx, need[2:6])
        x, counts, w1, w2, h, z = ctx.saved_tensors
        b1, b2 = ctx.biases
        ops = _ops()
        dy = _kernel_grad(dy)
        gx = gw1 = gb1 = gw2 = gb2 = None
        # every read of a weight comes before its update: dz reads w2, dx reads w1
        if need[0] or need[2] or need[3]:
            dz, dz_part = ops.grouped_gemm_nn_gelu_backward(dy, w2, z, counts)
        if need[4]:
            gw2 = _weight_grad(ctx, "grouped", w2, dy, h, counts)
        if need[0]:
            gx = ops.grouped_gemm_nn(dz, w1, counts)
        if need[2]:
            gw1 = _weight_grad(ctx, "grouped", w1, dz, x, counts)
        if need[3]:
            gb1 = _bias_grad(ctx, b1, ops.grouped_column_sum(dz_part, counts))
        if need[5]:
            gb2 = _bias_grad(ctx, b2, ops.grouped_column_sum(dy, counts))
        return gx, None, gw1, gb1, gw2, gb2, None, None


def _grouped_composition(x, counts, w1, b1, w2, b2):
    """Per-expert loop on the grouped layout in fp32 (fp64 for fp64 inputs); reads the counts on the host."""
    acc = torch.float64 if x.dtype == torch.float64 else torch.float32
    R = x.shape[0]
    starts = expert_group_starts(counts).tolist()
    y = x.new_zeros((R, w2.shape[1]), dtype=acc)
    for e, (s, c) in enumerate(zip(starts, counts.tolist())):
        # an empty group still takes part (with no rows), so that y depends on x and the weights on every rank: the
        # backward of a collective upstream of x then runs on every rank, in the same order
        s = min(s, R)
        rows = min(s + max(int(c), 0), R) - s
        h = F.gelu(torch.addmm(b1[e].to(acc), x[s:s + rows].to(acc), w1[e].to(acc).t()), approximate="tanh")
        y = y.index_copy(0, torch.arange(s, s + rows, device=x.device),
                         torch.addmm(b2[e].to(acc), h, w2[e].to(acc).t()))
    return y.to(x.dtype)


def grouped_expert_mlp(x: torch.Tensor, counts: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor,
                       b2: torch.Tensor, *, optimizer: Optional[InBackwardSGD] = None,
                       accumulator: Optional[AccumulatedSGD] = None) -> torch.Tensor:
    """Dropless experts: ``y [R, O]`` with ``y[rows of e] = gelu_tanh(x[rows of e] W1_e^T + b1_e) W2_e^T + b2_e``.

    Expert e's rows are ``[start[e], start[e] + counts[e])`` of ``x [R, D]``, ``start`` as :func:`expert_group_starts`
    gives it; every other row of ``y`` is zero and gets no gradient into the weights, whatever ``x`` holds there.
    Rows that would lie past ``R`` do not exist.  ``counts`` is not differentiable.

    On the kernel path (:func:`grouped_expert_mlp_supported`) forward is two launches and backward at most six,
    whatever E and the counts are, with no host synchronisation.  Otherwise a per-expert ``addmm -> F.gelu -> addmm``
    loop runs in fp32 (fp64 for fp64 inputs), reading the counts on the host, and ``y`` has x's dtype.

    ``optimizer`` and ``accumulator`` as in :func:`expert_mlp`.  An expert with no rows has a zero gradient: the SGD
    step and the accumulation leave its weights and buffers exactly as they were."""
    _check_grouped(x, counts, w1, b1, w2, b2)
    _check_update("grouped_expert_mlp", optimizer, accumulator)
    if grouped_expert_mlp_supported(x, counts, w1, b1, w2, b2):
        return _GroupedExpertMLP.apply(x, counts, w1, b1, w2, b2, optimizer, accumulator)
    return _grouped_composition(x, counts, *_owned(optimizer, accumulator, (w1, b1, w2, b2), "grouped_expert_mlp"))
