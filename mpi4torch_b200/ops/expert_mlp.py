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
"""
from __future__ import annotations

import torch
import torch.nn.functional as F
from torch.autograd.function import once_differentiable

import mpi4torch_b200 as m4t

from .fused_linear import _ops


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


class _ExpertMLP(torch.autograd.Function):
    """Kernel path of :func:`expert_mlp`.  Backward takes the bf16 upstream gradient dy and fills plain gradients;
    an input that needs no gradient gets none, and no launch is spent on it."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        ops = _ops()
        h, z = ops.batched_linear_bias_gelu_forward(x, w1, b1)
        ctx.save_for_backward(x, w1, w2, h, z)
        return ops.batched_linear_bias_forward(h, w2, b2)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, w1, w2, h, z = ctx.saved_tensors
        ops = _ops()
        need = ctx.needs_input_grad
        dy = _kernel_grad(dy)
        gx = gw1 = gb1 = gw2 = gb2 = None
        if need[0] or need[1] or need[2]:
            dz, dz_part = ops.batched_gemm_nn_gelu_backward(dy, w2, z)
        if need[3]:
            gw2 = ops.batched_wgrad_bf16(dy, h)
        if need[0]:
            gx = ops.batched_gemm_nn(dz, w1)
        if need[1]:
            gw1 = ops.batched_wgrad_bf16(dz, x)
        if need[2]:
            gb1 = ops.batched_column_sum(dz_part)
        if need[4]:
            gb2 = dy.sum(1, dtype=torch.float32)
        return gx, gw1, gb1, gw2, gb2


def _composition(x, w1, b1, w2, b2):
    acc = torch.float64 if x.dtype == torch.float64 else torch.float32
    z = torch.baddbmm(b1.to(acc).unsqueeze(1), x.to(acc), w1.to(acc).transpose(1, 2))
    h = F.gelu(z, approximate="tanh")
    return torch.baddbmm(b2.to(acc).unsqueeze(1), h, w2.to(acc).transpose(1, 2)).to(x.dtype)


def expert_mlp(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor) -> torch.Tensor:
    """``y [E, M, O]`` with ``y_e = gelu_tanh(x_e W1_e^T + b1_e) W2_e^T + b2_e`` for each of the E stacked experts.

    On the kernel path (:func:`expert_mlp_supported`) ``z`` and ``h`` are stored as bf16 between the two GEMMs and
    ``y`` is bf16; forward is two launches and backward at most five, whatever E is.  Otherwise the composition
    ``baddbmm -> F.gelu(approximate="tanh") -> baddbmm`` runs in fp32 (fp64 for fp64 inputs) and ``y`` has x's
    dtype."""
    _check_shapes(x, w1, b1, w2, b2)
    if expert_mlp_supported(x, w1, b1, w2, b2):
        return _ExpertMLP.apply(x, w1, b1, w2, b2)
    return _composition(x, w1, b1, w2, b2)


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
    def forward(ctx, x, counts, w1, b1, w2, b2):
        ops = _ops()
        h, z = ops.grouped_linear_bias_gelu_forward(x, w1, b1, counts)
        ctx.save_for_backward(x, counts, w1, w2, h, z)
        ctx.mark_non_differentiable(counts)
        return ops.grouped_linear_bias_forward(h, w2, b2, counts)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, counts, w1, w2, h, z = ctx.saved_tensors
        ops = _ops()
        need = ctx.needs_input_grad
        dy = _kernel_grad(dy)
        gx = gw1 = gb1 = gw2 = gb2 = None
        if need[0] or need[2] or need[3]:
            dz, dz_part = ops.grouped_gemm_nn_gelu_backward(dy, w2, z, counts)
        if need[4]:
            gw2 = ops.grouped_wgrad_bf16(dy, h, counts)
        if need[0]:
            gx = ops.grouped_gemm_nn(dz, w1, counts)
        if need[2]:
            gw1 = ops.grouped_wgrad_bf16(dz, x, counts)
        if need[3]:
            gb1 = ops.grouped_column_sum(dz_part, counts)
        if need[5]:
            gb2 = ops.grouped_column_sum(dy, counts)
        return gx, None, gw1, gb1, gw2, gb2


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
                       b2: torch.Tensor) -> torch.Tensor:
    """Dropless experts: ``y [R, O]`` with ``y[rows of e] = gelu_tanh(x[rows of e] W1_e^T + b1_e) W2_e^T + b2_e``.

    Expert e's rows are ``[start[e], start[e] + counts[e])`` of ``x [R, D]``, ``start`` as :func:`expert_group_starts`
    gives it; every other row of ``y`` is zero and gets no gradient into the weights, whatever ``x`` holds there.
    Rows that would lie past ``R`` do not exist.  ``counts`` is not differentiable.

    On the kernel path (:func:`grouped_expert_mlp_supported`) forward is two launches and backward at most six,
    whatever E and the counts are, with no host synchronisation.  Otherwise a per-expert ``addmm -> F.gelu -> addmm``
    loop runs in fp32 (fp64 for fp64 inputs), reading the counts on the host, and ``y`` has x's dtype."""
    _check_grouped(x, counts, w1, b1, w2, b2)
    if grouped_expert_mlp_supported(x, counts, w1, b1, w2, b2):
        return _GroupedExpertMLP.apply(x, counts, w1, b1, w2, b2)
    return _grouped_composition(x, counts, w1, b1, w2, b2)
