"""FP8 training of the data-parallel linear layer: ``dp_linear_mse(..., fp8=True)`` (DESIGN §4.4).

The recipe, on the kernel path and in the torch composition alike:

* per-tensor current scaling: ``s`` is the largest power of two with ``amax * s <= F`` (F = 448 for E4M3, 57344 for
  E5M2), its exponent clamped to [-126, 126]; ``amax = 0`` gives ``s = 1``; a NaN or Inf in the tensor gives
  ``1/s = NaN``, so every product that reads it is NaN.  ``q = fp8(v * s)`` rounds to nearest even and saturates
  (``cvt.rn.satfinite``); ``v * s`` and the dequantization ``acc * (1/s_a) * (1/s_b)`` are exact.
* ``x`` and the weight average ``W̄`` are E4M3, the output gradient ``dy`` E5M2.
* The scales are device scalars: the host never reads them, so the step has no host synchronisation.

Kernel path (CUDA, bf16, world communicator, B, D and O multiples of 128), one step:

    W̄ = W (one rank) or AllreduceFused(W, SUM, 1/P)
    quantize_fp8(W̄) ; quantize_fp8(x) row-major + transposed
    linear_mse_forward_fp8_local -> dy (bf16), loss, amax(dy)
    quantize_fp8(dy, e5m2) transposed, with that amax
    backward: G = gemm_fp8_tn(dyᵀ, xᵀ) * g, then AllreduceFused(G, 1/P) into .grad, or the in-backward SGD update
    (gemm_fp8_tn_sgd_ at one rank, allreduce_axpy_ of G otherwise); x.grad is the bf16 dgrad of dy and W̄.

Elsewhere the same recipe runs as a torch composition on the torch fp8 dtypes.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

import mpi4torch_b200 as m4t

E4M3, E5M2 = "e4m3", "e5m2"
# format -> (torch dtype, largest finite value F, fe with F = 0.875 * 2^fe)
FORMATS = {E4M3: (torch.float8_e4m3fn, 448.0, 9), E5M2: (torch.float8_e5m2, 57344.0, 16)}


def _ops():
    return torch.ops.mpi4torch_b200


def fp8_scale(amax: torch.Tensor, fmt: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(s, 1/s)`` of the recipe for a one-element amax tensor, as fp32 tensors on its device (no host read)."""
    _, _, fe = FORMATS[fmt]
    a = amax.reshape(1).float()
    m, ex = torch.frexp(a)  # a = m * 2^ex, m in [0.5, 1)
    e = (fe - ex - (m > 0.875).to(ex.dtype)).clamp(-126, 126)
    finite = torch.isfinite(a)
    e = torch.where(finite & (a > 0), e, torch.zeros_like(e)).to(torch.int32)
    s = ((e + 127) << 23).view(torch.float32)
    inv = ((127 - e) << 23).view(torch.float32)
    return s, torch.where(finite, inv, torch.full_like(inv, float("nan")))


def quantize_fp8_reference(x: torch.Tensor, fmt: str, amax: Optional[torch.Tensor] = None):
    """``(q, 1/s)``: the torch form of ``quantize_fp8`` (the operand is taken in fp32)."""
    dtype, fmax, _ = FORMATS[fmt]
    xf = x.float()
    s, inv = fp8_scale(xf.abs().amax() if amax is None else amax, fmt)
    return (xf * s).clamp(-fmax, fmax).to(dtype), inv  # clamp: satfinite (NaN stays NaN)


def dequantize(q: torch.Tensor, scale_inv: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    return q.to(dtype) * scale_inv.to(dtype)


def dp_linear_mse_fp8_supported(x: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, comm) -> bool:
    """Does ``dp_linear_mse(..., fp8=True)`` run on the fp8 kernels for these tensors?"""
    if not (comm.is_world and x.is_cuda and weight.is_cuda and target.is_cuda and x.dim() == 2 and target.dim() == 2
            and weight.dim() == 2 and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16
            and target.dtype == torch.bfloat16 and weight.is_contiguous() and x.stride(1) == 1
            and target.stride(1) == 1 and target.stride(0) % 2 == 0 and target.data_ptr() % 4 == 0):
        return False
    (B, D), O = x.shape, weight.shape[0]
    if not (weight.shape[1] == D and tuple(target.shape) == (B, O) and B % 128 == 0 and D % 128 == 0 and O % 128 == 0
            and B > 0 and D > 0 and O > 0):
        return False
    return m4t.cuda_backend_ready() and hasattr(_ops(), "quantize_fp8")


class _DPLinearMSEFP8(torch.autograd.Function):
    """Local MSE loss of the data-parallel linear layer with fp8 GEMMs (kernel path; see the module docstring).

    Saves the fp8 ``xᵀ`` and ``dyᵀ`` with their scales (not the bf16 ``x``) when the weight needs a gradient, and the
    bf16 ``dy`` and ``W̄`` when ``x`` does: ``x.grad`` is the bf16 dgrad ``g * dy @ W̄``."""

    @staticmethod
    def forward(ctx, x, weight, target, comm_holder, loss_scale, opt):
        comm = comm_holder[0]
        ops = _ops()
        need_gx, need_gw = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if comm.size == 1:
            w_avg = weight.detach()
        else:
            w_avg = comm.AllreduceFused(weight.detach(), m4t.MPI_SUM, 1.0 / comm.size, None)
        wq, _, w_si = ops.quantize_fp8(w_avg, E4M3, True, False)
        xq, xt, x_si = ops.quantize_fp8(x, E4M3, True, need_gw)
        dy, local, dy_amax = ops.linear_mse_forward_fp8_local(xq, wq, x_si, w_si, target, loss_scale, 2.0 * loss_scale)
        dyt = dy_si = None
        if need_gw:
            _, dyt, dy_si = ops.quantize_fp8(dy, E5M2, False, True, dy_amax)
        if need_gx:
            # at one rank w_avg is the weight itself, which an in-backward update may change before this backward
            ctx.save_for_backward(dyt, xt, dy_si, x_si, dy, w_avg.clone() if comm.size == 1 else w_avg)
        else:
            ctx.save_for_backward(dyt, xt, dy_si, x_si, None, None)
        ctx.comm, ctx.opt, ctx.weight = comm, opt, weight
        return local

    @staticmethod
    def backward(ctx, g):
        from mpi4torch_b200.ops.fused_linear import _dgrad  # fused_linear imports this module

        dyt, xt, dy_si, x_si, dy, w_avg = ctx.saved_tensors
        comm, opt, weight = ctx.comm, ctx.opt, ctx.weight
        ops = _ops()
        g = g.reshape(1).to(torch.float32)
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = _dgrad(dy, w_avg) * g.to(dy.dtype)
        if ctx.needs_input_grad[1]:
            if opt is not None:
                opt.updates += 1
                if comm.size == 1:
                    ops.gemm_fp8_tn_sgd_(weight, dyt, xt, dy_si, x_si, -opt.lr, g)
                else:
                    # summed in a fixed rank order: the weights stay bit-identical on every rank
                    ops.allreduce_axpy_(weight, ops.gemm_fp8_tn(dyt, xt, dy_si, x_si, g), -opt.lr / comm.size)
                opt.remember(weight, None)
            else:
                gw = comm.AllreduceFused(ops.gemm_fp8_tn(dyt, xt, dy_si, x_si, g), m4t.MPI_SUM, 1.0 / comm.size, None)
        return gx, gw, None, None, None, None


class _LinearMSEFP8Composition(torch.autograd.Function):
    """The fp8 recipe in torch on an already averaged weight ``w_avg`` (differentiable: its gradient reaches the
    weight through the adjoint of ``AllreduceFused``).  Products are computed in fp32 (fp64 for fp64 inputs) on the
    dequantized operands; ``dy`` is rounded to the input dtype as the kernel rounds it to bf16."""

    @staticmethod
    def forward(ctx, x, w_avg, target, loss_scale):
        acc = torch.float64 if x.dtype == torch.float64 else torch.float32
        xq, x_si = quantize_fp8_reference(x, E4M3)
        wq, w_si = quantize_fp8_reference(w_avg, E4M3)
        xd = dequantize(xq, x_si, acc)
        d = xd @ dequantize(wq, w_si, acc).t() - target.to(acc)
        dy = (d * (2.0 * loss_scale)).to(x.dtype)
        ctx.save_for_backward(dy, xd, w_avg)
        return (d.square().sum() * loss_scale).reshape(1)

    @staticmethod
    def backward(ctx, g):
        dy, xd, w_avg = ctx.saved_tensors
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = (dy @ w_avg.to(dy.dtype)) * g.reshape(1).to(dy.dtype)
        if ctx.needs_input_grad[1]:
            dyq, dy_si = quantize_fp8_reference(dy, E5M2)
            gw = ((dequantize(dyq, dy_si, xd.dtype).t() @ xd) * g.reshape(1).to(xd.dtype)).to(w_avg.dtype)
        return gx, gw, None, None


def dp_linear_mse_fp8(x: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, comm, loss_scale: float,
                      optimizer=None) -> torch.Tensor:
    """``dp_linear_mse(..., fp8=True)``: the fp8 kernels where they apply, the torch composition elsewhere."""
    if dp_linear_mse_fp8_supported(x, weight, target, comm):
        return _DPLinearMSEFP8.apply(x, weight, target, [comm], float(loss_scale), optimizer)
    if optimizer is not None:
        raise RuntimeError("mpi4torch_b200: InBackwardSGD is only available on the fused CUDA path")
    w_avg = comm.AllreduceFused(weight, m4t.MPI_SUM, 1.0 / comm.size, None)
    return _LinearMSEFP8Composition.apply(x, w_avg, target, float(loss_scale))
