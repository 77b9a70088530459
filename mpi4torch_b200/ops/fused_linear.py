"""Data-parallel linear layer as autograd nodes backed by the fused wgmma kernels.

``allreduce_linear(x, W)``         y = x @ mean_ranks(W)^T
``dp_linear_mse(x, W, t, ...)``    loss_local = loss_scale * sum((x @ mean_ranks(W)^T - t)^2)

Both are ``torch.autograd.Function`` nodes (the reference builds its nodes the same way,
csrc/extension.cpp:254-308: forward communicates, backward runs the adjoint communication):

* forward  = ONE kernel: the parameter Allreduce (x 1/size) fused into the GEMM operand path
  (csrc/kernels/gemm_wgmma.cu, ``FUSED``), for ``dp_linear_mse`` with the loss and dL/dy
  produced by the GEMM epilogue;
* backward = the weight-gradient GEMM (csrc/kernels/wgrad_wgmma.cu, MN-major wgmma operands) and
  the adjoint Allreduce of the gradient.  With an :class:`InBackwardSGD` attached, backward is ONE
  kernel: wgrad GEMM -> reduce-scatter through the NVSwitch -> ``W += -lr/size * sum`` -> multicast of
  the new weights (-> Allreduce of the new weights for the next forward), i.e. the optimizer step runs
  inside ``loss.backward()`` and the weight receives no ``.grad``.  With an :class:`AccumulatedSGD`
  attached, backward adds this rank's gradient into an fp32 buffer (the wgrad kernel's accumulating
  epilogue) and issues no collective; ``step()`` all-reduces the buffers and updates once.

Elsewhere (CPU tensors, other dtypes/shapes, communicators created by ``Split``) the same math runs
as the composition ``F.linear(x, AllreduceFused(W, SUM, 1/size))``.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

import mpi4torch_b200 as m4t
from mpi4torch_b200.ops.fp8 import dp_linear_mse_fp8


def has_fused_kernel() -> bool:
    return hasattr(torch.ops.mpi4torch_b200, "allreduce_linear_fused")


def _ops():
    return torch.ops.mpi4torch_b200


class InBackwardSGD:
    """Plain SGD applied inside the backward kernel of :func:`dp_linear_mse` (optimizer-in-backward).

    Also owns the prefetched parameter average: after the fused update every rank's backward
    kernel has already all-reduced the NEW weights (x 1/size) into a symmetric buffer, so the next
    forward is a plain local GEMM.  The prefetch is dropped whenever the weight's version counter
    shows a modification the kernel did not make.

    ``updates`` counts the in-place weight updates applied through this optimizer.  The kernels write
    the weight through its data pointer, which torch's version counter does not see, so a node that
    saved the weight (or its prefetched average) for backward compares this count instead.
    """

    def __init__(self, lr: float, prefetch: bool = True, assume_replicated: bool = False):
        self.lr = float(lr)
        self.prefetch = bool(prefetch)
        # Opt-in shortcut, NOT the default: the fused update writes bit-identical weights on every rank (one owner
        # computes a tile and stores the same bits everywhere), so Allreduce(W)/size == W and the next forward
        # could skip the parameter collective altogether.  The default keeps the real all-reduce of the new
        # weights (prefetched inside the backward kernel).
        self.assume_replicated = bool(assume_replicated)
        self._wavg: Optional[torch.Tensor] = None
        self._weight_id = None
        self._version = -1
        self.updates = 0

    def take_prefetched(self, weight: torch.Tensor) -> Optional[torch.Tensor]:
        w_avg, self._wavg = self._wavg, None
        if w_avg is None or self._weight_id != id(weight) or self._version != weight._version:
            return None
        return w_avg

    def remember(self, weight: torch.Tensor, w_avg: Optional[torch.Tensor]) -> None:
        self._wavg = w_avg
        self._weight_id = id(weight)
        self._version = weight._version

    def invalidate(self) -> None:
        self._wavg = None


class AccumulatedSGD:
    """Plain SGD over gradients accumulated across micro-batches (gradient accumulation).

    The nodes (``dp_linear_mse``, ``dp_mlp_mse``, ``dp_mlp_cross_entropy``) take it as ``accumulator=``.  Their
    backward adds THIS rank's gradient of its local loss into a per-parameter buffer and issues no collective: on the
    kernel path ``wgrad_accumulate_`` (the wgrad GEMM with an fp32 read-modify-write epilogue) for the weights and
    ``buf += column_sum(...)`` for the biases; elsewhere a small autograd node adds the gradient of the parameter
    average.  The parameters get no ``.grad``, and a parameter with ``requires_grad=False`` gets no buffer.

    A buffer is fp32 for a 16-bit parameter and has the parameter's dtype otherwise.  It is allocated at the first
    backward that reaches its parameter and zeroed by :meth:`step`, which applies, per buffered parameter,
    ``p += AllreduceFused(buf, SUM, -lr / P)``: one parameter-sized collective per parameter and step, summed in a
    fixed order, so every rank ends with the same bits.

    Owned parameters (the experts of ``expert_mlp`` / ``grouped_expert_mlp``, which live on one rank only) register
    with ``buffer(param, None)``: :meth:`step` applies ``p -= lr * buf`` to them locally, with no collective.  One
    accumulator can hold replicated and owned parameters together.

    The parameter averages ``mean_ranks(p)`` that the forwards read are computed once per step (by the first
    forward) and reused by the later forwards of the same step.  ``updates`` counts the calls of :meth:`step`; a
    backward whose forward came before the last :meth:`step` raises ``RuntimeError``.  Several forwards before one
    backward (``(loss(xa) + loss(xb)).backward()``) are allowed and give the buffers of separate backwards.
    """

    def __init__(self, lr: float):
        self.lr = float(lr)
        self.updates = 0
        self._bufs = {}  # id(param) -> (param, buffer, comm)
        self._avgs = {}  # id(param) -> (param, version, average)

    def buffer(self, param: torch.Tensor, comm) -> torch.Tensor:
        """The gradient buffer of ``param`` (allocated zeroed at the first call).  ``comm`` is the communicator over
        which ``param`` is replicated, or ``None`` for a parameter this rank owns alone."""
        entry = self._bufs.get(id(param))
        if entry is None or entry[0] is not param:
            dtype = torch.float32 if param.dtype in (torch.bfloat16, torch.float16) else param.dtype
            entry = (param, torch.zeros(param.shape, dtype=dtype, device=param.device), comm)
            self._bufs[id(param)] = entry
        return entry[1]

    def buffers(self):
        """``(param, buffer)`` of every parameter that has a buffer."""
        return [(p, b) for p, b, _ in self._bufs.values()]

    def average(self, comm, param: torch.Tensor, compute=None) -> torch.Tensor:
        """``mean_ranks(param)`` (detached) for this step: computed by ``compute()`` (default ``AllreduceFused``;
        the parameter itself at one rank) at the first call after a :meth:`step`, reused until the next one or
        until the parameter's version counter shows an in-place change."""
        hit = self.cached_average(param)
        if hit is not None:
            return hit
        if compute is not None:
            avg = compute()
        elif comm.size == 1:
            avg = param.detach()
        else:
            avg = comm.AllreduceFused(param.detach(), m4t.MPI_SUM, 1.0 / comm.size, None)
        self.keep_average(param, avg)
        return self._avgs[id(param)][2]

    def cached_average(self, param: torch.Tensor) -> Optional[torch.Tensor]:
        entry = self._avgs.get(id(param))
        if entry is None or entry[0] is not param or entry[1] != param._version:
            return None
        return entry[2]

    def keep_average(self, param: torch.Tensor, avg: torch.Tensor) -> None:
        """Keep ``avg`` as this step's average of ``param``; it must be a tensor no later call overwrites."""
        self._avgs[id(param)] = (param, param._version, avg.detach())

    def check_fresh(self, updates_at_forward: int) -> None:
        if self.updates != updates_at_forward:
            raise RuntimeError("mpi4torch_b200: AccumulatedSGD.step() ran between this node's forward and its "
                               "backward, so its saved parameter averages are stale; run the backward of every "
                               "forward before step()")

    @torch.no_grad()
    def step(self) -> None:
        """One SGD update per buffered parameter from the sum of every rank's buffer (an owned parameter: from its
        own buffer); zeroes the buffers."""
        for p, buf, comm in self._bufs.values():
            if comm is None:
                p.add_(buf, alpha=-self.lr)
            else:
                p.add_(comm.AllreduceFused(buf, m4t.MPI_SUM, -self.lr / comm.size, None))
            buf.zero_()
        self.updates += 1
        self._avgs.clear()


class _AccumulateGrad(torch.autograd.Function):
    """Identity on the detached parameter average ``avg``; backward adds the incoming gradient into the accumulator's
    buffer of ``param`` (no collective) and gives ``param`` no gradient.  The composition paths' accumulation."""

    @staticmethod
    def forward(ctx, param, avg, acc, comm):
        ctx.acc, ctx.comm, ctx.param, ctx.updates = acc, comm, param, acc.updates
        return avg.view_as(avg)

    @staticmethod
    def backward(ctx, grad):
        ctx.acc.check_fresh(ctx.updates)
        buf = ctx.acc.buffer(ctx.param, ctx.comm)
        buf.add_(grad.to(buf.dtype))
        return None, None, None, None


def accumulated_average(acc: AccumulatedSGD, comm, param: torch.Tensor) -> torch.Tensor:
    """This step's ``mean_ranks(param)`` whose gradient goes into ``acc`` (composition paths).  At one rank it is a
    copy: ``step()`` updates the parameter in place while a stale node may still hold the average."""
    avg = acc.average(comm, param, (lambda: param.detach().clone()) if comm.size == 1 else None)
    return _AccumulateGrad.apply(param, avg, acc, comm) if param.requires_grad else avg


def owned_accumulated(acc: AccumulatedSGD, param: torch.Tensor) -> torch.Tensor:
    """``param`` as a composition path reads it when ``acc`` accumulates the gradient of a parameter this rank owns
    (no collective, ``step()`` updates it locally): a copy, since ``step()`` updates the parameter in place while a
    stale node may still hold it."""
    return _AccumulateGrad.apply(param, param.detach().clone(), acc, None) if param.requires_grad else param


def _wgrad_accumulate(buf: torch.Tensor, gy: torch.Tensor, x: torch.Tensor, gscale: Optional[torch.Tensor]) -> None:
    """buf += gscale * gy^T @ x, on the accumulating wgrad kernel when it applies."""
    if buf.is_cuda and m4t.cuda_backend_ready() and _ops().wgrad_accumulate_supported(buf, gy, x):
        _ops().wgrad_accumulate_(buf, gy, x, gscale)
        return
    g = gy.t().to(buf.dtype) @ x.to(buf.dtype)
    buf.add_(g if gscale is None else g * gscale.to(buf.dtype))


def _wgrad(gy: torch.Tensor, x: torch.Tensor, gscale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gscale * gy^T @ x on the library's own tensor-core kernel when it applies."""
    gy2, x2 = gy.reshape(-1, gy.shape[-1]), x.reshape(-1, x.shape[-1])
    if gy2.is_cuda and gy2.dtype == torch.bfloat16 and x2.dtype == torch.bfloat16 and m4t.cuda_backend_ready() \
            and _ops().wgrad_bf16_supported(gy2, x2):
        return _ops().wgrad_bf16(gy2, x2, gscale)
    g = gy2.t() @ x2
    return g if gscale is None else g * gscale.to(g.dtype)


def _dgrad(gy: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """gy @ w on the library's own kernel when it applies (mixed-major wgmma GEMM)."""
    if gy.is_cuda and gy.dim() == 2 and gy.dtype == torch.bfloat16 and w.dtype == torch.bfloat16 \
            and m4t.cuda_backend_ready() and hasattr(_ops(), "gemm_bf16_nn") and _ops().gemm_bf16_nn_supported(gy, w):
        return _ops().gemm_bf16_nn(gy, w)
    return gy @ w


class _AllreduceLinearFused(torch.autograd.Function):
    """y = x @ (Allreduce(W, SUM) / size)^T in one kernel; backward = dgrad / wgrad GEMMs + the adjoint
    Allreduce with the 1/size scale in its epilogue."""

    @staticmethod
    def forward(ctx, x, weight, comm_holder):
        comm = comm_holder[0]
        y, w_avg = _ops().allreduce_linear_fused(x, weight, 1.0 / comm.size)
        # w_avg aliases a two-deep symmetric buffer that later calls overwrite: keep a private copy,
        # and only when the input gradient will need it
        ctx.save_for_backward(x, w_avg.clone() if ctx.needs_input_grad[0] else None)
        ctx.comm = comm
        return y

    @staticmethod
    def backward(ctx, gy):
        x, w_avg = ctx.saved_tensors
        comm = ctx.comm
        gx = gw = None
        gy = gy.contiguous()
        if ctx.needs_input_grad[0]:
            gx = _dgrad(gy, w_avg)
        if ctx.needs_input_grad[1]:
            gw_local = _wgrad(gy, x)
            gw = comm.AllreduceFused(gw_local, m4t.MPI_SUM, 1.0 / comm.size, None)
        return gx, gw, None


def allreduce_linear(x: torch.Tensor, weight: torch.Tensor, comm=None, *, force_unfused: bool = False) -> torch.Tensor:
    """``x @ (Allreduce(weight, SUM) / size)^T`` (differentiable w.r.t. both)."""
    c = m4t.COMM_WORLD if comm is None else comm
    fused_ok = (not force_unfused and has_fused_kernel() and c.is_world and x.is_cuda and weight.is_cuda and c.size > 1
                and m4t.cuda_backend_ready() and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16
                and _ops().allreduce_linear_supported(x, weight))
    if fused_ok:
        return _AllreduceLinearFused.apply(x, weight, [c])
    w_avg = c.AllreduceFused(weight, m4t.MPI_SUM, 1.0 / c.size, None)
    return F.linear(x, w_avg)


class _DPLinearMSE(torch.autograd.Function):
    """Local MSE loss of the data-parallel linear layer.

    forward : (Allreduce(W)/size fused into) GEMM with the loss + dL/dy epilogue -> loss_local[1]
    backward: g * dy^T x  ->  adjoint Allreduce (x 1/size)  [-> SGD -> multicast -> next W_avg]
    The upstream gradient ``g`` (a device scalar: the adjoint of the loss Allreduce) is folded into
    the wgrad kernel's epilogue, never read on the host.
    """

    @staticmethod
    def forward(ctx, x, weight, target, comm_holder, loss_scale, opt, allow_fused):
        comm = comm_holder[0]
        ops = _ops()
        w_avg = opt.take_prefetched(weight) if opt is not None else None
        if w_avg is not None:
            dy, local = ops.linear_mse_forward_local(x, w_avg, target, loss_scale, 2.0 * loss_scale)
        else:
            dy, local, w_avg = ops.linear_mse_forward(x, weight, target, 1.0 / comm.size, loss_scale, 2.0 * loss_scale,
                                                      allow_fused)
        need_gx = ctx.needs_input_grad[0]
        ctx.save_for_backward(dy, x, w_avg.clone() if need_gx else None)
        ctx.comm, ctx.opt, ctx.weight = comm, opt, weight
        return local

    @staticmethod
    def backward(ctx, g):
        dy, x, w_avg = ctx.saved_tensors
        comm, opt, weight = ctx.comm, ctx.opt, ctx.weight
        ops = _ops()
        g = g.reshape(1).to(torch.float32)
        gx = gw = None
        if ctx.needs_input_grad[0]:
            gx = _dgrad(dy, w_avg) * g.to(dy.dtype)
        if ctx.needs_input_grad[1]:
            if opt is not None:
                # optimizer-in-backward: the weight is updated by the kernel, no .grad is produced
                scale = -opt.lr / comm.size
                opt.updates += 1
                if comm.size == 1:
                    ops.wgrad_sgd_(weight, dy, x, scale, g)
                    opt.remember(weight, None)
                elif opt.assume_replicated:
                    ops.wgrad_allreduce_sgd_(weight, dy, x, scale, g)
                    opt.remember(weight, weight.detach())  # the replicas are identical: their mean is the weight itself
                elif opt.prefetch:
                    w_next = ops.wgrad_allreduce_sgd_prefetch_(weight, dy, x, scale, g)
                    opt.remember(weight, w_next)
                else:
                    ops.wgrad_allreduce_sgd_(weight, dy, x, scale, g)
                    opt.remember(weight, None)
            else:
                gw_local = _wgrad(dy, x, g)
                gw = comm.AllreduceFused(gw_local, m4t.MPI_SUM, 1.0 / comm.size, None)
        return gx, gw, None, None, None, None, None


class _DPLinearMSEAccumulate(torch.autograd.Function):
    """:class:`_DPLinearMSE` with an :class:`AccumulatedSGD`: the forward reads this step's average of the weight (the
    first forward of a step computes and keeps it), and backward adds ``g * dy^T x`` into the accumulator's fp32 buffer
    (``wgrad_accumulate_``) with no collective; the weight gets no ``.grad``."""

    @staticmethod
    def forward(ctx, x, weight, target, comm_holder, loss_scale, acc, allow_fused):
        comm = comm_holder[0]
        ops = _ops()
        w_avg = acc.cached_average(weight)
        if w_avg is not None:
            dy, local = ops.linear_mse_forward_local(x, w_avg, target, loss_scale, 2.0 * loss_scale)
        else:
            dy, local, w_avg = ops.linear_mse_forward(x, weight, target, 1.0 / comm.size, loss_scale, 2.0 * loss_scale,
                                                      allow_fused)
            # with P > 1 the fused forward's w_avg lives in a two-deep symmetric buffer: keep a copy
            acc.keep_average(weight, w_avg if comm.size == 1 else w_avg.clone())
        ctx.save_for_backward(dy, x, w_avg.clone() if ctx.needs_input_grad[0] else None)
        ctx.comm, ctx.acc, ctx.weight, ctx.acc_updates = comm, acc, weight, acc.updates
        return local

    @staticmethod
    def backward(ctx, g):
        ctx.acc.check_fresh(ctx.acc_updates)
        dy, x, w_avg = ctx.saved_tensors
        g = g.reshape(1).to(torch.float32)
        gx = None
        if ctx.needs_input_grad[0]:
            gx = _dgrad(dy, w_avg) * g.to(dy.dtype)
        if ctx.needs_input_grad[1]:
            _wgrad_accumulate(ctx.acc.buffer(ctx.weight, ctx.comm), dy, x, g)
        return gx, None, None, None, None, None, None


def dp_linear_mse_supported(x: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, comm) -> bool:
    return (comm.is_world and x.is_cuda and x.dim() == 2 and target.dim() == 2 and x.dtype == torch.bfloat16
            and target.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and weight.is_cuda
            and x.stride(1) == 1 and target.stride(1) == 1 and weight.is_contiguous()
            and m4t.cuda_backend_ready() and hasattr(_ops(), "linear_mse_forward")
            and _ops().gemm_bf16_tn_supported(x, weight, target))


def in_backward_sgd_supported(x: torch.Tensor, weight: torch.Tensor, comm) -> bool:
    """Can backward run as the single fused wgrad -> reduce-scatter -> SGD -> multicast kernel?"""
    if not (x.is_cuda and m4t.cuda_backend_ready() and comm.is_world):
        return False
    dy_like = x.new_empty((x.shape[0], weight.shape[0]))
    if comm.size == 1:
        return bool(_ops().wgrad_bf16_supported(dy_like, x))
    return bool(_ops().wgrad_allreduce_sgd_supported(weight, dy_like, x))


def dp_linear_mse(x: torch.Tensor, weight: torch.Tensor, target: torch.Tensor, comm=None, *, loss_scale: float,
                  optimizer: Optional[InBackwardSGD] = None, allow_fused: bool = True,
                  accumulator: Optional[AccumulatedSGD] = None, fp8: bool = False) -> torch.Tensor:
    """``loss_scale * sum((x @ mean_ranks(weight)^T - target)^2)`` of THIS rank's batch as a
    differentiable one-element fp32 tensor; sum it over ranks with ``comm.Allreduce``.

    ``optimizer``: an :class:`InBackwardSGD` makes ``backward`` apply the SGD step itself (fused
    into the gradient reduce-scatter); the weight then receives no ``.grad``.
    ``accumulator``: an :class:`AccumulatedSGD` makes ``backward`` add this rank's gradient into its buffer
    (no collective, no ``.grad``); ``accumulator.step()`` updates the weight.  Not combinable with ``optimizer``.
    ``fp8``: run both GEMMs in fp8 with per-tensor power-of-two scaling (:mod:`mpi4torch_b200.ops.fp8`); ``x.grad``
    stays the bf16 dgrad.  Not combinable with ``accumulator``."""
    c = m4t.COMM_WORLD if comm is None else comm
    if accumulator is not None and optimizer is not None:
        raise ValueError("mpi4torch_b200: dp_linear_mse takes either optimizer= or accumulator=, not both")
    if fp8:
        if accumulator is not None:
            raise ValueError("mpi4torch_b200: dp_linear_mse(fp8=True) does not support accumulator=")
        return dp_linear_mse_fp8(x, weight, target, c, loss_scale, optimizer)
    if accumulator is not None:
        if dp_linear_mse_supported(x, weight, target, c):
            return _DPLinearMSEAccumulate.apply(x, weight, target, [c], float(loss_scale), accumulator,
                                                bool(allow_fused))
        y = F.linear(x, accumulated_average(accumulator, c, weight))
        acc = torch.float64 if y.dtype == torch.float64 else torch.float32
        return ((y.to(acc) - target.to(acc)).square().sum() * loss_scale).reshape(1)
    if dp_linear_mse_supported(x, weight, target, c):
        if optimizer is not None and not in_backward_sgd_supported(x, weight, c):
            raise RuntimeError("mpi4torch_b200: InBackwardSGD needs a bf16 CUDA weight from symmetric_empty() on the "
                               "world communicator with the NVLS transport up (and N % 256 == K % 256 == batch % 128 == 0)")
        return _DPLinearMSE.apply(x, weight, target, [c], float(loss_scale), optimizer, bool(allow_fused))
    if optimizer is not None:
        raise RuntimeError("mpi4torch_b200: InBackwardSGD is only available on the fused CUDA path")
    y = allreduce_linear(x, weight, c, force_unfused=not allow_fused)
    acc = torch.float64 if y.dtype == torch.float64 else torch.float32  # accumulate in fp32 (fp64 inputs stay fp64)
    return ((y.to(acc) - target.to(acc)).square().sum() * loss_scale).reshape(1)
