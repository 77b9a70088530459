"""Data-parallel two-layer MLP (``Linear -> GELU(tanh) -> Linear``, biases, MSE loss) as one autograd node
backed by the library's wgmma kernels.

``dp_mlp_mse(x, W1, b1, W2, b2, t, ...)``  loss_local = loss_scale * sum((y - t)^2),
    z = x @ mean_ranks(W1)^T + mean_ranks(b1),  h = gelu_tanh(z),  y = h @ mean_ranks(W2)^T + mean_ranks(b2)

Forward is two GEMMs with their epilogues (csrc/kernels/gemm_wgmma.cu): bias + GELU storing z and h, then
bias + MSE storing dL/dy, adding the loss and writing column-sum partials of dL/dy (y itself is never stored).
Backward is the GELU-backward GEMM (dz, with its column-sum partials), the two weight-gradient GEMMs and the
deterministic column-sum reduce for the biases.  With :class:`InBackwardSGD` optimizers the weights are
updated inside backward by the wgrad kernels (with P > 1: reduce-scatter -> SGD -> multicast -> average of
the new weights for the next forward, one kernel per weight) and the biases by ``allreduce_axpy_``; the
parameters then receive no ``.grad``.  With an :class:`AccumulatedSGD` backward instead adds this rank's gradients
into fp32 buffers (``wgrad_accumulate_`` for the weights, column sums for the biases) with no collective, and the
forwards of one step share the parameter averages computed by its first forward.

``dp_mlp_cross_entropy(x, W1, b1, W2, b2, labels, ...)``  loss_local = loss_scale * sum_rows CE(y, labels)
    The same node with a softmax cross-entropy output layer: the second GEMM stores the bf16 logits and per-tile
    softmax partials, and ``xent_finish`` turns the logits into dL/dy = loss_scale * (softmax(y) - onehot) in place,
    with the loss and the same column-sum partials.  The backward is the MSE node's, unchanged.

Elsewhere (CPU tensors, other dtypes, shapes the kernels reject, communicators created by ``Split``) the same
math runs as the composition ``F.linear -> F.gelu(tanh) -> F.linear -> MSE`` (or ``F.cross_entropy``) on
``AllreduceFused`` averages, which gives the same gradients.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F

import mpi4torch_b200 as m4t

from .fused_linear import AccumulatedSGD, InBackwardSGD, _ops, accumulated_average


def _average(comm, p: torch.Tensor) -> torch.Tensor:
    return p if comm.size == 1 else comm.AllreduceFused(p, m4t.MPI_SUM, 1.0 / comm.size, None)


def _update_weight(ops, comm, opt: InBackwardSGD, weight, dy, x, g) -> None:
    scale = -opt.lr / comm.size
    opt.updates += 1
    if comm.size == 1:
        ops.wgrad_sgd_(weight, dy, x, scale, g)
        opt.remember(weight, None)
    elif opt.prefetch:
        opt.remember(weight, ops.wgrad_allreduce_sgd_prefetch_(weight, dy, x, scale, g))
    else:
        ops.wgrad_allreduce_sgd_(weight, dy, x, scale, g)
        opt.remember(weight, None)


def _mlp_forward(ctx, x, w1, b1, w2, b2, comm, opts, output_layer, acc=None):
    """Forward of the MLP nodes up to the loss: the parameter averages (the prefetched ones, or with an accumulator
    this step's), the bias + GELU GEMM, then ``output_layer(ops, h, w2_avg, b2_avg) -> (dy, loss, dy_part)``, which
    stores dL/dy and its column-sum partials.  Saves what :meth:`_DPMLPMSE.backward` reads."""
    ops = _ops()
    if acc is not None:
        w1_avg, b1_avg, w2_avg, b2_avg = (acc.average(comm, p) for p in (w1, b1, w2, b2))
    else:
        w1_avg = opts[0].take_prefetched(w1) if opts is not None else None
        w2_avg = opts[1].take_prefetched(w2) if opts is not None else None
        w1_avg = _average(comm, w1) if w1_avg is None else w1_avg
        w2_avg = _average(comm, w2) if w2_avg is None else w2_avg
        b1_avg, b2_avg = _average(comm, b1), _average(comm, b2)
    h, z = ops.linear_bias_gelu_forward(x, w1_avg, b1_avg)
    dy, local, dy_part = output_layer(ops, h, w2_avg, b2_avg)
    ctx.save_for_backward(x, h, z, dy, w1_avg, w2_avg, dy_part)
    ctx.comm, ctx.opts, ctx.params, ctx.acc = comm, opts, (w1, b1, w2, b2), acc
    # w1_avg / w2_avg are the weights themselves (P = 1) or the prefetch buffers (P > 1), which the next in-backward
    # update rewrites without bumping torch's version counter: backward checks these counts instead
    ctx.opt_updates = None if opts is None else (opts[0].updates, opts[1].updates)
    ctx.acc_updates = None if acc is None else acc.updates
    return local


class _DPMLPMSE(torch.autograd.Function):
    """Local MSE loss of the data-parallel two-layer MLP; backward folds the upstream device scalar ``g``
    into the kernels' epilogues (never read on the host)."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, target, comm_holder, loss_scale, opts, acc=None):
        def output_layer(ops, h, w2_avg, b2_avg):
            return ops.linear_bias_mse_forward_local(h, w2_avg, b2_avg, target, loss_scale, 2.0 * loss_scale)

        return _mlp_forward(ctx, x, w1, b1, w2, b2, comm_holder[0], opts, output_layer, acc)

    @staticmethod
    def backward(ctx, g):
        if ctx.acc is not None:
            return _accumulate_backward(ctx, g)
        x, h, z, dy, w1_avg, w2_avg, dy_part = ctx.saved_tensors
        comm, opts = ctx.comm, ctx.opts
        w1, b1, w2, b2 = ctx.params
        if opts is not None and (opts[0].updates, opts[1].updates) != ctx.opt_updates:
            raise RuntimeError("mpi4torch_b200: the MLP weights were updated in place by another backward since this "
                               "node's forward, so its saved weights are stale; with InBackwardSGD, run one backward "
                               "per forward")
        ops = _ops()
        g = g.reshape(1).to(torch.float32)
        need = ctx.needs_input_grad
        # Order of the reads and updates.  Every read of a layer's averaged weight is enqueued before that
        # layer's fused update, which may overwrite it: at P = 1 the average IS the weight (wgrad_sgd_ updates it
        # in place), and with a prefetching optimizer it is the buffer the update kernel refills with the next
        # average.  Across ranks this needs no copy either: the update kernel writes the new average of a tile
        # into a peer's buffer only after every rank's partial gradients of that tile have arrived, and a rank
        # produces its partials only after its own earlier reads, which come first in its stream.
        #   1. dz reads W2_avg;  2. layer-2 update;  3. dx reads W1_avg;  4. layer-1 update;  5. biases.
        # In-backward mode updates only the parameters that require a gradient, so a frozen one stays as it is.
        dz, dz_part = ops.gemm_nn_gelu_backward(dy, w2_avg, z, g)
        gx = gw1 = gb1 = gw2 = gb2 = None
        if opts is not None:
            if need[3]:
                _update_weight(ops, comm, opts[1], w2, dy, h, g)
        elif need[3]:
            gw2 = comm.AllreduceFused(ops.wgrad_bf16(dy, h, g), m4t.MPI_SUM, 1.0 / comm.size, None)
        if need[0]:
            gx = ops.gemm_bf16_nn(dz, w1_avg)
        if opts is not None:
            if need[1]:
                _update_weight(ops, comm, opts[0], w1, dz, x, None)
        elif need[1]:
            gw1 = comm.AllreduceFused(ops.wgrad_bf16(dz, x, None), m4t.MPI_SUM, 1.0 / comm.size, None)
        db2 = ops.column_sum(dy_part, g)
        db1 = ops.column_sum(dz_part, None)
        if opts is not None:
            # one path for every P, summed in a fixed order: the biases stay bit-identical across ranks
            if need[4]:
                ops.allreduce_axpy_(b2, db2, -opts[1].lr / comm.size)
            if need[2]:
                ops.allreduce_axpy_(b1, db1, -opts[0].lr / comm.size)
        else:
            if need[4]:
                gb2 = comm.AllreduceFused(db2, m4t.MPI_SUM, 1.0 / comm.size, None)
            if need[2]:
                gb1 = comm.AllreduceFused(db1, m4t.MPI_SUM, 1.0 / comm.size, None)
        return gx, gw1, gb1, gw2, gb2, None, None, None, None, None


def _accumulate_backward(ctx, g):
    """Backward of the MLP nodes with an :class:`AccumulatedSGD`: this rank's gradients of the parameter averages
    are added into the accumulator's buffers, with no collective; only ``x`` gets a gradient.  The averages are this
    step's, and nothing overwrites them before ``step()``, so the order of the reads does not matter here."""
    comm, acc = ctx.comm, ctx.acc
    acc.check_fresh(ctx.acc_updates)  # first: at one rank the saved averages are the parameters that step() updated
    x, h, z, dy, w1_avg, w2_avg, dy_part = ctx.saved_tensors
    w1, b1, w2, b2 = ctx.params
    ops = _ops()
    g = g.reshape(1).to(torch.float32)
    need = ctx.needs_input_grad
    dz, dz_part = ops.gemm_nn_gelu_backward(dy, w2_avg, z, g)
    if need[3]:
        ops.wgrad_accumulate_(acc.buffer(w2, comm), dy, h, g)
    if need[1]:
        ops.wgrad_accumulate_(acc.buffer(w1, comm), dz, x, None)
    if need[4]:
        acc.buffer(b2, comm).add_(ops.column_sum(dy_part, g))
    if need[2]:
        acc.buffer(b1, comm).add_(ops.column_sum(dz_part, None))
    gx = ops.gemm_bf16_nn(dz, w1_avg) if need[0] else None
    return gx, None, None, None, None, None, None, None, None, None


class _DPMLPCrossEntropy(_DPMLPMSE):
    """Local softmax cross-entropy loss of the data-parallel two-layer MLP.  Only the output layer differs from
    :class:`_DPMLPMSE`: it stores ``dL/dy = loss_scale * (softmax(y) - onehot(labels))`` and its column-sum
    partials, so the backward is inherited unchanged.  ``loss_args`` is ``(loss_scale, ignore_index)``."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, labels, comm_holder, loss_args, opts, acc=None):
        loss_scale, ignore_index = loss_args

        def output_layer(ops, h, w2_avg, b2_avg):
            return ops.linear_bias_xent_forward_local(h, w2_avg, b2_avg, labels, loss_scale, loss_scale, ignore_index)

        return _mlp_forward(ctx, x, w1, b1, w2, b2, comm_holder[0], opts, output_layer, acc)


def _kernel_ops_present() -> bool:
    return hasattr(_ops(), "linear_bias_gelu_forward")


def _mlp_kernels_supported(x, w1, b1, w2, b2, c) -> bool:
    """The rules both MLP losses share: D, H, O multiples of 128, the batch a multiple of 64, contiguous bf16 weights
    and input, contiguous fp32 biases, every operand of the two forward GEMMs aligned as the kernels read it."""
    if not (c.is_world and m4t.cuda_backend_ready() and _kernel_ops_present()):
        return False
    if not all(t.is_cuda and t.dim() == 2 and t.dtype == torch.bfloat16 and t.is_contiguous() for t in (x, w1, w2)):
        return False
    if not all(b.is_cuda and b.dim() == 1 and b.dtype == torch.float32 and b.is_contiguous() for b in (b1, b2)):
        return False
    (B, D), (H, D1), (O, H1) = x.shape, w1.shape, w2.shape
    if not (D1 == D and H1 == H and b1.shape[0] == H and b2.shape[0] == O):
        return False
    if not (B % 64 == 0 and D % 128 == 0 and H % 128 == 0 and O % 128 == 0 and B > 0):
        return False
    # base alignment and row strides of every operand the two forward GEMMs read (h is allocated by the first)
    ops = _ops()
    return bool(ops.gemm_bf16_tn_supported(x, w1, None, b1) and ops.gemm_bf16_tn_supported(x.new_empty((B, H)), w2, None, b2))


def dp_mlp_mse_supported(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor,
                         target: torch.Tensor, comm=None) -> bool:
    """Does :func:`dp_mlp_mse` run on the library's kernels for these tensors (plain-gradient mode)?
    D, H, O must be multiples of 128, the batch a multiple of 64, and every operand aligned as the kernels read
    it (see ``gemm_bf16_tn_supported``)."""
    c = m4t.COMM_WORLD if comm is None else comm
    if not _mlp_kernels_supported(x, w1, b1, w2, b2, c):
        return False
    if not (target.is_cuda and target.dim() == 2 and target.dtype == torch.bfloat16 and target.is_contiguous()
            and tuple(target.shape) == (x.shape[0], w2.shape[0])):
        return False
    return bool(_ops().gemm_bf16_tn_supported(x.new_empty((x.shape[0], w1.shape[0])), w2, target, b2))


def dp_mlp_cross_entropy_supported(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor,
                                   b2: torch.Tensor, labels: torch.Tensor, comm=None) -> bool:
    """Does :func:`dp_mlp_cross_entropy` run on the library's kernels for these tensors (plain-gradient mode)?
    The rules of :func:`dp_mlp_mse_supported` (C = number of classes in place of O), and ``labels`` a contiguous
    1-d int64 CUDA tensor with one label per row."""
    c = m4t.COMM_WORLD if comm is None else comm
    if not (labels.is_cuda and labels.dim() == 1 and labels.dtype == torch.int64 and labels.is_contiguous()
            and x.dim() == 2 and labels.shape[0] == x.shape[0] and labels.device == x.device):
        return False
    return _mlp_kernels_supported(x, w1, b1, w2, b2, c) and hasattr(_ops(), "linear_bias_xent_forward_local")


def mlp_in_backward_sgd_supported(x: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, comm=None) -> bool:
    """Can backward update both weights inside their wgrad kernels?  With P > 1 the weights must come from
    ``symmetric_empty()``, D, H, O must be multiples of 256, the batch a multiple of 128, and the arena must
    have room for both weights' buffers."""
    c = m4t.COMM_WORLD if comm is None else comm
    B = x.shape[0]
    h_like = x.new_empty((B, w1.shape[0]))
    dy_like = x.new_empty((B, w2.shape[0]))
    if c.size == 1:
        return bool(_ops().wgrad_bf16_supported(h_like, x) and _ops().wgrad_bf16_supported(dy_like, h_like))
    return bool(_ops().wgrad_allreduce_sgd_supported(w1, h_like, x)
                and _ops().wgrad_allreduce_sgd_supported(w2, dy_like, h_like))


def dp_mlp_mse(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor,
               target: torch.Tensor, comm=None, *, loss_scale: float,
               optimizers: Optional[Sequence[InBackwardSGD]] = None,
               accumulator: Optional[AccumulatedSGD] = None) -> torch.Tensor:
    """``loss_scale * sum((MLP(x) - target)^2)`` of THIS rank's batch as a differentiable one-element fp32
    tensor, with every parameter averaged over ranks; sum it over ranks with ``comm.Allreduce``.

    ``optimizers``: ``(opt1, opt2)``, one :class:`InBackwardSGD` per layer, makes ``backward`` apply the SGD
    step to ``(w1, b1)`` and ``(w2, b2)`` itself; the parameters then receive no ``.grad``.  Two rules hold in
    that mode:
      * only parameters with ``requires_grad`` are updated: a frozen weight or bias stays unchanged;
      * run one backward per forward.  Backward reads the weights (or their prefetched averages) as they were at
        this node's forward, and another node's backward updates them in place, so a node whose weights were
        updated since its forward raises ``RuntimeError`` instead of computing its gradients from the new ones.
        For example ``(model.loss(xa, ta) + model.loss(xb, tb)).backward()`` raises after applying one update.

    ``accumulator``: an :class:`AccumulatedSGD` makes ``backward`` add this rank's gradients into its buffers instead
    (no collective, no ``.grad``, frozen parameters skipped); ``accumulator.step()`` then applies one update.  Several
    forwards may precede one backward in this mode.  It cannot be combined with ``optimizers``."""
    c = m4t.COMM_WORLD if comm is None else comm
    _check_one_optimizer("dp_mlp_mse", optimizers, accumulator)
    if dp_mlp_mse_supported(x, w1, b1, w2, b2, target, c):
        optimizers = _kernel_optimizers("dp_mlp_mse", optimizers, x, w1, w2, c)
        return _DPMLPMSE.apply(x, w1, b1, w2, b2, target, [c], float(loss_scale), optimizers, accumulator)
    y, acc = _composition(x, w1, b1, w2, b2, c, optimizers, accumulator)
    return ((y.to(acc) - target.to(acc)).square().sum() * loss_scale).reshape(1)


def dp_mlp_cross_entropy(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: torch.Tensor,
                         labels: torch.Tensor, comm=None, *, loss_scale: float, ignore_index: int = -100,
                         optimizers: Optional[Sequence[InBackwardSGD]] = None,
                         accumulator: Optional[AccumulatedSGD] = None) -> torch.Tensor:
    """``loss_scale * sum_rows cross_entropy(MLP(x), labels)`` of THIS rank's batch (``F.cross_entropy`` with
    ``reduction="sum"``) as a differentiable one-element fp32 tensor, with every parameter averaged over ranks;
    sum it over ranks with ``comm.Allreduce``.  ``labels``: one int64 class index per row of ``x``.  A row labelled
    ``ignore_index`` adds nothing to the loss or the gradients.  On the kernel path any other label outside
    ``[0, C)`` makes the loss NaN (``F.cross_entropy`` raises instead).

    The softmax is taken over the bf16 logits ``bf16(h @ W2^T + b2)``.  ``optimizers`` as in :func:`dp_mlp_mse`,
    with the same two rules: frozen parameters are not updated, and one backward per forward.
    The kernels need C % 128 == 0: pad the classes to the next multiple of 128 and give the padded classes bias
    ``-inf``, which gives them probability 0 and gradient 0, so their bias stays ``-inf``.
    ``accumulator`` as in :func:`dp_mlp_mse`."""
    if not (labels.dim() == 1 and labels.dtype == torch.int64 and x.dim() == 2 and labels.shape[0] == x.shape[0]):
        raise ValueError(f"mpi4torch_b200: dp_mlp_cross_entropy needs int64 labels of shape ({x.shape[0]},), got "
                         f"{labels.dtype} of shape {tuple(labels.shape)}")
    c = m4t.COMM_WORLD if comm is None else comm
    _check_one_optimizer("dp_mlp_cross_entropy", optimizers, accumulator)
    if dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels, c):
        optimizers = _kernel_optimizers("dp_mlp_cross_entropy", optimizers, x, w1, w2, c)
        return _DPMLPCrossEntropy.apply(x, w1, b1, w2, b2, labels, [c], (float(loss_scale), int(ignore_index)),
                                        optimizers, accumulator)
    y, acc = _composition(x, w1, b1, w2, b2, c, optimizers, accumulator)
    return (F.cross_entropy(y.to(acc), labels, reduction="sum", ignore_index=ignore_index) * loss_scale).reshape(1)


def _check_one_optimizer(name, optimizers, accumulator):
    if optimizers is not None and accumulator is not None:
        raise ValueError(f"mpi4torch_b200: {name} takes either optimizers= or accumulator=, not both")


def _kernel_optimizers(name, optimizers, x, w1, w2, c):
    if optimizers is None:
        return None
    if len(optimizers) != 2:
        raise ValueError(f"mpi4torch_b200: {name} takes one InBackwardSGD per layer")
    if not mlp_in_backward_sgd_supported(x, w1, w2, c):
        raise RuntimeError("mpi4torch_b200: InBackwardSGD for the MLP needs, with more than one rank, bf16 weights "
                           "from symmetric_empty() with D, H, O % 256 == 0 and batch % 128 == 0")
    return tuple(optimizers)


def _composition(x, w1, b1, w2, b2, c, optimizers, accumulator=None):
    """Off the kernel path: the MLP output ``y`` as the torch composition on ``AllreduceFused`` averages (with an
    accumulator: this step's averages, whose gradients go into its buffers), and the dtype the loss accumulates in
    (fp32; fp64 inputs stay fp64)."""
    if optimizers is not None:
        raise RuntimeError("mpi4torch_b200: InBackwardSGD is only available on the CUDA kernel path")
    if accumulator is not None:
        avg = lambda p: accumulated_average(accumulator, c, p)  # noqa: E731
    else:
        avg = lambda p: c.AllreduceFused(p, m4t.MPI_SUM, 1.0 / c.size, None)  # noqa: E731
    acc = torch.float64 if x.dtype == torch.float64 else torch.float32
    h = F.gelu(F.linear(x, avg(w1), avg(b1).to(x.dtype)), approximate="tanh")
    return F.linear(h, avg(w2), avg(b2).to(h.dtype)), acc
