"""Data-parallel two-layer MLP: ``Linear(D, H) -> GELU(tanh) -> Linear(H, O)`` with biases and an MSE loss.

One training step, every rank, on the autograd graph:

    local = dp_mlp_mse(x, W1, b1, W2, b2, t)   bias+GELU GEMM -> bias+MSE GEMM (loss, dL/dy, bias-gradient partials)
    loss  = comm.Allreduce(local, MPI_SUM)     the library's differentiable Allreduce
    loss.backward()                            GELU-backward GEMM, the two wgrad GEMMs (with the SGD step and, with
                                               more than one rank, the gradient reduce-scatter and the next step's
                                               weight average inside them), column sums -> bias updates

With ``sgd_in_backward=False`` (or off the kernel path) the parameters get ordinary ``.grad`` tensors and
``train_step`` applies SGD.  With ``sgd_in_backward=True`` a parameter set to ``requires_grad_(False)`` is not
updated, and each ``loss()`` needs its ``backward()`` before the next ``loss()`` is computed: a backward whose
forward came before another backward's weight update raises ``RuntimeError``, because its saved weights were
overwritten.  So summing two losses and calling ``backward()`` once raises, after applying one of the two updates.  Biases are fp32 when the weights are 16-bit: a bf16 bias would lose SGD updates
below 2^-8 of its value.

``train_step(x, t, micro_batches=K)`` with K > 1 is gradient accumulation: the batch is split into K chunks, each
chunk's forward and backward add this rank's gradients into the fp32 buffers of ``model.accumulator`` (an
:class:`AccumulatedSGD`, whatever ``sgd_in_backward`` says) with no parameter-sized collective, and one
``accumulator.step()`` all-reduces the buffers and updates the parameters.  The accumulator is also the supported
way to combine several losses into one update: pass ``accumulator=model.accumulator`` to ``dp_mlp_mse``, sum the
losses, call ``backward()`` once, then ``model.accumulator.step()``.

``DPMLPClassifier`` is the same model with a softmax cross-entropy loss over integer class labels
(``dp_mlp_cross_entropy``); only the output layer's forward kernels differ.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import mpi4torch_b200 as m4t
from mpi4torch_b200.ops import (AccumulatedSGD, InBackwardSGD, dp_mlp_cross_entropy, dp_mlp_cross_entropy_supported,
                                dp_mlp_mse, dp_mlp_mse_supported, mlp_in_backward_sgd_supported)


class DPMLPModel:
    """The data-parallel two-layer MLP with an MSE loss (see the module docstring for one step).

    ``model.accumulator`` (an :class:`AccumulatedSGD`) is the supported way to combine several losses into one update:
    pass ``accumulator=model.accumulator`` to ``dp_mlp_mse``, call ``backward()`` on each loss or on their sum, then
    ``model.accumulator.step()``.  ``train_step(x, t, micro_batches=K)`` does this for K chunks of one batch.  With the
    in-backward optimizers, summing two ``loss()`` results and calling ``backward()`` once raises instead."""

    def __init__(self, in_features: int, hidden_features: int, out_features: int, comm=None, device="cuda",
                 dtype=torch.bfloat16, lr: float = 1e-4, seed: int = 0, sgd_in_backward: bool = True,
                 prefetch: bool = True):
        self.comm = m4t.COMM_WORLD if comm is None else comm
        g = torch.Generator().manual_seed(seed)  # identical initial parameters on every rank
        w1 = torch.randn(hidden_features, in_features, generator=g) * (in_features ** -0.5)
        w2 = torch.randn(out_features, hidden_features, generator=g) * (hidden_features ** -0.5)
        dev = torch.device(device)
        symmetric = (dev.type == "cuda" and dtype == torch.bfloat16 and self.comm.size > 1 and self.comm.is_world
                     and m4t.cuda_backend_ready() and hasattr(torch.ops.mpi4torch_b200, "symmetric_empty"))
        self.w1 = self._weight(w1, dev, dtype, symmetric)
        self.w2 = self._weight(w2, dev, dtype, symmetric)
        bias_dtype = torch.float32 if dtype in (torch.bfloat16, torch.float16) else dtype
        self.b1 = torch.zeros(hidden_features, device=dev, dtype=bias_dtype, requires_grad=True)
        self.b2 = torch.zeros(out_features, device=dev, dtype=bias_dtype, requires_grad=True)
        self.lr = lr
        self.sgd_in_backward = sgd_in_backward
        self.optimizers = (InBackwardSGD(lr, prefetch=prefetch), InBackwardSGD(lr, prefetch=prefetch))
        self.accumulator = AccumulatedSGD(lr)  # train_step(..., micro_batches > 1)
        self._opt_ok = {}

    @staticmethod
    def _weight(w: torch.Tensor, dev: torch.device, dtype, symmetric: bool) -> torch.Tensor:
        if symmetric:
            # in the symmetric heap the fused backward kernels (and the NVSwitch) update it in place
            storage = torch.ops.mpi4torch_b200.symmetric_empty(list(w.shape), dtype)
            storage.copy_(w.to(dtype))
            return storage.requires_grad_()
        return w.to(device=dev, dtype=dtype).requires_grad_()

    def parameters(self):
        return [self.w1, self.b1, self.w2, self.b2]

    def _in_backward(self, x: torch.Tensor, target: torch.Tensor) -> bool:
        if not self.sgd_in_backward:
            return False
        key = (x.device, x.dtype, tuple(x.shape), tuple(x.stride()), tuple(target.shape))
        ok = self._opt_ok.get(key)
        if ok is None:
            ok = (self._kernels_supported(x, target)
                  and mlp_in_backward_sgd_supported(x, self.w1, self.w2, self.comm))
            self._opt_ok[key] = ok
        return ok

    def _kernels_supported(self, x: torch.Tensor, target: torch.Tensor) -> bool:
        return dp_mlp_mse_supported(x, self.w1, self.b1, self.w2, self.b2, target, self.comm)

    def _local_loss(self, x, target, loss_scale, optimizers=None, accumulator=None):
        return dp_mlp_mse(x, self.w1, self.b1, self.w2, self.b2, target, self.comm, loss_scale=loss_scale,
                          optimizers=optimizers, accumulator=accumulator)

    def loss(self, x: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """Global mean-squared-error loss as a differentiable one-element tensor."""
        opts = self.optimizers if self._in_backward(x, target) else None
        local = self._local_loss(x, target, 1.0 / (x.shape[0] * self.comm.size), optimizers=opts)
        return self.comm.Allreduce(local, m4t.MPI_SUM)

    def train_step(self, x: torch.Tensor, target: torch.Tensor, micro_batches: int = 1) -> torch.Tensor:
        """forward + backward + SGD update through the autograd graph; returns the (global) loss.

        ``micro_batches`` = K > 1: K forwards and backwards over equal chunks of this rank's batch (K must divide it)
        into ``self.accumulator``, then one update; the loss returned is the whole batch's."""
        if micro_batches != 1:
            return accumulated_step(self.comm, self.accumulator, self._local_loss, x, target, micro_batches)
        value = self.loss(x, target)
        value.backward()
        if any(p.grad is not None for p in self.parameters()):  # the optimizers did not run inside backward
            for opt in self.optimizers:
                opt.invalidate()
            with torch.no_grad():
                for p in self.parameters():
                    if p.grad is not None:
                        p.add_(p.grad, alpha=-self.lr)
                        p.grad = None
        return value.detach().reshape(())


def accumulated_step(comm, accumulator: AccumulatedSGD, local_loss, x: torch.Tensor, target: torch.Tensor,
                     micro_batches: int) -> torch.Tensor:
    """One SGD step over ``micro_batches`` equal chunks of this rank's batch, accumulated in ``accumulator``:
    ``local_loss(x_chunk, target_chunk, loss_scale, accumulator=...)`` per chunk with ``loss_scale = 1 / (B * P)``
    of the WHOLE batch, so the buffers hold the whole batch's gradient; then one ``accumulator.step()``.  Returns
    the global loss of the whole batch (the sum of the chunks' global losses)."""
    B = x.shape[0]
    K = int(micro_batches)
    if K < 1 or B % K != 0:
        raise ValueError(f"mpi4torch_b200: micro_batches={micro_batches} must be a positive divisor of the batch "
                         f"size {B}")
    loss_scale = 1.0 / (B * comm.size)
    total = None
    for xc, tc in zip(x.split(B // K), target.split(B // K)):
        value = comm.Allreduce(local_loss(xc, tc, loss_scale, accumulator=accumulator), m4t.MPI_SUM)
        value.backward()
        total = value.detach() if total is None else total + value.detach()
    accumulator.step()
    return total.reshape(())


class DPMLPClassifier(DPMLPModel):
    """The same MLP with ``num_classes`` outputs, trained with softmax cross-entropy (``dp_mlp_cross_entropy``).

    ``loss(x, labels)`` is ``sum over every rank's non-ignored rows of CE / (B * P)``: rows labelled ``ignore_index``
    add nothing to the numerator but still count in the denominator B * P, so with ignored rows this is not
    ``F.cross_entropy``'s ``mean`` (which divides by the number of non-ignored rows).  ``train_step(x, labels)`` is
    inherited.

    The kernels need ``num_classes % 128 == 0``; other class counts run the torch composition.  To keep such a model
    on the kernels, pad the classes: build it with ``num_classes`` rounded up to a multiple of 128 and set the padded
    classes' bias to ``-inf`` (``model.b2.data[n:] = float("-inf")``).  Their logits are ``-inf``, so they get
    probability 0 and gradient 0, their bias stays ``-inf``, and the loss and the real classes' gradients are those
    of the unpadded model.  Read the first ``n`` columns of :meth:`logits`.
    """

    def __init__(self, in_features: int, hidden_features: int, num_classes: int, comm=None, device="cuda",
                 dtype=torch.bfloat16, lr: float = 1e-4, seed: int = 0, sgd_in_backward: bool = True,
                 prefetch: bool = True, ignore_index: int = -100):
        super().__init__(in_features, hidden_features, num_classes, comm=comm, device=device, dtype=dtype, lr=lr,
                         seed=seed, sgd_in_backward=sgd_in_backward, prefetch=prefetch)
        self.ignore_index = ignore_index

    def _kernels_supported(self, x: torch.Tensor, labels: torch.Tensor) -> bool:
        return dp_mlp_cross_entropy_supported(x, self.w1, self.b1, self.w2, self.b2, labels, self.comm)

    def _local_loss(self, x, labels, loss_scale, optimizers=None, accumulator=None):
        return dp_mlp_cross_entropy(x, self.w1, self.b1, self.w2, self.b2, labels, self.comm, loss_scale=loss_scale,
                                    ignore_index=self.ignore_index, optimizers=optimizers, accumulator=accumulator)

    def loss(self, x: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """Global cross-entropy loss (sum over non-ignored rows / (B * P)) as a differentiable one-element tensor."""
        opts = self.optimizers if self._in_backward(x, labels) else None
        local = self._local_loss(x, labels, 1.0 / (x.shape[0] * self.comm.size), optimizers=opts)
        return self.comm.Allreduce(local, m4t.MPI_SUM)

    @torch.no_grad()
    def logits(self, x: torch.Tensor) -> torch.Tensor:
        """``h @ W2^T + b2`` with ``h = gelu_tanh(x @ W1^T + b1)``, this rank's parameters, for evaluation."""
        h = F.gelu(F.linear(x, self.w1, self.b1.to(x.dtype)), approximate="tanh")
        return F.linear(h, self.w2, self.b2.to(h.dtype))
