"""Data-parallel linear layer (BASELINE.json config: "4096x4096 linear layer:
Allreduce(params)->GEMM fused, loss Allreduce backward").

One training step, every rank, written the way the reference's data-parallel example is
(reference examples/simple_linear_regression.py:27-35) - all of it on the autograd graph:

    local = dp_linear_mse(x, W, t)             node 1: Allreduce(W)/size -> GEMM -> MSE   (one kernel)
    loss  = comm.Allreduce(local, MPI_SUM)     node 2: the library's differentiable Allreduce
    loss.backward()                            node 2's adjoint Allreduce of the scalar gradient, then
                                               node 1's backward: wgrad GEMM -> adjoint Allreduce of dW
                                               (-> SGD -> multicast of W -> next step's W average:
                                               one kernel when the optimizer runs in backward)

With ``sgd_in_backward=False`` the weight gets an ordinary ``.grad`` and ``train_step`` applies SGD.
``train_step(x, t, micro_batches=K)`` with K > 1 accumulates the gradients of K equal chunks of the batch in
``model.accumulator`` (an :class:`AccumulatedSGD`, fp32 buffers, no parameter-sized collective in backward) and
then updates once.

``fp8=True`` runs both GEMMs of the step in fp8 (``dp_linear_mse(..., fp8=True)``, DESIGN §4.4): E4M3 ``x`` and weight
average, E5M2 ``dy``, per-tensor power-of-two scales kept on the device.  The in-backward optimizer then updates the
weight in the fp8 wgrad kernel's epilogue at one rank and through ``allreduce_axpy_`` at several.  Micro-batch
accumulation is not available with fp8.
"""
from __future__ import annotations

import torch

import mpi4torch_b200 as m4t
from mpi4torch_b200.models.dp_mlp import accumulated_step
from mpi4torch_b200.ops import (AccumulatedSGD, InBackwardSGD, allreduce_linear, dp_linear_mse,
                                in_backward_sgd_supported)
from mpi4torch_b200.ops.fp8 import dp_linear_mse_fp8_supported


class DPLinearModel:
    def __init__(self, in_features: int = 4096, out_features: int = 4096, comm=None, device="cuda",
                 dtype=torch.bfloat16, lr: float = 1e-4, seed: int = 0, fused: bool = True,
                 sgd_in_backward: bool = True, prefetch: bool = True, assume_replicated: bool = False,
                 fp8: bool = False):
        self.comm = m4t.COMM_WORLD if comm is None else comm
        g = torch.Generator().manual_seed(seed)  # identical initial weights on every rank
        w = torch.randn(out_features, in_features, generator=g) * (in_features ** -0.5)
        dev = torch.device(device)
        if (dev.type == "cuda" and dtype == torch.bfloat16 and self.comm.size > 1 and self.comm.is_world
                and m4t.cuda_backend_ready()
                and hasattr(torch.ops.mpi4torch_b200, "symmetric_empty")):
            # keep the parameter in the symmetric heap: the fused kernels (and the NVSwitch) then
            # read and update it in place, no staging copy
            storage = torch.ops.mpi4torch_b200.symmetric_empty(list(w.shape), dtype)
            storage.copy_(w.to(dtype))
            self.weight = storage.requires_grad_()
        else:
            self.weight = w.to(device=device, dtype=dtype).requires_grad_()
        self.lr = lr
        self.fused = fused  # Allreduce->GEMM in one kernel when the NVLS path is up
        self.sgd_in_backward = sgd_in_backward  # fused wgrad -> reduce-scatter -> SGD -> multicast in backward
        self.optimizer = InBackwardSGD(lr, prefetch=prefetch, assume_replicated=assume_replicated)
        self.accumulator = AccumulatedSGD(lr)  # train_step(..., micro_batches > 1)
        self.fp8 = bool(fp8)
        self._opt_ok = {}

    # ------------------------------------------------------------------ graph construction
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return allreduce_linear(x, self.weight, self.comm, force_unfused=not self.fused)

    def _in_backward(self, x: torch.Tensor) -> bool:
        if not self.sgd_in_backward:
            return False
        key = (x.device, x.dtype, tuple(x.shape), tuple(x.stride()))
        ok = self._opt_ok.get(key)
        if ok is None:
            if self.fp8:
                # the fp8 in-backward update runs wherever the fp8 kernels do
                t_like = x.new_empty((x.shape[0], self.weight.shape[0])) if x.dim() == 2 else x
                ok = dp_linear_mse_fp8_supported(x, self.weight, t_like, self.comm)
            else:
                ok = (x.dim() == 2 and x.dtype == torch.bfloat16 and self.weight.dtype == torch.bfloat16
                      and in_backward_sgd_supported(x, self.weight, self.comm))
            self._opt_ok[key] = ok
        return ok

    def loss(self, x: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
        """Global mean-squared-error loss as a differentiable one-element tensor."""
        opt = self.optimizer if self._in_backward(x) else None
        local = dp_linear_mse(x, self.weight, target, self.comm, loss_scale=1.0 / (x.shape[0] * self.comm.size),
                              optimizer=opt, allow_fused=self.fused, fp8=self.fp8)
        return self.comm.Allreduce(local, m4t.MPI_SUM)

    def _local_loss(self, x, target, loss_scale, accumulator):
        return dp_linear_mse(x, self.weight, target, self.comm, loss_scale=loss_scale, allow_fused=self.fused,
                             accumulator=accumulator)

    def train_step(self, x: torch.Tensor, target: torch.Tensor, micro_batches: int = 1) -> torch.Tensor:
        """forward + backward + SGD update through the autograd graph; returns the (global) loss.

        ``micro_batches`` = K > 1: K forwards and backwards over equal chunks of this rank's batch (K must divide it)
        into ``self.accumulator``, then one update; the loss returned is the whole batch's."""
        if micro_batches != 1:
            if self.fp8:
                raise ValueError("mpi4torch_b200: train_step(micro_batches > 1) is not available with fp8=True")
            return accumulated_step(self.comm, self.accumulator, self._local_loss, x, target, micro_batches)
        value = self.loss(x, target)
        value.backward()
        if self.weight.grad is not None:  # the optimizer did not run inside backward
            self.optimizer.invalidate()
            with torch.no_grad():
                self.weight.add_(self.weight.grad, alpha=-self.lr)
            self.weight.grad = None
        return value.detach().reshape(())

    def invalidate_prefetch(self) -> None:
        """Call after modifying ``weight`` by hand (not needed: the version counter is checked)."""
        self.optimizer.invalidate()

    def make_graphed_step(self, x: torch.Tensor, target: torch.Tensor, warmup: int = 3):
        """Capture one training step (forward, backward, update) into a CUDA graph.

        Returns ``(replay, static_x, static_target, loss)``: copy a batch into the static tensors,
        call ``replay()``, read ``loss`` (a device tensor the graph overwrites).  Collective kernels
        are capturable because their flag epochs and staging parity live in device memory; every
        rank must capture and replay the same sequence.  The fused Allreduce->GEMM *forward* kernel
        still takes a host-side step counter, so capture needs either ``fused=False`` or the
        prefetching in-backward optimizer (whose steady-state step contains no fused forward).
        """
        if self.fp8 and self.comm.size > 1:
            raise RuntimeError("graph capture of the fp8 step is available at one rank")
        prefetching = self._in_backward(x) and self.optimizer.prefetch and self.comm.size > 1
        if self.comm.size > 1 and self.fused and not prefetching:
            raise RuntimeError("graph capture needs fused=False or the prefetching in-backward optimizer "
                               "(the fused forward kernel takes a host-side step counter)")
        static_x, static_t = x.clone(), target.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(warmup, 1)):  # allocator warm-up, lazy module loading
                self.train_step(static_x, static_t)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.comm.Barrier()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            loss = self.train_step(static_x, static_t)
        if prefetching:
            # the captured step consumed and re-produced the prefetched average: keep it valid for replays
            self.optimizer.remember(self.weight, self.optimizer._wavg)
        return graph.replay, static_x, static_t, loss
