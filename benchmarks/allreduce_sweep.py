#!/usr/bin/env python
"""Allreduce forward+backward bus-bandwidth sweep, 1 KiB .. 1 GiB bf16
(BASELINE.json config 2), ours next to the comparators BASELINE.md names:

  ours     hand-written sm_90a kernels over the symmetric heap (this library)
  nccl     NCCL through torch.distributed, wrapped in the same autograd adjoint
  staged   host-staged: D2H -> CPU shared-memory reduce -> H2D  (what the
           reference does without a CUDA-aware MPI, csrc/extension.cpp:75-89)

Run under the launcher or torchrun:
    python -m mpi4torch_b200.launch -np 8 benchmarks/allreduce_sweep.py [--full] [--raw]
Every number is CUDA-event timed on the launching stream and the max over ranks.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import mpi4torch_b200 as m4t  # noqa: E402
from benchmarks.extras import FULL_SIZES, QUICK_SIZES, _time_fwd_bwd, busbw_gbs, ours_fwd_bwd  # noqa: E402


class _NcclAllreduce(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        import torch.distributed as dist

        y = x.clone()
        dist.all_reduce(y)
        return y

    @staticmethod
    def backward(ctx, g):
        import torch.distributed as dist

        g = g.clone()
        dist.all_reduce(g)
        return g


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--full", action="store_true")
    ap.add_argument("--no-nccl", action="store_true")
    ap.add_argument("--no-staged", action="store_true")
    ap.add_argument("--raw", action="store_true", help="also time the bare forward collective (no autograd)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    comm = m4t.COMM_WORLD
    P, R = comm.size, comm.rank
    dev = torch.device("cuda", torch.cuda.current_device())
    sizes = FULL_SIZES if args.full else QUICK_SIZES
    use_nccl = not args.no_nccl and P > 1
    if use_nccl:
        import torch.distributed as dist

        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{os.environ['MASTER_PORT']}", rank=R,
                                world_size=P, device_id=dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = []
    for nbytes in sizes:
        n = nbytes // 2
        x = torch.randn(n, device=dev, dtype=torch.float32).to(torch.bfloat16).requires_grad_()
        g = torch.ones(n, device=dev, dtype=torch.bfloat16)
        iters = 20 if nbytes <= (1 << 24) else 5
        fl = flush if nbytes <= (128 << 20) else None
        row = {"bytes": nbytes}
        ms = _time_fwd_bwd(lambda: ours_fwd_bwd(comm, x, g), iters, 3, comm, fl)
        row["ours_ms"] = ms
        row["ours_busbw"] = busbw_gbs(nbytes, ms, P)
        if args.raw:
            xr = x.detach()

            def raw():
                comm.Allreduce(xr, m4t.MPI_SUM)

            ms = _time_fwd_bwd(lambda: raw, iters, 3, comm, fl)
            row["ours_fwd_only_ms"] = ms
        if use_nccl:
            def nccl():
                x.grad = None
                _NcclAllreduce.apply(x).backward(g)

            ms = _time_fwd_bwd(lambda: nccl, iters, 3, comm, fl)
            row["nccl_ms"] = ms
            row["nccl_busbw"] = busbw_gbs(nbytes, ms, P)
            if args.raw:
                import torch.distributed as dist

                buf = x.detach().clone()
                ms = _time_fwd_bwd(lambda: (lambda: dist.all_reduce(buf)), iters, 3, comm, fl)
                row["nccl_fwd_only_ms"] = ms
        if not args.no_staged and nbytes <= (1 << 26):
            m4t.deactivate_cuda_aware_mpi_support()
            try:
                ms = _time_fwd_bwd(lambda: ours_fwd_bwd(comm, x, g), max(2, iters // 4), 1, comm, None)
            finally:
                m4t.activate_nvlink_transport()
            row["staged_ms"] = ms
            row["staged_busbw"] = busbw_gbs(nbytes, ms, P)
        rows.append(row)
        if R == 0:
            print(json.dumps(row), flush=True)
        del x, g
    if R == 0 and args.out:
        with open(args.out, "w") as f:
            json.dump({"world": P, "heap_mode": m4t.heap_mode(), "nvls": m4t.has_nvls(), "rows": rows}, f, indent=1)
    if use_nccl:
        import torch.distributed as dist

        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
