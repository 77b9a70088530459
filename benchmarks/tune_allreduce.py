#!/usr/bin/env python
"""Parameter sweep for the large-message allreduce (grid size x chunk size),
forward collective only, no autograd.  Prints algorithm bandwidth (GB/s)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi4torch_b200 as m4t  # noqa: E402

comm = m4t.COMM_WORLD
dev = torch.device("cuda", torch.cuda.current_device())
_C = m4t._C


def timeit(fn, iters=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    comm.Barrier()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    t = torch.tensor([a.elapsed_time(b) / iters], dtype=torch.float64)
    return float(comm.Allreduce(t, m4t.MPI_MAX)[0])


sizes = [int(s) for s in os.environ.get("TUNE_SIZES", f"{64 << 20},{256 << 20}").split(",")]
blocks_list = [int(s) for s in os.environ.get("TUNE_BLOCKS", "32,64,128,132,264").split(",")]
chunks = [int(s) for s in os.environ.get("TUNE_CHUNKS_KB", "1024,4096,16384,1048576").split(",")]
algos = [int(s) for s in os.environ.get("TUNE_ALGOS", "3,2").split(",")]
for nbytes in sizes:
    x = torch.randn(nbytes // 2, device=dev, dtype=torch.float32).to(torch.bfloat16)
    for algo in algos:
        if algo == 3 and not m4t.has_nvls():
            continue
        _C.set_tuning("force_algo", algo)
        for blocks in blocks_list:
            for ck in chunks:
                _C.set_tuning("ar_blocks", blocks)
                _C.set_tuning("chunk_bytes", ck * 1024)
                ms = timeit(lambda: comm.Allreduce(x, m4t.MPI_SUM))
                if comm.rank == 0:
                    print(json.dumps({"bytes": nbytes, "algo": algo, "blocks": blocks, "chunk_kb": ck, "ms": round(ms, 4),
                                      "algbw_gbs": round(nbytes / ms / 1e6, 1)}), flush=True)
    _C.set_tuning("force_algo", 0)
