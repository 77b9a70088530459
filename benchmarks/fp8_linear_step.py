#!/usr/bin/env python
"""Training step of the data-parallel linear layer (DPLinearModel, in-backward SGD) with fp8 GEMMs against the bf16
step, on one GPU.  One process; prints one JSON line.

    python benchmarks/fp8_linear_step.py [--batch 8192 --d 4096 --o 4096 --steps 200 --warmup 200 --reps 8]

* step time: the two models alternated in ABBA order (bf16, fp8, fp8, bf16, ...), ``--reps`` windows of ``--steps``
  steps per model, timed with device events, after ``--warmup`` steps of each so that the clocks have settled.  Both
  arms report min / median / max; ``fp8_minus_bf16_ms`` is the median and range of the differences of adjacent windows,
  which cancels the drift of the card's clocks that the two medians alone still carry;
* from a torch.profiler run of its own: the device time of every kernel of one step of each model, ``gemm_fp8_tn``
  against ``gemm_bf16_tn`` and ``torch._scaled_mm`` on the forward shape, and the quantize kernels' bandwidth from the
  bytes their shapes imply;
* the loss of both models after ``--loss-steps`` steps on the same synthetic regression.
"""
import argparse
import json
import os
import statistics
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi4torch_b200 as m4t  # noqa: E402
from benchmarks.mlp_step import card, time_ms  # noqa: E402
from mpi4torch_b200.models import DPLinearModel  # noqa: E402


def kernel_times(fn, iters, out_dir, tag):
    """{kernel name: mean device ms per call of fn} from a profiler run of `iters` calls."""
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, f"fp8_linear_{tag}.json"))
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "device_time_total", 0) > 0:
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t > 0:
                out[e.key] = t / 1000.0 / iters
    return out


def short(name):
    for key in ("gemm_fp8_kernel<1", "gemm_fp8_kernel<2", "gemm_fp8_kernel<0", "quantize_fp8_amax", "quantize_fp8_cast",
                "gemm_bf16_wgmma_kernel", "wgrad_bf16_wgmma_kernel", "allreduce", "local_epilogue"):
        if key in name:
            return {"gemm_fp8_kernel<1": "gemm_fp8_mse", "gemm_fp8_kernel<2": "gemm_fp8_sgd",
                    "gemm_fp8_kernel<0": "gemm_fp8_tn"}.get(key, key)
    return name[:60]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--d", type=int, default=4096)
    ap.add_argument("--o", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--reps", type=int, default=8)
    ap.add_argument("--loss-steps", type=int, default=100)
    ap.add_argument("--out", default=None, help="directory for the profiler traces")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_linear_step.py measures on the GPU; none is visible")
    comm = m4t.COMM_WORLD
    assert comm.size == 1 and m4t.cuda_backend_ready()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    B, D, O = a.batch, a.d, a.o
    res = {"card": card(), "shape": [B, D, O]}
    g = torch.Generator(device="cuda").manual_seed(0)
    teacher = torch.randn(O, D, device="cuda", generator=g) * D ** -0.5
    x = torch.randn(B, D, device="cuda", generator=g)
    t = (x @ teacher.t()).to(torch.bfloat16)
    x = x.to(torch.bfloat16)
    models = {"bf16": DPLinearModel(D, O, comm, lr=1e-3, seed=0),
              "fp8": DPLinearModel(D, O, comm, lr=1e-3, seed=0, fp8=True)}

    # ---- step time, alternated
    for m in models.values():
        for _ in range(a.warmup):
            m.train_step(x, t)
    torch.cuda.synchronize()
    times = {k: [] for k in models}
    diffs = []
    for r in range(a.reps):
        order = ("bf16", "fp8") if r % 2 == 0 else ("fp8", "bf16")
        pair = {k: time_ms(lambda m=models[k]: m.train_step(x, t), a.steps) for k in order}
        for k, v in pair.items():
            times[k].append(v)
        diffs.append(pair["fp8"] - pair["bf16"])
    res["step_ms"] = {k: {"min": min(v), "median": statistics.median(v), "max": max(v), "all": [round(u, 4) for u in v]}
                      for k, v in times.items()}
    res["fp8_minus_bf16_ms"] = {"median": statistics.median(diffs), "min": min(diffs), "max": max(diffs)}

    # ---- per-kernel times of one step
    for k, m in models.items():
        kt = kernel_times(lambda m=m: m.train_step(x, t), 20, a.out, k)
        merged = {}
        for name, ms in kt.items():
            merged[short(name)] = merged.get(short(name), 0.0) + ms
        res[f"kernels_ms_{k}"] = {n: round(v, 4) for n, v in sorted(merged.items(), key=lambda kv: -kv[1])}

    # ---- GEMM against GEMM on the forward shape, and the quantize kernels' bandwidth
    ops = torch.ops.mpi4torch_b200
    w = models["bf16"].weight.detach()
    xq, _, sx = ops.quantize_fp8(x, "e4m3", True, False)
    wq, _, sw = ops.quantize_fp8(w, "e4m3", True, False)
    calls = {
        "gemm_fp8_tn": lambda: ops.gemm_fp8_tn(xq, wq, sx, sw),
        "gemm_bf16_tn": lambda: ops.gemm_bf16_tn(x, w),
        "torch._scaled_mm": lambda: torch._scaled_mm(xq, wq.t(), scale_a=sx, scale_b=sw, out_dtype=torch.bfloat16),
        "quantize_x_both": lambda: ops.quantize_fp8(x, "e4m3", True, True),
    }
    flops = 2.0 * B * D * O
    gemm = {}
    for name, fn in calls.items():
        kt = kernel_times(fn, 50, None, name)
        gemm[name] = {short(n): round(v, 4) for n, v in kt.items()}
    for name in ("gemm_fp8_tn", "gemm_bf16_tn", "torch._scaled_mm"):
        ms = sum(gemm[name].values())
        gemm[name]["tflops"] = round(flops / (ms * 1e-3) / 1e12, 1)
    q = gemm["quantize_x_both"]
    # amax reads x (2 B/element); the cast reads x and writes q and q^T (1 B each)
    amax_ms, cast_ms = q.get("quantize_fp8_amax", 0.0), q.get("quantize_fp8_cast", 0.0)
    q["amax_gbps"] = round(2.0 * B * D / (amax_ms * 1e-3) / 1e9, 1) if amax_ms else None
    q["cast_gbps"] = round(4.0 * B * D / (cast_ms * 1e-3) / 1e9, 1) if cast_ms else None
    res["ops_ms"] = gemm

    # ---- loss after N steps on the same regression, from the same initial weights
    losses = {}
    for k, fp8 in (("bf16", False), ("fp8", True)):
        m = DPLinearModel(D, O, comm, lr=0.5, seed=1, fp8=fp8)
        gen = torch.Generator(device="cuda").manual_seed(5)
        first = last = None
        for i in range(a.loss_steps):
            xb = torch.randn(B, D, device="cuda", generator=gen)
            lv = m.train_step(xb.to(torch.bfloat16), (xb @ teacher.t()).to(torch.bfloat16))
            if i == 0:
                first = float(lv)
        last = float(lv)
        losses[k] = {"first": first, "last": last}
    res["loss_after_steps"] = {"steps": a.loss_steps, **losses}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
