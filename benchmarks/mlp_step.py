#!/usr/bin/env python
"""Training step of the data-parallel two-layer MLP (DPMLPModel: Linear -> GELU(tanh) -> Linear, biases, MSE) on
one GPU, against the eager bf16 composition (two nn.Linear, F.gelu, MSE, loss.backward(), SGD), and each MLP
epilogue kernel against its plain counterpart on the same shape.  One process; the arms are alternated and timed
with device events.  Prints one JSON line.

    python benchmarks/mlp_step.py [--batch 8192 --d 4096 --h 16384 --o 4096 --steps 20 --warmup 5 --reps 3]

``--loss cross_entropy`` times DPMLPClassifier (softmax cross-entropy over O classes) against the eager composition
with ``F.cross_entropy``, ``gemm_bias_xent`` against ``gemm_bf16_tn``, and ``xent_finish`` alone (as the whole
cross-entropy op minus its GEMM), with the bytes xent_finish moves.

``--micro-batches K [K ...]`` (MSE) adds gradient accumulation: the DPMLPModel step with ``train_step(x, t,
micro_batches=K)`` for each K, alternated with the K = 1 in-backward step, the eager composition with K
``backward()`` calls into ``.grad`` and then SGD, and, from a torch.profiler run of its own, ``wgrad_accumulate_``
against ``wgrad_bf16`` and ``wgrad_sgd_`` on the first layer's micro-batch shape, next to the bytes each moves.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi4torch_b200 as m4t  # noqa: E402
from mpi4torch_b200.models import DPMLPClassifier, DPMLPModel  # noqa: E402
from mpi4torch_b200.utils.timing import ClockSampler  # noqa: E402


def time_ms(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def card():
    """Name, power limit and max SM clock, read-only."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                              "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = [s.strip() for s in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit_w": float(power), "max_sm_mhz": float(clock)}
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "max_sm_mhz": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--d", type=int, default=4096)
    ap.add_argument("--h", type=int, default=16384)
    ap.add_argument("--o", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3, help="alternations of the arms; medians are reported")
    ap.add_argument("--loss", choices=("mse", "cross_entropy"), default="mse")
    ap.add_argument("--micro-batches", type=int, nargs="+", default=[],
                    help="gradient-accumulation arms: micro-batches per step (each must divide --batch)")
    args = ap.parse_args()
    if args.micro_batches and args.loss != "mse":
        raise SystemExit("--micro-batches times the MSE model")
    if not torch.cuda.is_available():
        raise SystemExit("mlp_step.py needs a GPU")
    comm = m4t.COMM_WORLD
    if not m4t.cuda_backend_ready():
        raise SystemExit("the native CUDA backend did not initialise")
    B, D, H, O = args.batch, args.d, args.h, args.o
    ops = torch.ops.mpi4torch_b200
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, D, device="cuda", generator=g).to(torch.bfloat16)
    t = torch.randn(B, O, device="cuda", generator=g).to(torch.bfloat16)
    lr = 1e-4

    xent = args.loss == "cross_entropy"
    if xent:
        t = torch.randint(0, O, (B,), device="cuda", generator=g)
        model = DPMLPClassifier(D, H, O, comm, device="cuda", lr=lr, seed=0)
    else:
        model = DPMLPModel(D, H, O, comm, device="cuda", lr=lr, seed=0)
    if not model._in_backward(x, t):
        raise SystemExit(f"shape {(B, D, H, O)} is off the MLP kernel path")

    lin1 = torch.nn.Linear(D, H, device="cuda", dtype=torch.bfloat16)
    lin2 = torch.nn.Linear(H, O, device="cuda", dtype=torch.bfloat16)
    eager_params = list(lin1.parameters()) + list(lin2.parameters())

    def eager_step(K=1):
        for xc, tc in zip(x.split(B // K), t.split(B // K)):  # K backward() calls add into .grad
            y = lin2(F.gelu(lin1(xc), approximate="tanh"))
            loss = F.cross_entropy(y.float(), tc) if xent else (y.float() - tc.float()).square().mean()
            (loss if K == 1 else loss / K).backward()
        with torch.no_grad():
            grads = [p.grad for p in eager_params]
            torch._foreach_add_(eager_params, grads, alpha=-lr)
        for p in eager_params:
            p.grad = None

    # each MLP kernel and its plain counterpart on the same shape
    w1, b1 = model.w1.detach(), model.b1.detach()
    w2, b2 = model.w2.detach(), model.b2.detach()
    h, z = ops.linear_bias_gelu_forward(x, w1, b1)
    if xent:
        dy, _, _ = ops.linear_bias_xent_forward_local(h, w2, b2, t, 1.0 / B, 1.0 / B)
        # the whole op (gemm_bias_xent, then xent_finish) against the plain GEMM; xent_kernel_times splits it
        out_pair = {"gemm_bias_xent+xent_finish": (lambda: ops.linear_bias_xent_forward_local(h, w2, b2, t, 1.0 / B, 1.0 / B),
                                                   lambda: ops.gemm_bf16_tn(h, w2))}
    else:
        dy, _, _ = ops.linear_bias_mse_forward_local(h, w2, b2, t, 1.0 / B, 2.0 / B)
        out_pair = {"gemm_bias_mse_colsum": (lambda: ops.linear_bias_mse_forward_local(h, w2, b2, t, 1.0 / B, 2.0 / B),
                                             lambda: ops.linear_mse_forward_local(h, w2, t, 1.0 / B, 2.0 / B))}
    pairs = {
        "gemm_bias_gelu": (lambda: ops.linear_bias_gelu_forward(x, w1, b1), lambda: ops.gemm_bf16_tn(x, w1)),
        **out_pair,
        "gemm_nn_gelu_bwd_colsum": (lambda: ops.gemm_nn_gelu_backward(dy, w2, z), lambda: ops.gemm_bf16_nn(dy, w2)),
    }

    arms = {"model": lambda: model.train_step(x, t), "eager": eager_step}
    for name, (new, plain) in pairs.items():
        arms[name] = new
        arms[name + ":plain"] = plain
    for K in args.micro_batches:
        arms[f"model_k{K}"] = lambda K=K: model.train_step(x, t, micro_batches=K)
        arms[f"eager_k{K}"] = lambda K=K: eager_step(K)
    if xent:  # the MSE step of the same shape, alternated with the others
        mse_model = DPMLPModel(D, H, O, comm, device="cuda", lr=lr, seed=0)
        t_mse = torch.randn(B, O, device="cuda", generator=g).to(torch.bfloat16)
        arms["mse_model"] = lambda: mse_model.train_step(x, t_mse)
    for fn in arms.values():  # warm every shape: module loading, allocator, cuBLAS heuristics
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()

    table0 = dict(m4t._C.kernel_launch_table())
    time_ms(arms["model"], 1)
    kernels_per_step = {k: v - table0.get(k, 0) for k, v in dict(m4t._C.kernel_launch_table()).items()
                        if v - table0.get(k, 0) > 0}

    sampler = ClockSampler(gpu_index=torch.cuda.current_device()).start()
    samples = {k: [] for k in arms}
    for _ in range(args.reps):
        for name, fn in arms.items():
            samples[name].append(time_ms(fn, args.steps))
    clocks = sampler.stop()
    ms = {k: statistics.median(v) for k, v in samples.items()}

    gemm_flop = 2.0 * B * (2 * H * D + 3 * H * O)  # fwd1 + wgrad1 over H*D, fwd2 + dgrad2 + wgrad2 over H*O
    res = {
        "shape": {"B": B, "D": D, "H": H, "O": O},
        "model_ms_per_step": round(ms["model"], 4),
        "model_tflops": round(gemm_flop / ms["model"] / 1e9, 1),
        "eager_ms_per_step": round(ms["eager"], 4),
        "eager_tflops": round(gemm_flop / ms["eager"] / 1e9, 1),
        "kernels": {name: {"ms": round(ms[name], 4), "plain_ms": round(ms[name + ":plain"], 4),
                           "overhead": round(ms[name] / ms[name + ":plain"] - 1.0, 4)} for name in pairs},
        "kernels_per_step": kernels_per_step,
        "spread_ms": {k: [round(min(v), 4), round(max(v), 4)] for k, v in samples.items()},
        "sm_mhz_median": clocks.get("sm_mhz"),
        "throttle_reasons": clocks.get("reasons"),
        **card(),
    }
    if args.micro_batches:
        res["micro_batches"] = {
            K: {"model_ms_per_step": round(ms[f"model_k{K}"], 4), "eager_ms_per_step": round(ms[f"eager_k{K}"], 4),
                "vs_k1_in_backward": round(ms[f"model_k{K}"] / ms["model"] - 1.0, 4)} for K in args.micro_batches}
        Bc = B // max(args.micro_batches)
        dz = torch.randn(Bc, H, device="cuda", generator=g).to(torch.bfloat16)
        res["wgrad_kernels"] = wgrad_kernel_times(ops, dz, x[:Bc], args.steps * args.reps)
    if xent:
        res["loss"] = "cross_entropy"
        res["mse_model_ms_per_step"] = round(ms["mse_model"], 4)
        res["step_overhead_vs_mse"] = round(ms["model"] / ms["mse_model"] - 1.0, 4)
        res["xent_kernels"] = xent_kernel_times(ops, h, w2, b2, t, B, args.steps * args.reps)
    print(json.dumps(res), flush=True)


def wgrad_kernel_times(ops, dy, x, calls):
    """Device time per launch of wgrad_accumulate_, wgrad_bf16 and wgrad_sgd_ for G [N, K] = dy[Mb, N]^T x[Mb, K], each
    in a torch.profiler run of its own (the plain and SGD ops are one kernel instantiation), and the bytes each
    epilogue moves: 8 N K for the fp32 read-modify-write, 2 N K for the bf16 store, 4 N K for the SGD's bf16
    read-modify-write."""
    from torch.profiler import ProfilerActivity, profile

    N, K = dy.shape[1], x.shape[1]
    acc = torch.zeros(N, K, device="cuda")
    w = torch.zeros(N, K, device="cuda", dtype=torch.bfloat16)
    gs = torch.ones(1, device="cuda")
    runs = {"wgrad_accumulate": (lambda: ops.wgrad_accumulate_(acc, dy, x, gs), 8),
            "wgrad_bf16": (lambda: ops.wgrad_bf16(dy, x, gs), 2),
            "wgrad_sgd": (lambda: ops.wgrad_sgd_(w, dy, x, -1e-30, gs), 4)}
    out = {"shape": {"Mb": dy.shape[0], "N": N, "K": K}}
    for name, (fn, bytes_per_elem) in runs.items():
        fn()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                fn()
            torch.cuda.synchronize()
        ev = [e for e in prof.key_averages() if "wgrad_bf16_wgmma_kernel" in e.key and e.count >= calls]
        moved = bytes_per_elem * N * K
        entry = {"epilogue_bytes": moved}
        if len(ev) == 1:
            t_ms = ev[0].device_time_total / ev[0].count / 1e3
            entry.update(ms=round(t_ms, 4), epilogue_gb_per_s=round(moved / t_ms / 1e6, 1))
        out[name] = entry
    return out


def xent_kernel_times(ops, h, w2, b2, labels, B, calls):
    """Device time per launch of gemm_bias_xent, xent_finish and gemm_bf16_tn on the output layer's shape, from a
    torch.profiler run of its own (after the event-timed arms), and the bytes xent_finish moves."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            ops.linear_bias_xent_forward_local(h, w2, b2, labels, 1.0 / B, 1.0 / B)
            ops.gemm_bf16_tn(h, w2)
        torch.cuda.synchronize()
    want = {"gemm_bias_xent": "gemm_bf16_wgmma_kernel<false, 5, false>", "xent_finish": "xent_finish_kernel",
            "gemm_bf16_tn": "gemm_bf16_wgmma_kernel<false, 0, false>"}
    times = {}
    for ev in prof.key_averages():
        for key, pattern in want.items():
            if pattern in ev.key and ev.count >= calls:
                times[key] = round(ev.device_time_total / ev.count / 1e3, 4)  # ms per launch
    M, C = h.shape[0], w2.shape[0]
    tiles = (C + 255) // 256
    # logits read + dy written (bf16), column-sum partials written, tile pairs and labels read, row losses
    moved = 2 * M * C * 2 + (M + 15) // 16 * C * 4 + tiles * M * 8 + M * 8 + 2 * M * 4
    out = {"ms": times, "xent_finish_bytes": moved}
    if "xent_finish" in times:
        out["xent_finish_gb_per_s"] = round(moved / times["xent_finish"] / 1e6, 1)
    if "gemm_bias_xent" in times and "gemm_bf16_tn" in times:
        out["gemm_bias_xent_overhead"] = round(times["gemm_bias_xent"] / times["gemm_bf16_tn"] - 1.0, 4)
    return out


if __name__ == "__main__":
    main()
