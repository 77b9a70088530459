"""Forward + backward of the experts of a mixture-of-experts layer (``expert_mlp``) at one rank, three arms:

* ``batched``: the ``expert_mlp`` node, one launch per GEMM for all E experts;
* ``loop``: the same math with the same bits as a loop over experts of the single-expert ops
  (``linear_bias_gelu_forward``, whose ``z`` output stands in for the bias-only layer, ``gemm_nn_gelu_backward``,
  ``wgrad_bf16``, ``gemm_bf16_nn``, ``column_sum``);
* ``eager``: bf16 ``baddbmm`` / ``F.gelu`` / autograd.

Two shapes: E = 8, M = 256, D = 1024, H = 4096, where one expert's GEMM is a fraction of a wave, and E = 8,
M = 1024, D = 4096, H = 16384, where it is several waves.  Step times come from CUDA events over windows of
``--steps`` calls, the arms alternated, ``--reps`` windows each (min / median / max reported); per-kernel times from
a separate ``torch.profiler`` run; FLOP/s from the shapes (forward 2 E M (D H + H O), backward twice that).  The card
name and power limit are read in the same run.

    python benchmarks/moe_step.py [--shapes small,large] [--out DIR]

With ``--routing uniform|skewed`` it compares instead, on the same E * M routed (token, choice) pairs:

* ``grouped``: the dropless ``grouped_expert_mlp`` node, every expert on exactly its pairs;
* ``batched``: ``expert_mlp`` with the capacity of the largest count (rounded up to 128), so neither arm drops a pair;
* ``grouped_mm``: eager bf16 on ``torch._grouped_mm`` with autograd, where this torch has it.

Uniform routing gives every expert M pairs.  Skewed routing is seeded: expert 0 takes ``--skew`` (default 4) times the
mean load and the others share the rest at random.  FLOP/s count the routed rows only.

    python benchmarks/moe_step.py --routing skewed [--shapes small,large]

With ``--update`` naming more than ``grad`` it compares how the expert parameters are trained, one training step of
the experts each (x requires a gradient too, as in a layer):

* ``grad``: the plain node, bf16 ``.grad`` of the weights, then the torch SGD pass ``p -= lr * p.grad`` it implies;
* ``sgd``: ``optimizer=InBackwardSGD(lr)``, the SGD step in the wgrad kernels' epilogue, no ``.grad``;
* ``accumulate``: ``accumulator=AccumulatedSGD(lr)``, one micro-batch added into the fp32 buffers (its ``step()``,
  once per K micro-batches, is not in the timed window).

It runs the large batched shape and the skewed grouped case (expert 0 at ``--skew`` times the mean load) and reports
the step medians (arms alternated), the per-kernel device times of a separate profiler run and the peak device memory
of one step of each arm.

    python benchmarks/moe_step.py --update grad,sgd,accumulate
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mpi4torch_b200 as m4t  # noqa: E402
from benchmarks.fp8_linear_step import kernel_times  # noqa: E402
from benchmarks.mlp_step import card, time_ms  # noqa: E402
from mpi4torch_b200.ops import (AccumulatedSGD, InBackwardSGD, expert_group_starts, expert_mlp,  # noqa: E402
                                 expert_mlp_supported, grouped_expert_mlp, grouped_expert_mlp_supported)
from mpi4torch_b200.ops.expert_mlp import grouped_rows  # noqa: E402

SHAPES = {"small": (8, 256, 1024, 4096), "large": (8, 1024, 4096, 16384)}  # E, M, D, H (O = D)


def short(name):
    """A kernel's name with its template arguments (the last one of the GEMMs and the column sum is BATCHED)."""
    return name.split("(CU")[0].split("(float")[0].replace("void ", "").replace("m4t::", "").replace(
        "(anonymous namespace)::", "")[:80]


def make_arms(E, M, D, H):
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device="cuda") * scale)  # noqa: E731
    x = r(E, M, D).to(torch.bfloat16)
    w1, w2 = r(E, H, D, scale=D ** -0.5).to(torch.bfloat16), r(E, D, H, scale=H ** -0.5).to(torch.bfloat16)
    b1, b2 = r(E, H, scale=0.1), r(E, D, scale=0.1)
    dy = r(E, M, D).to(torch.bfloat16)
    params = [t.requires_grad_() for t in (x, w1, b1, w2, b2)]
    assert expert_mlp_supported(*params)
    ops = torch.ops.mpi4torch_b200

    def batched():
        y = expert_mlp(*params)
        y.backward(dy)

    def loop():
        for e in range(E):
            xe, w1e, w2e = x.detach()[e], w1.detach()[e], w2.detach()[e]
            h, z = ops.linear_bias_gelu_forward(xe, w1e, b1.detach()[e])
            ops.linear_bias_gelu_forward(h, w2e, b2.detach()[e])
            dz, part = ops.gemm_nn_gelu_backward(dy[e], w2e, z)
            ops.wgrad_bf16(dy[e], h)
            ops.gemm_bf16_nn(dz, w1e)
            ops.wgrad_bf16(dz, xe)
            ops.column_sum(part)
        dy.sum(1, dtype=torch.float32)

    bf = [t.detach().to(torch.bfloat16).requires_grad_() for t in params]

    def eager():
        xe, w1e, b1e, w2e, b2e = bf
        h = F.gelu(torch.baddbmm(b1e.unsqueeze(1), xe, w1e.transpose(1, 2)), approximate="tanh")
        y = torch.baddbmm(b2e.unsqueeze(1), h, w2e.transpose(1, 2))
        y.backward(dy)

    def clear():
        for t in params + bf:
            t.grad = None

    return {"batched": batched, "loop": loop, "eager": eager}, clear


def route_counts(E, M, routing, skew):
    """[E] pair counts summing to E * M: uniform, or expert 0 at skew x the mean and a seeded split of the rest."""
    if routing == "uniform":
        return [M] * E
    g = torch.Generator().manual_seed(7)
    top = int(skew * M)
    rest = torch.multinomial(torch.ones(E - 1), E * M - top, replacement=True, generator=g)
    counts = [top] + torch.bincount(rest, minlength=E - 1).tolist()
    assert max(counts) == top and sum(counts) == E * M
    return counts


def make_routing_arms(E, M, D, H, counts):
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device="cuda") * scale)  # noqa: E731
    w1, w2 = r(E, H, D, scale=D ** -0.5).to(torch.bfloat16), r(E, D, H, scale=H ** -0.5).to(torch.bfloat16)
    b1, b2 = r(E, H, scale=0.1), r(E, D, scale=0.1)
    cnt = torch.tensor(counts, dtype=torch.int32, device="cuda")
    starts = expert_group_starts(cnt).tolist()
    R = grouped_rows(E * M, E)
    xg, dyg = torch.zeros(R, D, device="cuda", dtype=torch.bfloat16), torch.zeros(R, D, device="cuda", dtype=torch.bfloat16)
    C = -(-max(counts) // 128) * 128
    xb, dyb = (torch.zeros(E, C, D, device="cuda", dtype=torch.bfloat16) for _ in range(2))
    xd, dyd = r(E * M, D).to(torch.bfloat16), r(E * M, D).to(torch.bfloat16)  # dense, for torch._grouped_mm
    at = 0
    for e, c in enumerate(counts):
        xg[starts[e]:starts[e] + c], dyg[starts[e]:starts[e] + c] = xd[at:at + c], dyd[at:at + c]
        xb[e, :c], dyb[e, :c] = xd[at:at + c], dyd[at:at + c]
        at += c
    pg = [t.requires_grad_() for t in (xg, w1.clone(), b1.clone(), w2.clone(), b2.clone())]
    pb = [t.requires_grad_() for t in (xb, w1.clone(), b1.clone(), w2.clone(), b2.clone())]
    assert grouped_expert_mlp_supported(pg[0], cnt, *pg[1:]) and expert_mlp_supported(*pb)

    def grouped():
        grouped_expert_mlp(pg[0], cnt, *pg[1:]).backward(dyg)

    def batched():
        expert_mlp(*pb).backward(dyb)

    arms = {"grouped": grouped, "batched": batched}
    pe = [t.detach().clone().requires_grad_() for t in (xd, w1, w2)]
    be = [t.to(torch.bfloat16).requires_grad_() for t in (b1, b2)]
    offs = torch.cumsum(cnt, 0, dtype=torch.int32)
    rows_of = torch.repeat_interleave(torch.arange(E, device="cuda"), cnt.long())
    note = None
    if hasattr(torch, "_grouped_mm"):
        def grouped_mm():
            x, w1e, w2e = pe
            h = F.gelu(torch._grouped_mm(x, w1e.transpose(1, 2), offs=offs) + be[0][rows_of], approximate="tanh")
            y = torch._grouped_mm(h, w2e.transpose(1, 2), offs=offs) + be[1][rows_of]
            y.backward(dyd)
        try:
            grouped_mm()
            torch.cuda.synchronize()
            arms["grouped_mm"] = grouped_mm
        except RuntimeError as err:  # this torch build has no kernel for it here
            note = f"torch._grouped_mm unavailable: {str(err).splitlines()[0][:200]}"
    else:
        note = "torch._grouped_mm is not in this torch"

    def clear():
        for t in pg + pb + pe + be:
            t.grad = None

    return arms, clear, {"capacity_batched": C, "rows_grouped": R, "note": note}


def routing_main(a):
    for tag in a.shapes.split(","):
        E, M, D, H = SHAPES[tag]
        counts = route_counts(E, M, a.routing, a.skew)
        arms, clear, info = make_routing_arms(E, M, D, H, counts)
        res = {"card": card(), "routing": a.routing, "shape": {"E": E, "M_mean": M, "D": D, "H": H, "O": D},
               "counts": counts, "max_over_mean": max(counts) / M, **info}
        for fn in arms.values():
            for _ in range(a.warmup):
                fn()
                clear()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        names = list(arms)
        for rep in range(a.reps):
            for k in (names if rep % 2 == 0 else names[::-1]):
                times[k].append(time_ms(lambda k=k: (arms[k](), clear()), a.steps))
        flops = 3 * 2.0 * E * M * (D * H + H * D)  # routed rows only
        res["step_ms"] = {k: {"min": round(min(v), 4), "median": round(statistics.median(v), 4), "max": round(max(v), 4)}
                          for k, v in times.items()}
        for k in arms:
            kt = kernel_times(lambda k=k: (arms[k](), clear()), 10, None, k)
            total = sum(kt.values())
            res[f"device_ms_{k}"] = round(total, 4)
            res[f"device_tflops_{k}"] = round(flops / (total * 1e-3) / 1e12, 1)
        print(json.dumps(res), flush=True)


UPDATE_LR = 1e-6  # small enough that thousands of timed steps leave the weights' magnitudes unchanged


def make_update_arms(kind, E, M, D, H, counts, modes):
    """One training step of the experts per call, in each update mode of `modes`."""
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device="cuda") * scale)  # noqa: E731
    init = [r(E, H, D, scale=D ** -0.5).to(torch.bfloat16), r(E, H, scale=0.1),
            r(E, D, H, scale=H ** -0.5).to(torch.bfloat16), r(E, D, scale=0.1)]
    if kind == "batched":
        x, dy = r(E, M, D).to(torch.bfloat16), r(E, M, D).to(torch.bfloat16)
        node = lambda xx, ps, **u: expert_mlp(xx, *ps, **u)  # noqa: E731
        assert expert_mlp_supported(x, *init)
    else:
        cnt = torch.tensor(counts, dtype=torch.int32, device="cuda")
        R = grouped_rows(sum(counts), E)
        x, dy = torch.zeros(R, D, device="cuda", dtype=torch.bfloat16), torch.zeros(R, D, device="cuda", dtype=torch.bfloat16)
        for s, c in zip(expert_group_starts(cnt).tolist(), counts):
            x[s:s + c], dy[s:s + c] = r(c, D).to(torch.bfloat16), r(c, D).to(torch.bfloat16)
        node = lambda xx, ps, **u: grouped_expert_mlp(xx, cnt, *ps, **u)  # noqa: E731
        assert grouped_expert_mlp_supported(x, cnt, *init)
    arms = {}
    for mode in modes:
        ps = [t.clone().requires_grad_() for t in init]
        xm = x.clone().requires_grad_()
        update = {"sgd": {"optimizer": InBackwardSGD(UPDATE_LR)},
                  "accumulate": {"accumulator": AccumulatedSGD(UPDATE_LR)}}.get(mode, {})

        def step(ps=ps, xm=xm, update=update, mode=mode):
            node(xm, ps, **update).backward(dy)
            xm.grad = None
            if mode == "grad":
                with torch.no_grad():
                    for p in ps:
                        p.add_(p.grad, alpha=-UPDATE_LR)
                        p.grad = None

        arms[mode] = step
    return arms


def update_main(a, modes):
    skewed = route_counts(*SHAPES["large"][:2], "skewed", a.skew)
    for kind, counts in (("batched", None), ("grouped", skewed)):
        E, M, D, H = SHAPES["large"]
        res = {"card": card(), "update": kind, "shape": {"E": E, "M": M, "D": D, "H": H, "O": D}, "lr": UPDATE_LR}
        if counts:
            res["counts"] = counts
        arms = make_update_arms(kind, E, M, D, H, counts, modes)
        peak = {}
        for k, fn in arms.items():  # one step each, measured alone, after the first (the buffers are allocated)
            fn()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            peak[k] = {"peak_mib": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1),
                       "peak_above_resident_mib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)}
        for fn in arms.values():
            for _ in range(a.warmup):
                fn()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        names = list(arms)
        for rep in range(a.reps):
            for k in (names if rep % 2 == 0 else names[::-1]):
                times[k].append(time_ms(arms[k], a.steps))
        res["step_ms"] = {k: {"min": round(min(v), 4), "median": round(statistics.median(v), 4), "max": round(max(v), 4)}
                          for k, v in times.items()}
        res["memory"] = peak
        for k in arms:
            kt = kernel_times(arms[k], 10, None, k)
            merged = {}
            for name, ms in kt.items():
                merged[short(name)] = merged.get(short(name), 0.0) + ms
            res[f"kernels_ms_{k}"] = {n: round(v, 4) for n, v in sorted(merged.items(), key=lambda kv: -kv[1])}
            res[f"device_ms_{k}"] = round(sum(merged.values()), 4)
        print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="small,large")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--out", default=None, help="directory for the profiler traces")
    ap.add_argument("--routing", choices=("uniform", "skewed"), default=None,
                    help="compare the grouped (dropless) node with the batched one under this routing")
    ap.add_argument("--skew", type=float, default=4.0, help="skewed routing: max / mean load")
    ap.add_argument("--update", default="grad",
                    help="comma-separated update modes from grad, sgd, accumulate; grad alone: the comparison above")
    a = ap.parse_args()
    modes = a.update.split(",")
    if not set(modes) <= {"grad", "sgd", "accumulate"}:
        raise SystemExit("--update takes grad, sgd and accumulate")
    if not torch.cuda.is_available():
        raise SystemExit("moe_step.py measures on the GPU; none is visible")
    assert m4t.COMM_WORLD.size == 1 and m4t.cuda_backend_ready()
    if modes != ["grad"]:
        update_main(a, modes)
        return
    if a.routing:
        routing_main(a)
        return
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    for tag in a.shapes.split(","):
        E, M, D, H = SHAPES[tag]
        arms, clear = make_arms(E, M, D, H)
        res = {"card": card(), "shape": {"E": E, "M": M, "D": D, "H": H, "O": D}}
        for fn in arms.values():
            for _ in range(a.warmup):
                fn()
                clear()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        names = list(arms)
        for rep in range(a.reps):
            order = names if rep % 2 == 0 else names[::-1]
            for k in order:
                times[k].append(time_ms(lambda k=k: (arms[k](), clear()), a.steps))
        flops = 3 * 2.0 * E * M * (D * H + H * D)
        res["step_ms"] = {k: {"min": round(min(v), 4), "median": round(statistics.median(v), 4), "max": round(max(v), 4),
                              "tflops_at_median": round(flops / (statistics.median(v) * 1e-3) / 1e12, 1)}
                          for k, v in times.items()}
        for k in ("batched", "loop"):
            kt = kernel_times(lambda k=k: (arms[k](), clear()), 10, None, k)
            merged = {}
            for name, ms in kt.items():
                merged[short(name)] = merged.get(short(name), 0.0) + ms
            total = sum(merged.values())
            res[f"kernels_ms_{k}"] = {n: round(v, 4) for n, v in sorted(merged.items(), key=lambda kv: -kv[1])}
            res[f"device_ms_{k}"] = round(total, 4)
            res[f"device_tflops_{k}"] = round(flops / (total * 1e-3) / 1e12, 1)
        res["launches_per_step"] = {"batched": 7, "loop": 7 * E}
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
