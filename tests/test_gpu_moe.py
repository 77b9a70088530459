"""The batched expert kernels and the ``expert_mlp`` node on one GPU.

Every batched op equals, bit for bit, the existing single-expert op applied to each expert's slice: on random normal
inputs, for E in {1, 3, 8}, at shapes whose total tile count runs from S - 1 to 2S + 1 (S = SM count) with partial
256-wide tiles.  The node's output and five gradients equal the per-expert loop of existing ops, and on exactly
representable inputs the float64 emulation.  Forward and backward launch a fixed set of kernels whatever E is, and
inputs the predicates reject take the composition without launching anything.  ExpertParallelMLP at one rank matches
its composition on a CPU copy."""
import re

import pytest
import torch

from conftest import run_spmd
from test_gpu_exact_arithmetic import _gen, assert_exact_gemm, assert_same_bits, exact_bf16, exact_f32, rne_bf16, ternary
from test_gpu_mlp_exact import gelu_saturated, hidden_layer, output_weights

pytestmark = pytest.mark.gpu


def _m4t():
    import mpi4torch_b200 as m4t

    assert m4t.cuda_backend_ready()
    return m4t


def _ops():
    _m4t()
    return torch.ops.mpi4torch_b200


def _launches():
    return dict(_m4t()._C.kernel_launch_table())


def _sms():
    # collection runs without a GPU too: the H100 SXM's count stands in there
    try:
        return torch.cuda.get_device_properties(0).multi_processor_count
    except Exception:  # no device, or no driver
        return 132


def _shapes():
    """(E, M, N, K).  Forward tiles are E * M / 128 * ceil(N / 256): S - 1, S + 1 and 2S + 1 at E = 1 (with S = 132:
    131, 133 = 7 x 19 and 265 = 53 x 5), 3 x 11 x 4 = 132 at E = 3, and 8 x 2 x 5 = 80 and 8 x 3 x 6 = 144 (half tiles
    at N = 1408) at E = 8."""
    S = _sms()
    return [(1, 128 * (S - 1), 256, 128), (1, 128 * 7, 256 * 19, 128) if S + 1 == 133 else (1, 128 * (S + 1), 256, 128),
            (1, 128 * 53, 1280, 256) if 2 * S + 1 == 265 else (1, 128 * (2 * S + 1), 256, 128),
            (3, 128 * 11, 1024, 256), (8, 256, 1280, 384), (8, 384, 1408, 128)]


def _ids(s):
    return "E{}_M{}_N{}_K{}".format(*s)


def _randn(*shape, dtype=torch.bfloat16, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda", dtype=torch.float32).to(dtype)


@pytest.mark.parametrize("shape", _shapes(), ids=_ids)
def test_batched_forward_ops_bitwise(shape):
    E, M, N, K = shape
    ops = _ops()
    x, w, b = _randn(E, M, K, seed=1), _randn(E, N, K, seed=2), _randn(E, N, dtype=torch.float32, seed=3)
    assert ops.batched_gemm_tn_supported(x, w, b)
    h, z = ops.batched_linear_bias_gelu_forward(x, w, b)
    y = ops.batched_linear_bias_forward(x, w, b)
    for e in range(E):
        h1, z1 = ops.linear_bias_gelu_forward(x[e], w[e], b[e])
        assert_same_bits(h[e], h1, f"{shape} h[{e}]")
        assert_same_bits(z[e], z1, f"{shape} z[{e}]")
        assert_same_bits(y[e], z1, f"{shape} bias-only y[{e}]")


@pytest.mark.parametrize("shape", _shapes(), ids=_ids)
def test_batched_backward_ops_bitwise(shape):
    E, M, N, K = shape
    ops = _ops()
    g = torch.full((1,), 0.375, device="cuda")
    dy, w, z = _randn(E, M, K, seed=4), _randn(E, K, N, seed=5), _randn(E, M, N, seed=6)
    assert ops.batched_gemm_nn_supported(dy, w)
    dz, part = ops.batched_gemm_nn_gelu_backward(dy, w, z, g)
    c = ops.batched_gemm_nn(dy, w)
    db = ops.batched_column_sum(part, g)
    assert tuple(part.shape) == (E, M // 16, N)
    for e in range(E):
        dz1, part1 = ops.gemm_nn_gelu_backward(dy[e], w[e], z[e], g)
        assert_same_bits(dz[e], dz1, f"{shape} dz[{e}]")
        assert_same_bits(part[e], part1, f"{shape} partials[{e}]")
        assert_same_bits(c[e], ops.gemm_bf16_nn(dy[e], w[e]), f"{shape} nn[{e}]")
        assert_same_bits(db[e], ops.column_sum(part1, g), f"{shape} column sum[{e}]")


@pytest.mark.parametrize("shape", _shapes(), ids=_ids)
def test_batched_wgrad_bitwise(shape):
    # the wgrad of [E, M, N] x [E, M, K]: tiles E * N / 128 * ceil(K / 256); the roles of N and K are swapped so that
    # the partial 128-wide last tile of K = 1408 is covered as well
    E, M, K, N = shape
    ops = _ops()
    g = torch.full((1,), 3.0, device="cuda")
    dy, x = _randn(E, M, N, seed=7), _randn(E, M, K, seed=8)
    assert ops.batched_wgrad_bf16_supported(dy, x)
    gw = ops.batched_wgrad_bf16(dy, x, g)
    assert tuple(gw.shape) == (E, N, K)
    for e in range(E):
        assert_same_bits(gw[e], ops.wgrad_bf16(dy[e], x[e], g), f"{shape} wgrad[{e}]")


def _loop_node(x, w1, b1, w2, b2, dy):
    """The node's math as a loop over experts of the existing single-expert ops."""
    ops = _ops()
    out = {k: [] for k in ("y", "gx", "gw1", "gb1", "gw2")}
    for e in range(x.shape[0]):
        h, z = ops.linear_bias_gelu_forward(x[e], w1[e], b1[e])
        out["y"].append(ops.linear_bias_gelu_forward(h, w2[e], b2[e])[1])
        dz, part = ops.gemm_nn_gelu_backward(dy[e], w2[e], z)
        out["gw2"].append(ops.wgrad_bf16(dy[e], h))
        out["gx"].append(ops.gemm_bf16_nn(dz, w1[e]))
        out["gw1"].append(ops.wgrad_bf16(dz, x[e]))
        out["gb1"].append(ops.column_sum(part))
    res = {k: torch.stack(v) for k, v in out.items()}
    res["gb2"] = dy.sum(1, dtype=torch.float32)
    return res


def _node(x, w1, b1, w2, b2, dy):
    from mpi4torch_b200.ops import expert_mlp, expert_mlp_supported

    ins = [t.detach().clone().requires_grad_() for t in (x, w1, b1, w2, b2)]
    assert expert_mlp_supported(*ins)
    y = expert_mlp(*ins)
    y.backward(dy)
    return y.detach(), [t.grad for t in ins]


NODE_SHAPES = [(1, 128, 128, 256, 128), (3, 256, 256, 384, 128), (8, 256, 128, 512, 256)]  # E, M, D, H, O


@pytest.mark.parametrize("shape", NODE_SHAPES, ids=lambda s: "E{}_M{}_D{}_H{}_O{}".format(*s))
def test_node_matches_loop_of_existing_ops(shape):
    E, M, D, H, O = shape
    x, w1, w2 = _randn(E, M, D, seed=11), _randn(E, H, D, seed=12) * 0.1, _randn(E, O, H, seed=13) * 0.1
    b1, b2 = _randn(E, H, dtype=torch.float32, seed=14), _randn(E, O, dtype=torch.float32, seed=15)
    dy = _randn(E, M, O, seed=16) * 3  # an upstream gradient other than ones
    y, grads = _node(x, w1, b1, w2, b2, dy)
    want = _loop_node(x, w1, b1, w2, b2, dy)
    assert_same_bits(y, want["y"], f"{shape} y")
    for name, got in zip(("gx", "gw1", "gb1", "gw2", "gb2"), grads):
        assert_same_bits(got, want[name], f"{shape} {name}")


def _emulate_expert(x, w1, b1, w2, b2, dy, what):
    """One expert in float64, rounding where the kernels round (the premises of each GEMM asserted)."""
    M = x.shape[0]
    r = lambda v: rne_bf16(v).double()  # noqa: E731
    assert_exact_gemm(x, w1.t(), b1.expand(M, -1), what=f"{what} z")
    z = r(x @ w1.t() + b1)
    h, gp = gelu_saturated(z, what)
    assert_exact_gemm(h, w2.t(), b2.expand(M, -1), what=f"{what} y")
    assert_exact_gemm(dy, w2, what=f"{what} dz")
    dz32 = (dy @ w2) * gp
    dz = r(dz32)
    ones = torch.ones(1, M, dtype=x.dtype, device=x.device)
    assert_exact_gemm(ones, dz32, what=f"{what} gb1")
    for a, b, n in ((dz, w1, "gx"), (dz.t(), x, "gw1"), (dy.t(), h, "gw2")):
        assert_exact_gemm(a, b, what=f"{what} {n}")
    return {"y": r(h @ w2.t() + b2), "gx": r(dz @ w1), "gw1": r(dz.t() @ x), "gb1": dz32.sum(0), "gw2": r(dy.t() @ h),
            "gb2": dy.sum(0)}


def test_node_matches_float64_emulation_on_exact_inputs():
    E, M, D, H, O = 3, 256, 128, 256, 128
    cols = {k: [] for k in ("x", "w1", "b1", "w2", "b2", "dy")}
    for e in range(E):
        gen = _gen(E, M, D, H, O, e)
        x, w1, b1, kind = hidden_layer(M, D, H, gen)
        cols["x"].append(x), cols["w1"].append(w1), cols["b1"].append(b1)
        cols["w2"].append(output_weights(O, kind, gen, 2.0))
        cols["b2"].append(ternary((O,), 0.5, gen, 2.0 ** -4))
        cols["dy"].append(ternary((M, O), 0.25, gen, 2.0 ** -3))
    t = {k: torch.stack(v) for k, v in cols.items()}
    want = [_emulate_expert(*(t[k][e] for k in ("x", "w1", "b1", "w2", "b2", "dy")), what=f"expert {e}") for e in range(E)]
    y, grads = _node(exact_bf16(t["x"]), exact_bf16(t["w1"]), exact_f32(t["b1"]), exact_bf16(t["w2"]),
                     exact_f32(t["b2"]), exact_bf16(t["dy"]))
    assert bool((torch.stack([w["gx"] for w in want]) != 0).any()), "the case has no input gradient"
    assert_same_bits(y, exact_bf16(torch.stack([w["y"] for w in want])), "y")
    for name, got in zip(("gx", "gw1", "gb1", "gw2", "gb2"), grads):
        ref = torch.stack([w[name] for w in want])
        assert_same_bits(got, exact_f32(ref) if name.startswith("gb") else exact_bf16(ref), name)


def _node_launches(E, requires=(True,) * 5):
    from mpi4torch_b200.ops import expert_mlp

    M, D, H, O = 128, 128, 256, 128
    ins = [_randn(E, M, D), _randn(E, H, D), _randn(E, H, dtype=torch.float32), _randn(E, O, H),
           _randn(E, O, dtype=torch.float32)]
    ins = [t.requires_grad_(q) for t, q in zip(ins, requires)]
    before = _launches()
    y = expert_mlp(*ins)
    mid = _launches()
    y.backward(_randn(E, M, O))
    after = _launches()
    diff = lambda a, b: {k: b[k] - a.get(k, 0) for k in b if b[k] != a.get(k, 0)}  # noqa: E731
    return diff(before, mid), diff(mid, after)


def test_launches_independent_of_experts():
    fwd = {"gemm_bias_gelu_batched": 1, "gemm_bias_batched": 1}
    bwd = {"gemm_nn_gelu_bwd_colsum_batched": 1, "wgrad_bf16_batched": 2, "gemm_nn_batched": 1,
           "column_sum_batched": 1}
    for E in (1, 3, 8):
        assert _node_launches(E) == (fwd, bwd), E
    # frozen inputs: no gradient and no launch for them
    assert _node_launches(3, (False, False, False, True, True)) == (fwd, {"wgrad_bf16_batched": 1})
    assert _node_launches(3, (True, False, False, False, False))[1] == {"gemm_nn_gelu_bwd_colsum_batched": 1,
                                                                      "gemm_nn_batched": 1}


def _rejected_cases():
    E, M, D, H, O = 2, 128, 128, 256, 128
    x, w1, b1, w2, b2 = (_randn(E, M, D), _randn(E, H, D), _randn(E, H, dtype=torch.float32), _randn(E, O, H),
                         _randn(E, O, dtype=torch.float32))
    misaligned = torch.empty(E * H + 1, device="cuda")[1:].view(E, H)
    misaligned.copy_(b1)
    return {
        "M=64": (x[:, :64].contiguous(), w1, b1, w2, b2),
        "strided experts": (_randn(E, 2 * M, D)[:, :M], w1, b1, w2, b2),
        "strided weights": (x, _randn(2 * E, H, D)[::2], b1, w2, b2),
        "misaligned bias": (x, w1, misaligned, w2, b2),
        "fp32 x": (x.float(), w1, b1, w2, b2),
    }


@pytest.mark.parametrize("case", ["M=64", "strided experts", "strided weights", "misaligned bias", "fp32 x"])
def test_rejected_inputs_take_the_composition_and_launch_nothing(case):
    from mpi4torch_b200.ops import expert_mlp, expert_mlp_supported

    ins = [t.detach().requires_grad_() for t in _rejected_cases()[case]]
    assert not expert_mlp_supported(*ins)
    before = _m4t()._C.kernel_launch_count()
    y = expert_mlp(*ins)
    y.float().sum().backward()
    torch.cuda.synchronize()
    assert _m4t()._C.kernel_launch_count() == before, case
    # the composition's value, in fp32
    x, w1, b1, w2, b2 = (t.detach().float() for t in ins)
    ref = torch.baddbmm(b2[:, None], torch.nn.functional.gelu(torch.baddbmm(b1[:, None], x, w1.transpose(1, 2)),
                                                             approximate="tanh"), w2.transpose(1, 2))
    torch.testing.assert_close(y.float(), ref.to(y.dtype).float(), rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("top_k", [1, 2])
def test_expert_parallel_layer_matches_composition(top_k):
    from mpi4torch_b200.parallel import ExpertParallelMLP

    m4t = _m4t()
    layer = ExpertParallelMLP(256, 512, 4, 128, m4t.COMM_WORLD, top_k=top_k, device="cuda", seed=5)
    # the same parameters on the CPU, where the experts run the composition
    cpu = ExpertParallelMLP(256, 512, 4, 128, m4t.COMM_WORLD, top_k=top_k, device="cpu", seed=5)
    x = _randn(384, 256, seed=21)
    r = _randn(384, 256, dtype=torch.float32, seed=22)
    xg, xc = x.clone().requires_grad_(), x.cpu().requires_grad_()
    before = _launches()
    out, info = layer(xg)
    (out.float() * r).sum().backward()
    assert _launches().get("gemm_bias_gelu_batched", 0) == before.get("gemm_bias_gelu_batched", 0) + 1
    out_c, info_c = cpu(xc)
    (out_c.float() * r.cpu()).sum().backward()
    assert torch.equal(info.expert.cpu(), info_c.expert), "routing differs"
    assert bool(info.dropped.any()) or top_k == 1
    pairs = [(out, out_c, "out"), (xg.grad, xc.grad, "x.grad")]
    pairs += [(getattr(layer, n).grad, getattr(cpu, n).grad, f"{n}.grad") for n in ("router", "w1", "b1", "w2", "b2")]
    for got, ref, name in pairs:
        got, ref = got.double().cpu(), ref.double()
        err = float((got - ref).abs().max())
        assert err <= 3e-2 * float(ref.abs().max()), f"top_k={top_k} {name}: {err} vs max {float(ref.abs().max())}"


def test_moe_example_trains_on_cuda():
    res = run_spmd(1, ["examples/moe_layer.py", "--device", "cuda", "--steps", "20"], device="cuda", timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    assert "gemm" not in res.stderr
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", res.stdout)]
    assert len(losses) == 20 and losses[-1] < losses[0], losses
