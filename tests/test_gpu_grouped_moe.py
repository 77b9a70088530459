"""The grouped (dropless) expert kernels and the ``grouped_expert_mlp`` node on one GPU.

Every grouped op equals, bit for bit, the existing single-expert op on each group's valid rows, and writes zero in
every other row, for count patterns with empty groups, one-row groups, groups of 127 / 128 / 129 rows, everything in
one group and groups whose tiles straddle a wave.  Padding rows hold NaN in every input, so a kernel that let one
reach a valid output or a weight gradient fails.  With uniform counts the node equals the batched node; on exactly
representable inputs it equals the float64 emulation.  Forward and backward read no count on the host and launch a
fixed set of kernels whatever E and the counts are."""
import pytest
import torch

from test_gpu_exact_arithmetic import _gen, assert_same_bits, exact_bf16, exact_f32, ternary
from test_gpu_mlp_exact import hidden_layer, output_weights
from test_gpu_moe import _emulate_expert, _launches, _m4t, _ops, _randn, _sms

pytestmark = pytest.mark.gpu


def _starts(counts):
    out, s = [], 0
    for c in counts:
        out.append(s)
        s += 128 * (-(-max(c, 0) // 128))
    return out


def _rows(counts):
    return 128 * (-(-sum(max(c, 0) for c in counts) // 128) + len(counts))


def _cases():
    """name -> counts.  'wave' has more 128-row m-blocks than the GPU has SMs, so one wave of tiles ends inside a
    group."""
    S = _sms()
    return {
        "mixed": [0, 1, 127, 128, 129, 300, 5, 64],
        "one_expert": [0, 700, 0],
        "empty_between": [256, 0, 384],
        "E1": [1000],
        "wave": [128 * (S // 3) + 1, 128 * (S // 3), 128 * (S // 3) + 77],
    }


def _grouped(counts, cols, seed, poison=float("nan")):
    """[R, cols] bf16: random normal rows in every group, `poison` in every other row."""
    R = _rows(counts)
    t = torch.full((R, cols), poison, device="cuda", dtype=torch.bfloat16)
    vals = _randn(R, cols, seed=seed)
    for s, c in zip(_starts(counts), counts):
        t[s:s + c] = vals[s:s + c]
    return t


def _counts(counts):
    return torch.tensor(counts, dtype=torch.int32, device="cuda")


def _padding(counts):
    """Bool [R]: the rows outside every group."""
    pad = torch.ones(_rows(counts), dtype=torch.bool, device="cuda")
    for s, c in zip(_starts(counts), counts):
        pad[s:s + c] = False
    return pad


def _assert_zero_padding(t, counts, what):
    rest = t[_padding(counts)]
    assert bool((rest == 0).all()), f"{what}: {int((rest != 0).sum())} non-zero padding entries"


@pytest.mark.parametrize("case", list(_cases()))
def test_grouped_forward_ops_bitwise(case):
    counts = _cases()[case]
    E, N, K = len(counts), 384, 256
    ops = _ops()
    x, w, b = _grouped(counts, K, 1), _randn(E, N, K, seed=2), _randn(E, N, dtype=torch.float32, seed=3)
    cnt = _counts(counts)
    assert ops.grouped_gemm_tn_supported(x, w, cnt, b)
    h, z = ops.grouped_linear_bias_gelu_forward(x, w, b, cnt)
    y = ops.grouped_linear_bias_forward(x, w, b, cnt)
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if c == 0:
            continue
        h1, z1 = ops.linear_bias_gelu_forward(x[s:s + c], w[e], b[e])
        assert_same_bits(h[s:s + c], h1, f"{case} h[{e}]")
        assert_same_bits(z[s:s + c], z1, f"{case} z[{e}]")
        assert_same_bits(y[s:s + c], z1, f"{case} bias-only y[{e}]")
    for t, n in ((h, "h"), (z, "z"), (y, "y")):
        _assert_zero_padding(t, counts, f"{case} {n}")


@pytest.mark.parametrize("case", list(_cases()))
def test_grouped_backward_ops_bitwise(case):
    counts = _cases()[case]
    E, N, K = len(counts), 384, 256
    ops = _ops()
    dy, w, z = _grouped(counts, K, 4), _randn(E, K, N, seed=5), _grouped(counts, N, 6)
    cnt = _counts(counts)
    assert ops.grouped_gemm_nn_supported(dy, w, cnt)
    dz, part = ops.grouped_gemm_nn_gelu_backward(dy, w, z, cnt)
    c_nn = ops.grouped_gemm_nn(dy, w, cnt)
    db = ops.grouped_column_sum(part, cnt)
    assert tuple(part.shape) == (dy.shape[0] // 16, N) and tuple(db.shape) == (E, N)
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if c == 0:
            assert bool((db[e] == 0).all()), f"{case} column sum of empty group {e}"
            continue
        dz1, part1 = ops.gemm_nn_gelu_backward(dy[s:s + c], w[e], z[s:s + c])
        assert_same_bits(dz[s:s + c], dz1, f"{case} dz[{e}]")
        assert_same_bits(part[s // 16:s // 16 + part1.shape[0]], part1, f"{case} partials[{e}]")
        assert_same_bits(c_nn[s:s + c], ops.gemm_bf16_nn(dy[s:s + c], w[e]), f"{case} nn[{e}]")
        assert_same_bits(db[e], ops.column_sum(part1), f"{case} column sum[{e}]")
    _assert_zero_padding(dz, counts, f"{case} dz")
    _assert_zero_padding(c_nn, counts, f"{case} nn")


@pytest.mark.parametrize("case", list(_cases()))
def test_grouped_wgrad_and_row_sums(case):
    counts = _cases()[case]
    E, N, K = len(counts), 256, 384  # K = 384: a half 128-wide last tile
    ops = _ops()
    g = torch.full((1,), 3.0, device="cuda")
    dy, x, cnt = _grouped(counts, N, 7), _grouped(counts, K, 8), _counts(counts)
    assert ops.grouped_wgrad_bf16_supported(dy, x, cnt)
    gw = ops.grouped_wgrad_bf16(dy, x, cnt, g)
    assert tuple(gw.shape) == (E, N, K)
    sums = [ops.grouped_column_sum(dy, cnt) for _ in range(2)]
    assert torch.equal(sums[0], sums[1]), f"{case}: row sums differ between two runs"
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if c == 0:
            assert bool((gw[e] == 0).all()), f"{case}: empty expert {e} has a non-zero gradient"
            assert bool((sums[0][e] == 0).all())
            continue
        pad = -(-c // 64) * 64
        dy_e = torch.zeros(pad, N, device="cuda", dtype=torch.bfloat16)
        x_e = torch.zeros(pad, K, device="cuda", dtype=torch.bfloat16)
        dy_e[:c], x_e[:c] = dy[s:s + c], x[s:s + c]
        assert_same_bits(gw[e], ops.wgrad_bf16(dy_e, x_e, g), f"{case} wgrad[{e}]")
        ref = dy[s:s + c].double().sum(0)
        err = float((sums[0][e].double() - ref).abs().max())
        assert err <= 1e-5 * float(dy[s:s + c].double().abs().sum(0).max()), f"{case} row sum[{e}] off by {err}"


def test_oversized_counts_stay_inside_the_operands():
    """Counts whose layout needs more rows than R: group 1 keeps the rows up to R, group 2 has none.  The operands sit
    between NaN guard rows, so a read outside them would reach the results."""
    ops = _ops()
    R, N, K, guard = 512, 256, 256, 256
    counts = [300, 5000, 100]
    E = len(counts)
    cnt = _counts(counts)

    def guarded(cols, seed):
        buf = torch.full((R + 2 * guard, cols), float("nan"), device="cuda", dtype=torch.bfloat16)
        buf[guard:guard + R] = _randn(R, cols, seed=seed)
        return buf, buf[guard:guard + R]

    (xb, x), (dyb, dy) = guarded(K, 1), guarded(N, 2)
    xb0, dyb0 = xb.clone(), dyb.clone()
    w, b, wn = _randn(E, N, K, seed=3), _randn(E, N, dtype=torch.float32, seed=4), _randn(E, K, N, seed=5)
    h, z = ops.grouped_linear_bias_gelu_forward(x, w, b, cnt)
    c_nn = ops.grouped_gemm_nn(dy, wn, cnt)
    gw = ops.grouped_wgrad_bf16(dy, x, cnt)
    db = ops.grouped_column_sum(dy, cnt)
    torch.cuda.synchronize()
    assert torch.equal(xb.view(torch.int16), xb0.view(torch.int16)) and torch.equal(dyb.view(torch.int16),
                                                                                   dyb0.view(torch.int16))
    for t in (h, z, c_nn, gw, db):
        assert bool(torch.isfinite(t.float()).all()), "a guard row reached a result"
    spans = [(0, 300), (384, 512)]  # group 1 starts at 384 and is cut at R; group 2 would start past R
    for e, (s, t) in enumerate(spans):
        assert_same_bits(z[s:t], ops.linear_bias_gelu_forward(x[s:t], w[e], b[e])[1], f"z[{e}]")
        assert_same_bits(c_nn[s:t], ops.gemm_bf16_nn(dy[s:t], wn[e]), f"nn[{e}]")
        pad = -(-(t - s) // 64) * 64
        dy_e = torch.zeros(pad, N, device="cuda", dtype=torch.bfloat16)
        x_e = torch.zeros(pad, K, device="cuda", dtype=torch.bfloat16)
        dy_e[:t - s], x_e[:t - s] = dy[s:t], x[s:t]
        assert_same_bits(gw[e], ops.wgrad_bf16(dy_e, x_e), f"wgrad[{e}]")
    assert bool((z[300:384] == 0).all()) and bool((gw[2] == 0).all()) and bool((db[2] == 0).all())


def _node(x, counts, w1, b1, w2, b2, dy):
    from mpi4torch_b200.ops import grouped_expert_mlp, grouped_expert_mlp_supported

    ins = [t.detach().clone().requires_grad_() for t in (x, w1, b1, w2, b2)]
    assert grouped_expert_mlp_supported(ins[0], counts, *ins[1:])
    y = grouped_expert_mlp(ins[0], counts, *ins[1:])
    y.backward(dy)
    return y.detach(), [t.grad for t in ins]


def _weights(E, D, H, O, seed):
    return (_randn(E, H, D, seed=seed) * 0.1, _randn(E, H, dtype=torch.float32, seed=seed + 1),
            _randn(E, O, H, seed=seed + 2) * 0.1, _randn(E, O, dtype=torch.float32, seed=seed + 3))


def test_uniform_counts_match_the_batched_node():
    from test_gpu_moe import _node as batched_node

    E, M, D, H, O = 3, 256, 128, 384, 256
    x = _randn(E, M, D, seed=11)
    w1, b1, w2, b2 = _weights(E, D, H, O, 12)
    dy = _randn(E, M, O, seed=16) * 3
    yb, gb = batched_node(x, w1, b1, w2, b2, dy)
    counts = _counts([M] * E)
    y, g = _node(x.reshape(E * M, D), counts, w1, b1, w2, b2, dy.reshape(E * M, O))
    assert_same_bits(y.reshape(E, M, O), yb, "y")
    assert_same_bits(g[0].reshape(E, M, D), gb[0], "dx")
    assert_same_bits(g[1], gb[1], "dW1")
    assert_same_bits(g[3], gb[3], "dW2")
    for got, ref, name in ((g[2], gb[2], "db1"), (g[4], gb[4], "db2")):
        err = float((got.double() - ref.double()).abs().max())
        assert err <= 1e-5 * max(1.0, float(ref.abs().max())), f"{name} off by {err}"


def test_poisoned_padding_changes_nothing():
    counts = [0, 1, 129, 300]
    E, D, H, O = len(counts), 128, 256, 128
    w1, b1, w2, b2 = _weights(E, D, H, O, 30)
    cnt = _counts(counts)
    clean = _node(_grouped(counts, D, 31, 0.0), cnt, w1, b1, w2, b2, _grouped(counts, O, 32, 0.0))
    nan = _node(_grouped(counts, D, 31), cnt, w1, b1, w2, b2, _grouped(counts, O, 32))
    assert_same_bits(nan[0], clean[0], "y")
    _assert_zero_padding(nan[0], counts, "y")
    _assert_zero_padding(nan[1][0], counts, "dx")
    for a, b, name in zip(nan[1], clean[1], ("dx", "dW1", "db1", "dW2", "db2")):
        assert_same_bits(a, b, name)


def test_node_reads_no_count_on_the_host():
    from mpi4torch_b200.ops import grouped_expert_mlp

    counts = [3, 0, 250]
    E, D, H, O = len(counts), 128, 256, 128
    w1, b1, w2, b2 = (t.requires_grad_() for t in _weights(E, D, H, O, 40))
    x = _grouped(counts, D, 41, 0.0).requires_grad_()
    dy = _grouped(counts, O, 42, 0.0)
    cnt = _counts(counts)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = grouped_expert_mlp(x, cnt, w1, b1, w2, b2)
        y.backward(dy)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert x.grad is not None and w1.grad is not None


def _node_launches(counts, requires=(True,) * 5):
    from mpi4torch_b200.ops import grouped_expert_mlp

    E, D, H, O = len(counts), 128, 256, 128
    ins = [_grouped(counts, D, 50, 0.0), *_weights(E, D, H, O, 51)]
    ins = [t.requires_grad_(q) for t, q in zip(ins, requires)]
    cnt = _counts(counts)
    before = _launches()
    y = grouped_expert_mlp(ins[0], cnt, *ins[1:])
    mid = _launches()
    y.backward(_grouped(counts, O, 55, 0.0))
    after = _launches()
    diff = lambda a, b: {k: b[k] - a.get(k, 0) for k in b if b[k] != a.get(k, 0)}  # noqa: E731
    return diff(before, mid), diff(mid, after)


def test_launches_independent_of_experts_and_counts():
    fwd = {"gemm_bias_gelu_grouped": 1, "gemm_bias_grouped": 1}
    bwd = {"gemm_nn_gelu_bwd_colsum_grouped": 1, "wgrad_bf16_grouped": 2, "gemm_nn_grouped": 1,
           "column_sum_grouped": 1, "row_sum_grouped": 1}
    for counts in ([128], [0, 5, 700], [1] * 8, [0] * 8, [300, 0, 0, 0, 0, 0, 0, 9]):
        assert _node_launches(counts) == (fwd, bwd), counts
    # frozen inputs: no gradient and no launch for them
    assert _node_launches([7, 200], (False, False, False, True, True)) == (fwd, {"wgrad_bf16_grouped": 1,
                                                                                "row_sum_grouped": 1})
    assert _node_launches([7, 200], (True, False, False, False, False))[1] == {"gemm_nn_gelu_bwd_colsum_grouped": 1,
                                                                               "gemm_nn_grouped": 1}


def _rejected_cases():
    counts = [100, 28]
    E, D, H, O = 2, 128, 256, 128
    x = _grouped(counts, D, 60, 0.0)
    w1, b1, w2, b2 = _weights(E, D, H, O, 61)
    cnt = _counts(counts)
    return {
        "R=64": (x[:64].contiguous(), cnt, w1, b1, w2, b2),
        "int64 counts": (x, cnt.long(), w1, b1, w2, b2),
        "strided weights": (x, cnt, _randn(2 * E, H, D)[::2], b1, w2, b2),
        "fp32 x": (x.float(), cnt, w1, b1, w2, b2),
        "D=64": (x[:, :64].contiguous(), cnt, w1[:, :, :64].contiguous(), b1, w2, b2),
    }


@pytest.mark.parametrize("case", ["R=64", "int64 counts", "strided weights", "fp32 x", "D=64"])
def test_rejected_inputs_take_the_composition_and_launch_nothing(case):
    from mpi4torch_b200.ops import grouped_expert_mlp, grouped_expert_mlp_supported

    x, cnt, *ws = _rejected_cases()[case]
    ins = [t.detach().requires_grad_() for t in (x, *ws)]
    assert not grouped_expert_mlp_supported(ins[0], cnt, *ins[1:])
    before = _m4t()._C.kernel_launch_count()
    y = grouped_expert_mlp(ins[0], cnt, *ins[1:])
    y.float().sum().backward()
    torch.cuda.synchronize()
    assert _m4t()._C.kernel_launch_count() == before, case
    x, w1, b1, w2, b2 = (t.detach().float() for t in ins)
    ref = torch.zeros(x.shape[0], w2.shape[1], device="cuda")
    for e, (s, c) in enumerate(zip(_starts(cnt.tolist()), cnt.tolist())):
        c = max(0, min(s + c, x.shape[0]) - min(s, x.shape[0]))
        if c:
            hid = torch.nn.functional.gelu(x[s:s + c] @ w1[e].t() + b1[e], approximate="tanh")
            ref[s:s + c] = hid @ w2[e].t() + b2[e]
    torch.testing.assert_close(y.float(), ref.to(y.dtype).float(), rtol=2e-2, atol=2e-2)


def test_node_matches_float64_emulation_on_exact_inputs():
    counts = [256, 0, 128]
    E, D, H, O = len(counts), 128, 256, 128
    R = _rows(counts)
    parts = {k: torch.zeros(R, n, device="cuda", dtype=torch.float64) for k, n in (("x", D), ("dy", O))}
    cols = {k: [] for k in ("w1", "b1", "w2", "b2")}
    want = []
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        gen = _gen(E, max(c, 128), D, H, O, e)
        x, w1, b1, kind = hidden_layer(max(c, 128), D, H, gen)
        w2, b2 = output_weights(O, kind, gen, 2.0), ternary((O,), 0.5, gen, 2.0 ** -4)
        dy = ternary((max(c, 128), O), 0.25, gen, 2.0 ** -3)
        for k, v in (("w1", w1), ("b1", b1), ("w2", w2), ("b2", b2)):
            cols[k].append(v)
        if c:
            parts["x"][s:s + c], parts["dy"][s:s + c] = x[:c], dy[:c]
            want.append(_emulate_expert(x[:c], w1, b1, w2, b2, dy[:c], what=f"expert {e}"))
        else:
            want.append(None)
    t = {k: torch.stack(v) for k, v in cols.items()}
    y, grads = _node(exact_bf16(parts["x"]), _counts(counts), exact_bf16(t["w1"]), exact_f32(t["b1"]),
                     exact_bf16(t["w2"]), exact_f32(t["b2"]), exact_bf16(parts["dy"]))
    gx, gw1, gb1, gw2, gb2 = grads
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if not c:
            for g, n in ((gw1[e], "gw1"), (gb1[e], "gb1"), (gw2[e], "gw2"), (gb2[e], "gb2")):
                assert bool((g == 0).all()), f"empty expert {e}: {n}"
            continue
        w = want[e]
        assert_same_bits(y[s:s + c], exact_bf16(w["y"]), f"y[{e}]")
        assert_same_bits(gx[s:s + c], exact_bf16(w["gx"]), f"gx[{e}]")
        for got, name in ((gw1[e], "gw1"), (gw2[e], "gw2")):
            assert_same_bits(got, exact_bf16(w[name]), f"{name}[{e}]")
        for got, name in ((gb1[e], "gb1"), (gb2[e], "gb2")):
            assert_same_bits(got, exact_f32(w[name]), f"{name}[{e}]")
    _assert_zero_padding(y, counts, "y")


def _layer_reference(layer, x, r):
    """float64 of the layer's own routing on a CPU copy of its parameters: out and the gradients of sum(out * r)."""
    ps = [getattr(layer, n).detach().double().cpu().requires_grad_() for n in ("router", "w1", "b1", "w2", "b2")]
    router, w1, b1, w2, b2 = ps
    xd = x.detach().double().cpu().requires_grad_()
    probs = torch.softmax(xd @ router.t(), -1)
    gate, choice = probs.topk(layer.top_k, -1)
    out = torch.zeros_like(xd)
    for j in range(layer.top_k):
        g = choice[:, j]
        h = torch.nn.functional.gelu(torch.einsum("td,thd->th", xd, w1[g]) + b1[g], approximate="tanh")
        out = out + gate[:, j:j + 1] * (torch.einsum("th,toh->to", h, w2[g]) + b2[g])
    (out * r.double().cpu()).sum().backward()
    return choice, out, [xd.grad] + [p.grad for p in ps]


@pytest.mark.parametrize("top_k", [1, 2])
def test_dropless_layer_matches_float64(top_k):
    from mpi4torch_b200.parallel import ExpertParallelMLP

    m4t = _m4t()
    layer = ExpertParallelMLP(256, 512, 4, None, m4t.COMM_WORLD, top_k=top_k, device="cuda", seed=5)
    x = _randn(384, 256, seed=21).requires_grad_()
    r = _randn(384, 256, dtype=torch.float32, seed=22)
    before = _launches()
    out, info = layer(x)
    (out.float() * r).sum().backward()
    assert _launches().get("gemm_bias_gelu_grouped", 0) == before.get("gemm_bias_gelu_grouped", 0) + 1
    assert not bool(info.dropped.any())
    choice, ref_out, ref_grads = _layer_reference(layer, x, r)
    agree = float((choice == info.expert.cpu()).double().mean())
    assert agree >= 0.98, f"only {agree} of the choices agree with the float64 router"
    same = (choice == info.expert.cpu()).all(1)  # compare the tokens routed alike
    got = [x.grad] + [getattr(layer, n).grad for n in ("router", "w1", "b1", "w2", "b2")]
    for g, ref, name in [(out, ref_out, "out")] + list(zip(got, ref_grads, ("x", "router", "w1", "b1", "w2", "b2"))):
        g, ref = g.double().cpu(), ref.double()
        if name in ("out", "x"):
            g, ref = g[same], ref[same]
        err = float((g - ref).abs().max())
        assert err <= 3e-2 * max(1.0, float(ref.abs().max())), f"top_k={top_k} {name}: {err}"


def test_capacity_layer_is_unchanged():
    """An int capacity runs the batched exchange exactly as it did before dropless routing existed."""
    from mpi4torch_b200.ops import expert_mlp
    from mpi4torch_b200.parallel import ExpertParallelMLP, combine_from_experts, dispatch_to_experts

    m4t = _m4t()
    layer = ExpertParallelMLP(256, 512, 4, 128, m4t.COMM_WORLD, top_k=2, device="cuda", seed=5)
    x = _randn(384, 256, seed=21)
    out, info = layer(x)
    probs = torch.softmax(torch.nn.functional.linear(x.float(), layer.router), dim=-1)
    gate, choice = probs.topk(2, dim=-1)
    received, routing = dispatch_to_experts(x, choice, 4, 128, m4t.COMM_WORLD)
    back = combine_from_experts(expert_mlp(received, layer.w1, layer.b1, layer.w2, layer.b2), routing, m4t.COMM_WORLD)
    want = (gate.unsqueeze(-1) * back.to(gate.dtype)).sum(1).to(x.dtype)
    assert_same_bits(out, want, "out")
    assert torch.equal(info.dropped, routing.slot < 0) and bool(info.dropped.any())
