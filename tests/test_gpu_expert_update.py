"""Training the expert weights inside the expert wgrad kernels, on one GPU.

The update ops equal, bit for bit, the single-expert ops they generalise: ``batched_wgrad_sgd_`` and
``batched_wgrad_accumulate_`` equal ``wgrad_sgd_`` and ``wgrad_accumulate_`` on each expert's slice, and the grouped
ops equal them on each group's valid rows (zero-padded to 64), over the count patterns of test_gpu_grouped_moe.py with
NaN in every padding row.  An empty group's weight or buffer keeps its exact bits, -0 and NaN included.  The nodes with
``optimizer=`` give the plain mode's ``y`` and ``x.grad`` bit for bit (every read precedes its update), update the
parameters exactly as the op sequence on the plain node's operands, launch the plain mode's kernels with the wgrads
replaced, and synchronise nothing with the host.  With ``accumulator=`` the fp32 buffers equal the per-micro-batch op
sequence bit for bit.  ExpertParallelMLP at one rank gives the plain mode's output, ``x.grad`` and ``router.grad``."""
import re

import pytest
import torch

from conftest import run_spmd
from test_gpu_accum import ODD_G, _operands, fma_f32
from test_gpu_exact_arithmetic import _gen, assert_same_bits, bf16_ulp, exact_bf16, exact_f32
from test_gpu_grouped_moe import _cases, _counts, _grouped, _starts
from test_gpu_moe import _launches, _m4t, _ops, _randn

pytestmark = pytest.mark.gpu

LR = 0.01
BATCHED_SHAPES = [(1, 192, 128, 256), (3, 256, 384, 384), (8, 128, 256, 128)]  # E, M, N, K (K = 384: half last tile)


def _gscale():
    return torch.full((1,), 3.0, device="cuda")


@pytest.mark.parametrize("shape", BATCHED_SHAPES, ids=lambda s: "E{}_M{}_N{}_K{}".format(*s))
def test_batched_update_ops_equal_the_single_expert_ops(shape):
    E, M, N, K = shape
    ops = _ops()
    dy, x, g = _randn(E, M, N, seed=1), _randn(E, M, K, seed=2), _gscale()
    w = _randn(E, N, K, seed=3)
    buf = _randn(E, N, K, dtype=torch.float32, seed=4) * 100
    assert ops.batched_wgrad_sgd_supported(w, dy, x) and ops.batched_wgrad_accumulate_supported(buf, dy, x)
    for gs in (None, g):
        w_got, w_ref = w.clone(), w.clone()
        b_got, b_ref = buf.clone(), buf.clone()
        ops.batched_wgrad_sgd_(w_got, dy, x, -LR, gs)
        ops.batched_wgrad_accumulate_(b_got, dy, x, gs)
        for e in range(E):
            ops.wgrad_sgd_(w_ref[e], dy[e], x[e], -LR, gs)
            ops.wgrad_accumulate_(b_ref[e], dy[e], x[e], gs)
        assert_same_bits(w_got, w_ref, f"{shape} batched_wgrad_sgd_ gs={gs is not None}")
        assert_same_bits(b_got, b_ref, f"{shape} batched_wgrad_accumulate_ gs={gs is not None}")
        assert not torch.equal(w_got, w), "the SGD step changed nothing"


def _poisoned(E, N, K, counts, dtype, seed):
    """[E, N, K] with -0 and NaN entries in the weights of empty groups: bits an update of them would change."""
    t = _randn(E, N, K, dtype=dtype, seed=seed)
    for e, c in enumerate(counts):
        if c <= 0:
            t[e, 0::2] = -0.0
            t[e, 1::4] = float("nan")
    return t


def _padded(t, s, c):
    """Group rows [s, s + c) of t, zero-padded to a multiple of 64 rows: the single-expert ops' operand."""
    out = torch.zeros(-(-c // 64) * 64, t.shape[1], device="cuda", dtype=t.dtype)
    out[:c] = t[s:s + c]
    return out


def _same_raw_bits(got, ref, what):
    ig = torch.int16 if got.dtype == torch.bfloat16 else torch.int32
    assert torch.equal(got.view(ig), ref.view(ig)), f"{what}: bits changed"


@pytest.mark.parametrize("case", list(_cases()))
def test_grouped_update_ops_equal_the_single_expert_ops(case):
    counts = _cases()[case] + [0]  # and an empty last group
    E, N, K = len(counts), 256, 384
    ops = _ops()
    dy, x, cnt, g = _grouped(counts, N, 7), _grouped(counts, K, 8), _counts(counts), _gscale()
    w = _poisoned(E, N, K, counts, torch.bfloat16, 9)
    buf = _poisoned(E, N, K, counts, torch.float32, 10)
    assert ops.grouped_wgrad_sgd_supported(w, dy, x, cnt) and ops.grouped_wgrad_accumulate_supported(buf, dy, x, cnt)
    w_got, b_got = w.clone(), buf.clone()
    ops.grouped_wgrad_sgd_(w_got, dy, x, cnt, -LR, g)
    ops.grouped_wgrad_accumulate_(b_got, dy, x, cnt, g)
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if c == 0:
            _same_raw_bits(w_got[e], w[e], f"{case}: the weight of empty group {e}")
            _same_raw_bits(b_got[e], buf[e], f"{case}: the buffer of empty group {e}")
            continue
        w_ref, b_ref = w[e].clone(), buf[e].clone()
        ops.wgrad_sgd_(w_ref, _padded(dy, s, c), _padded(x, s, c), -LR, g)
        ops.wgrad_accumulate_(b_ref, _padded(dy, s, c), _padded(x, s, c), g)
        assert_same_bits(w_got[e], w_ref, f"{case} grouped_wgrad_sgd_[{e}]")
        assert_same_bits(b_got[e], b_ref, f"{case} grouped_wgrad_accumulate_[{e}]")
        assert bool(torch.isfinite(w_got[e].float()).all()), f"{case}: padding reached the weight of group {e}"


def test_accumulation_keeps_contributions_below_the_buffer_ulp():
    """Onto -fp32(g * G) the one-rounding fma leaves g * G's rounding error, far below the buffer's ulp, where a
    multiply rounded before the add would leave zero; batched and grouped alike."""
    ops = _ops()
    E, Mb, N, K = 2, 128, 256, 256
    gen = _gen(E, Mb, N, K, 71)
    parts = [_operands(Mb, N, K, gen) for _ in range(E)]
    G = torch.stack([dy.t() @ x for dy, x in parts])
    prev = -(ODD_G * G).float().double()
    want = fma_f32(ODD_G, G, prev)
    assert int((want != 0).sum()) > 1000
    gs = torch.full((1,), ODD_G, device="cuda")
    dy = exact_bf16(torch.stack([p[0] for p in parts]))
    x = exact_bf16(torch.stack([p[1] for p in parts]))
    buf = exact_f32(prev).clone()
    ops.batched_wgrad_accumulate_(buf, dy, x, gs)
    assert_same_bits(buf, want, "batched")
    buf = exact_f32(prev).clone()
    ops.grouped_wgrad_accumulate_(buf, dy.reshape(E * Mb, N), x.reshape(E * Mb, K), _counts([Mb] * E), gs)
    assert_same_bits(buf, want, "grouped")


def _rejected(kind):
    """(dy, x, extra, {case: (w for the SGD op, buf for the accumulating op)}): outputs both ops must reject before
    any launch.  M = K, so a weight can be dy's own memory."""
    E, M, N, K = 2, 128, 128, 128
    both = torch.zeros(E * M * K + 2 * E * N * K, device="cuda", dtype=torch.bfloat16)
    x = both[:E * M * K]
    dy_mem = torch.zeros(2 * E * N * K, device="cuda", dtype=torch.bfloat16)  # dy, and room for an fp32 alias of it
    dy = dy_mem[:E * M * N]
    if kind == "batched":
        dy, x, extra = dy.view(E, M, N), x.view(E, M, K), ()
    else:
        dy, x, extra = dy.view(E * M, N), x.view(E * M, K), (_counts([M, 5]),)
    dy.copy_(_randn(*dy.shape, seed=1))
    x.copy_(_randn(*x.shape, seed=2))
    over = both[E * M * K - 16:]  # starts 16 elements inside x, 16-byte aligned
    big = torch.zeros(2 * E * N * K + 8, device="cuda")
    return dy, x, extra, {
        "wrong dtype": (_randn(E, N, K, dtype=torch.float32), _randn(E, N, K)),
        "strided": (_randn(E, N, 2 * K)[:, :, :K], torch.zeros(E, N, 2 * K, device="cuda")[:, :, :K]),
        "misaligned": (big.view(torch.bfloat16)[2:2 + E * N * K].view(E, N, K), big[1:1 + E * N * K].view(E, N, K)),
        "shape mismatch": (_randn(E, N, K + 128), torch.zeros(E, N, K + 128, device="cuda")),
        "aliases dy": (dy.view(E, N, K), dy_mem.view(torch.float32).view(E, N, K)),
        "overlaps x": (over[:E * N * K].view(E, N, K), over.view(torch.float32)[:E * N * K].view(E, N, K)),
    }


@pytest.mark.parametrize("kind", ["batched", "grouped"])
@pytest.mark.parametrize("case", ["wrong dtype", "strided", "misaligned", "shape mismatch", "aliases dy", "overlaps x"])
def test_update_ops_reject_before_any_launch(kind, case):
    ops = _ops()
    dy, x, extra, cases = _rejected(kind)
    w, buf = cases[case]
    w0, buf0, x0, dy0 = w.clone(), buf.clone(), x.clone(), dy.clone()
    torch.cuda.synchronize()
    before = _m4t()._C.kernel_launch_count()
    assert not getattr(ops, f"{kind}_wgrad_sgd_supported")(w, dy, x, *extra)
    assert not getattr(ops, f"{kind}_wgrad_accumulate_supported")(buf, dy, x, *extra)
    with pytest.raises(RuntimeError):
        getattr(ops, f"{kind}_wgrad_sgd_")(w, dy, x, *extra, -LR)
    with pytest.raises(RuntimeError):
        getattr(ops, f"{kind}_wgrad_accumulate_")(buf, dy, x, *extra)
    torch.cuda.synchronize()
    assert _m4t()._C.kernel_launch_count() == before, case
    for got, was, n in ((w, w0, "w"), (buf, buf0, "buf"), (x, x0, "x"), (dy, dy0, "dy")):
        _same_raw_bits(got, was, f"{kind} {case} {n}")


# ---------------------------------------------------------------------------------------------------------------------
# The nodes
# ---------------------------------------------------------------------------------------------------------------------
def _batched_inputs(seed=20):
    E, M, D, H, O = 3, 256, 128, 384, 256
    return dict(x=_randn(E, M, D, seed=seed), w1=_randn(E, H, D, seed=seed + 1) * 0.1,
                b1=_randn(E, H, dtype=torch.float32, seed=seed + 2), w2=_randn(E, O, H, seed=seed + 3) * 0.1,
                b2=_randn(E, O, dtype=torch.float32, seed=seed + 4), dy=_randn(E, M, O, seed=seed + 5))


def _grouped_inputs(seed=30):
    counts = [0, 1, 129, 300]
    E, D, H, O = len(counts), 128, 256, 128
    return dict(x=_grouped(counts, D, seed), counts=_counts(counts), w1=_randn(E, H, D, seed=seed + 1) * 0.1,
                b1=_randn(E, H, dtype=torch.float32, seed=seed + 2), w2=_randn(E, O, H, seed=seed + 3) * 0.1,
                b2=_randn(E, O, dtype=torch.float32, seed=seed + 4), dy=_grouped(counts, O, seed + 5))


def _forward(kind, inp, ps, **update):
    from mpi4torch_b200.ops import expert_mlp, grouped_expert_mlp

    x, w1, b1, w2, b2 = ps
    if kind == "batched":
        return expert_mlp(x, w1, b1, w2, b2, **update)
    return grouped_expert_mlp(x, inp["counts"], w1, b1, w2, b2, **update)


def _leaves(inp, requires=(True,) * 5):
    return [inp[n].detach().clone().requires_grad_(q) for n, q in zip(("x", "w1", "b1", "w2", "b2"), requires)]


def _op_sequence(kind, inp, mode, micro=None):
    """The expected parameters (SGD) or buffers (accumulate) from the ops applied to the plain node's operands."""
    ops = _ops()
    x, w1, b1, w2, b2, dy = (inp[n] for n in ("x", "w1", "b1", "w2", "b2", "dy"))
    c = () if kind == "batched" else (inp["counts"],)
    h, z = getattr(ops, f"{kind}_linear_bias_gelu_forward")(x, w1, b1, *c)
    dz, part = getattr(ops, f"{kind}_gemm_nn_gelu_backward")(dy, w2, z, *c)
    if kind == "batched":
        db1, db2 = ops.batched_column_sum(part), dy.sum(1, dtype=torch.float32)
    else:
        db1, db2 = ops.grouped_column_sum(part, *c), ops.grouped_column_sum(dy, *c)
    if mode == "sgd":
        w1n, w2n = w1.clone(), w2.clone()
        getattr(ops, f"{kind}_wgrad_sgd_")(w2n, dy, h, *c, -LR)
        getattr(ops, f"{kind}_wgrad_sgd_")(w1n, dz, x, *c, -LR)
        return [w1n, b1.clone().add_(db1, alpha=-LR), w2n, b2.clone().add_(db2, alpha=-LR)]
    bufs = micro
    getattr(ops, f"{kind}_wgrad_accumulate_")(bufs[2], dy, h, *c)
    getattr(ops, f"{kind}_wgrad_accumulate_")(bufs[0], dz, x, *c)
    bufs[1].add_(db1)
    bufs[3].add_(db2)
    return bufs


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_node_in_backward_sgd_bitwise(kind):
    from mpi4torch_b200.ops import InBackwardSGD

    inp = _batched_inputs() if kind == "batched" else _grouped_inputs()
    plain = _leaves(inp)
    y_plain = _forward(kind, inp, plain)
    y_plain.backward(inp["dy"])
    ps = _leaves(inp)
    opt = InBackwardSGD(LR)
    before = _launches()
    y = _forward(kind, inp, ps, optimizer=opt)
    mid = _launches()
    y.backward(inp["dy"])
    after = _launches()
    assert_same_bits(y, y_plain, "y")
    assert_same_bits(ps[0].grad, plain[0].grad, "x.grad")
    assert all(p.grad is None for p in ps[1:]), "an expert parameter got a .grad"
    assert opt.updates == 1
    for got, want, n in zip(ps[1:], _op_sequence(kind, inp, "sgd"), ("w1", "b1", "w2", "b2")):
        assert_same_bits(got.detach(), want, f"{kind} {n}")
    # within one bf16 ulp of W - lr * G, with G the wgrad's fp32 sum (read through the accumulating op onto zeros)
    # where the plain mode's .grad is that sum rounded to bf16
    for i, n, G in ((1, "w1", _fp32_grads(kind, inp)[0]), (3, "w2", _fp32_grads(kind, inp)[1])):
        assert bool(((G.to(torch.bfloat16) == plain[i].grad) | (G == 0)).all()), f"{kind} {n}: .grad is not bf16(G)"
        ref = inp[n].double() - LR * G.double()
        err = (ps[i].detach().double() - ref).abs()
        bound = bf16_ulp(ref.abs())
        at = int((err - bound).argmax())
        assert bool((err <= bound).all()), (f"{kind} {n}: {float((err - bound).max())} past one ulp at {at}: got "
                                            f"{float(ps[i].detach().flatten()[at])}, W {float(inp[n].flatten()[at])}, "
                                            f"G {float(G.flatten()[at])}")
    # the plain mode's kernels, the wgrads in their SGD form
    plain_bwd = _backward_launches(kind, inp, {})
    want = {k.replace("wgrad_bf16_", "wgrad_sgd_"): v for k, v in plain_bwd.items()}
    diff = {k: after[k] - mid.get(k, 0) for k in after if after[k] != mid.get(k, 0)}
    assert diff == want, (diff, want)
    assert {k: mid[k] - before.get(k, 0) for k in mid if mid[k] != before.get(k, 0)} == _forward_launches(kind)


def _fp32_grads(kind, inp):
    """(G1, G2): the fp32 sums of the two wgrads on the plain node's operands."""
    ops = _ops()
    c = () if kind == "batched" else (inp["counts"],)
    h, z = getattr(ops, f"{kind}_linear_bias_gelu_forward")(inp["x"], inp["w1"], inp["b1"], *c)
    dz, _ = getattr(ops, f"{kind}_gemm_nn_gelu_backward")(inp["dy"], inp["w2"], z, *c)
    g1, g2 = torch.zeros(inp["w1"].shape, device="cuda"), torch.zeros(inp["w2"].shape, device="cuda")
    getattr(ops, f"{kind}_wgrad_accumulate_")(g1, dz, inp["x"], *c)
    getattr(ops, f"{kind}_wgrad_accumulate_")(g2, inp["dy"], h, *c)
    return g1, g2


def _forward_launches(kind):
    return {f"gemm_bias_gelu_{kind}": 1, f"gemm_bias_{kind}": 1}


def _backward_launches(kind, inp, update, requires=(True,) * 5):
    ps = _leaves(inp, requires)
    y = _forward(kind, inp, ps, **update)
    mid = _launches()
    y.backward(inp["dy"])
    after = _launches()
    return {k: after[k] - mid.get(k, 0) for k in after if after[k] != mid.get(k, 0)}


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_frozen_parameters_are_unchanged_and_cost_no_launch(kind):
    from mpi4torch_b200.ops import AccumulatedSGD, InBackwardSGD

    inp = _batched_inputs(40) if kind == "batched" else _grouped_inputs(40)
    requires = (True, False, True, True, False)  # w1 and b2 frozen
    plain = _backward_launches(kind, inp, {}, requires)
    for update, form in (({"optimizer": InBackwardSGD(LR)}, "wgrad_sgd_"),
                         ({"accumulator": AccumulatedSGD(LR)}, "wgrad_accumulate_")):
        ps = _leaves(inp, requires)
        y = _forward(kind, inp, ps, **update)
        mid = _launches()
        y.backward(inp["dy"])
        after = _launches()
        diff = {k: after[k] - mid.get(k, 0) for k in after if after[k] != mid.get(k, 0)}
        assert diff == {k.replace("wgrad_bf16_", form): v for k, v in plain.items()}, (diff, plain)
        _same_raw_bits(ps[1].detach(), inp["w1"], f"{kind} frozen w1")
        _same_raw_bits(ps[4].detach(), inp["b2"], f"{kind} frozen b2")
        if "accumulator" in update:
            assert len(update["accumulator"].buffers()) == 2
        else:
            assert not torch.equal(ps[3].detach(), inp["w2"])


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_second_backward_after_another_update_raises(kind):
    from mpi4torch_b200.ops import InBackwardSGD

    inp = _batched_inputs(50) if kind == "batched" else _grouped_inputs(50)
    ps = _leaves(inp)
    opt = InBackwardSGD(LR)
    ya = _forward(kind, inp, ps, optimizer=opt)
    yb = _forward(kind, inp, ps, optimizer=opt)
    ya.backward(inp["dy"])
    with pytest.raises(RuntimeError, match="updated in place by another backward"):
        yb.backward(inp["dy"])


@pytest.mark.parametrize("kind", ["batched", "grouped"])
@pytest.mark.parametrize("K", [1, 2, 4])
def test_node_accumulator_bitwise(kind, K):
    from mpi4torch_b200.ops import AccumulatedSGD

    micro = [(_batched_inputs(60 + 10 * k) if kind == "batched" else _grouped_inputs(60 + 10 * k)) for k in range(K)]
    # every micro-batch shares the parameters of the first
    for m in micro[1:]:
        for n in ("w1", "b1", "w2", "b2"):
            m[n] = micro[0][n]
    acc = AccumulatedSGD(LR)
    ps = _leaves(micro[0])
    for m in micro:
        xk = m["x"].clone().requires_grad_()
        ins = [xk] + ps[1:]
        _forward(kind, m, ins, accumulator=acc).backward(m["dy"])
        assert xk.grad is not None
    assert all(p.grad is None for p in ps[1:])
    bufs = {id(p): b for p, b in acc.buffers()}
    want = [torch.zeros(p.shape, device="cuda") for p in ps[1:]]
    sum64 = [torch.zeros(p.shape, device="cuda", dtype=torch.float64) for p in ps[1:]]
    for m in micro:
        _op_sequence(kind, m, "accumulate", want)
        plain = _leaves(m)
        _forward(kind, m, plain).backward(m["dy"])
        for s, p in zip(sum64, plain[1:]):
            s += p.grad.double()
    for p, w, s, n in zip(ps[1:], want, sum64, ("w1", "b1", "w2", "b2")):
        assert_same_bits(bufs[id(p)], w, f"{kind} K={K} buffer of {n}")
        err = float((bufs[id(p)].double() - s).abs().max())
        assert err <= 1e-2 * max(1.0, float(s.abs().max())), f"{kind} K={K} {n}: {err} from the float64 sum"


@pytest.mark.parametrize("kind", ["batched", "grouped"])
def test_update_modes_do_not_synchronise_with_the_host(kind):
    from mpi4torch_b200.ops import AccumulatedSGD, InBackwardSGD

    inp = _batched_inputs(80) if kind == "batched" else _grouped_inputs(80)
    for update in ({"optimizer": InBackwardSGD(LR)}, {"accumulator": AccumulatedSGD(LR)}):
        ps = _leaves(inp)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            _forward(kind, inp, ps, **update).backward(inp["dy"])
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert ps[0].grad is not None


@pytest.mark.parametrize("capacity", [128, None], ids=["capacity", "dropless"])
def test_layer_in_backward_sgd_keeps_the_plain_outputs(capacity):
    from mpi4torch_b200.ops import InBackwardSGD
    from mpi4torch_b200.parallel import ExpertParallelMLP

    comm = _m4t().COMM_WORLD
    layers = [ExpertParallelMLP(256, 512, 4, capacity, comm, top_k=2, device="cuda", seed=5) for _ in range(2)]
    r = _randn(384, 256, dtype=torch.float32, seed=22)
    res = []
    for layer, update in zip(layers, ({}, {"optimizer": InBackwardSGD(LR)})):
        x = _randn(384, 256, seed=21).requires_grad_()
        out, _ = layer(x, **update)
        (out.float() * r).sum().backward()
        res.append((out.detach(), x.grad, layer.router.grad))
    for got, want, n in zip(res[1], res[0], ("out", "x.grad", "router.grad")):
        assert_same_bits(got, want, n)
    plain, sgd = layers
    for n in ("w1", "b1", "w2", "b2"):
        assert getattr(sgd, n).grad is None
        assert not torch.equal(getattr(sgd, n), getattr(plain, n)), f"{n} was not updated"


def test_moe_example_trains_with_sgd_in_backward():
    res = run_spmd(1, ["examples/moe_layer.py", "--device", "cuda", "--steps", "20", "--sgd-in-backward"],
                   device="cuda", timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", res.stdout)]
    assert len(losses) == 20 and losses[-1] < losses[0], losses


@pytest.mark.parametrize("dropless", [False, True])
def test_moe_example_trains_with_micro_batches_on_cuda(dropless):
    res = run_spmd(1, ["examples/moe_layer.py", "--device", "cuda", "--steps", "20", "--micro-batches", "2"]
                   + (["--dropless"] if dropless else []), device="cuda", timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", res.stdout)]
    assert len(losses) == 20 and losses[-1] < losses[0], losses
