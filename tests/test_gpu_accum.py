"""Gradient accumulation on the GPU, bit for bit at one rank on exactly representable inputs.

``wgrad_accumulate_(acc, dy, x, g)`` is ``acc <- fmaf(g, dy^T x, acc)`` per element: the wgrad GEMM's fp32 sum, then
ONE rounding of the product plus the old buffer.  On the exact inputs of test_gpu_exact_arithmetic.py the GEMM sum is
exact, so the float64 value ``g * G + acc`` rounded once to fp32 is the kernel's result.  A grad_scale of 1 + 2^-20
makes ``g * G`` need more than 24 bits; onto the buffer ``-fp32(g * G)`` the fma leaves the product's rounding error,
where a multiply rounded before the add would leave zero.

The models: ``train_step(x, t, micro_batches=4)`` accumulates the chunks' exact gradients in fp32, and ``step()``
applies ``p + fp32(-lr * buf)``; with a power-of-two lr that is the full-batch in-backward update bit for bit.
"""
import pytest
import torch

from test_gpu_exact_arithmetic import (U24, WAVE_KBLOCKS, WGRAD_EDGE_SHAPES, _gen, _ops, _sm_count, assert_exact_gemm,
                                       assert_same_bits, exact_bf16, exact_f32, ints, mse_target, quantum, ternary,
                                       wave_tile_counts, wgrad_wave_shape)
from test_gpu_mlp_exact import (N_REAL, XENT_IGNORE, _check_b2, _check_params, _check_saturation, _xent_bounds,
                                emulate_node, emulate_sgd_in_backward, mse_case, xent_case)

pytestmark = pytest.mark.gpu

ODD_G = 1.0 + 2.0 ** -20  # fp32-representable; g * G needs up to 43 bits


def fma_f32(g, G, prev):
    """fp32(g * G + prev) with one rounding: exact in float64 for these inputs (checked), rounded once."""
    v = g * G + prev
    assert torch.equal(v - prev, g * G), "g * G + prev is not exact in float64"
    return v.float()


def _operands(Mb, N, K, gen):
    dy, x = ints((Mb, N), 16, gen, 2.0 ** -3), ints((Mb, K), 16, gen, 2.0 ** -4)
    assert_exact_gemm(dy.t(), x, what="wgrad_accumulate")
    return dy, x


def _prev(G, gen):
    """A nonzero fp32 buffer up to 2^28 quanta of G on a 2^8-quanta grid: most sums round, ties included."""
    q = quantum(G) if bool((G != 0).any()) else 2.0 ** -7
    return ints(G.shape, 2 ** 20, gen, q * 2.0 ** 8)


def check_accumulate(Mb, N, K, gen):
    ops = _ops()
    dy, x = _operands(Mb, N, K, gen)
    G = dy.t() @ x
    dyb, xb = exact_bf16(dy), exact_bf16(x)
    shape = (Mb, N, K)
    assert ops.wgrad_accumulate_supported(torch.zeros(N, K, device="cuda"), dyb, xb)
    # grad_scale absent, onto zeros: the exact G in fp32
    acc = torch.zeros(N, K, device="cuda")
    ops.wgrad_accumulate_(acc, dyb, xb)
    assert_same_bits(acc, exact_f32(G), f"wgrad_accumulate_ onto zeros {shape}")
    # a device grad_scale onto a nonzero buffer, a power of two and 1 + 2^-20
    for g, prev in ((2.0 ** 3, _prev(G, gen)), (ODD_G, _prev(G, gen)), (ODD_G, -(ODD_G * G).float().double())):
        acc = exact_f32(prev).clone()
        ops.wgrad_accumulate_(acc, dyb, xb, torch.full((1,), g, device="cuda"))
        assert_same_bits(acc, fma_f32(g, G, prev), f"wgrad_accumulate_ g={g} {shape}")


@pytest.mark.parametrize("shape", WGRAD_EDGE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_accumulate_tile_edges_bitwise(shape):
    check_accumulate(*shape, _gen(*shape, 31))


@pytest.mark.parametrize("kblocks", (1,) + WAVE_KBLOCKS)
@pytest.mark.parametrize("wave", range(4), ids=["S-1", "S", "S+1", "2S+1"])
def test_accumulate_wave_edges_bitwise(wave, kblocks):
    T = wave_tile_counts(_sm_count())[wave]
    Mb, N, K = wgrad_wave_shape(T, kblocks)
    check_accumulate(Mb, N, K, _gen(Mb, N, K, 32))


def test_fma_is_visible():
    """On the cancelling buffer the fma leaves nonzero residuals where multiply-then-add leaves zeros: the bitwise
    tests above tell the two roundings apart."""
    Mb, N, K = 192, 512, 384
    gen = _gen(Mb, N, K, 33)
    dy, x = _operands(Mb, N, K, gen)
    G = dy.t() @ x
    prev = -(ODD_G * G).float().double()
    assert int((fma_f32(ODD_G, G, prev) != 0).sum()) > 1000


@pytest.mark.parametrize("chunks", [2, 4])
def test_chunks_equal_whole_batch(chunks):
    """K calls on the K chunks of a batch leave the buffer of one call on the whole batch."""
    ops = _ops()
    Mb, N, K = 512, 384, 640
    gen = _gen(Mb, N, K, 34 + chunks)
    dy, x = _operands(Mb, N, K, gen)
    dyb, xb = exact_bf16(dy), exact_bf16(x)
    gs = torch.full((1,), 2.0 ** -2, device="cuda")
    whole = torch.zeros(N, K, device="cuda")
    ops.wgrad_accumulate_(whole, dyb, xb, gs)
    parts = torch.zeros(N, K, device="cuda")
    for dc, xc in zip(dyb.split(Mb // chunks), xb.split(Mb // chunks)):
        ops.wgrad_accumulate_(parts, dc, xc, gs)
    assert_same_bits(whole, exact_f32(2.0 ** -2 * (dy.t() @ x)), "one call")
    assert_same_bits(parts, whole, f"{chunks} chunked calls")


def test_nan_stays_in_its_elements():
    """A NaN in dy poisons exactly one row of the gradient; a NaN already in the buffer stays in its element only."""
    ops = _ops()
    Mb, N, K = 320, 384, 640
    gen = _gen(Mb, N, K, 36)
    dy, x = _operands(Mb, N, K, gen)
    G = dy.t() @ x
    prev = _prev(G, gen)
    i0, n0 = 77, 130
    j0, k0 = 301, 519
    dyb = exact_bf16(dy)
    dyb[i0, n0] = float("nan")
    acc = exact_f32(prev).clone()
    acc[j0, k0] = float("nan")
    ops.wgrad_accumulate_(acc, dyb, exact_bf16(x), torch.full((1,), 2.0, device="cuda"))
    ref = fma_f32(2.0, G, prev)
    ref[n0, :] = float("nan")
    ref[j0, k0] = float("nan")
    assert_same_bits(acc, ref, "wgrad_accumulate_ with NaNs")


def _rejected_buffers(N, K):
    dev = "cuda"
    flat = torch.zeros(N * K + 8, device=dev)
    wide = torch.zeros(N, K + 128, device=dev)
    return {
        "bf16": torch.zeros(N, K, device=dev, dtype=torch.bfloat16),
        "fp64": torch.zeros(N, K, device=dev, dtype=torch.float64),
        "cpu": torch.zeros(N, K),
        "rows+128": torch.zeros(N + 128, K, device=dev),
        "cols+128": torch.zeros(N, K + 128, device=dev),
        "transposed": torch.zeros(K, N, device=dev).t(),
        "row stride": wide[:, :K],
        "1-d": torch.zeros(N * K, device=dev),
        "offset 4 B": flat[1:1 + N * K].view(N, K),
        "offset 8 B": flat[2:2 + N * K].view(N, K),
    }


REJECTED = ["bf16", "fp64", "cpu", "rows+128", "cols+128", "transposed", "row stride", "1-d", "offset 4 B",
            "offset 8 B"]


@pytest.mark.parametrize("layout", REJECTED)
def test_rejected_buffers_raise_without_launch(layout):
    """Every buffer layout that wgrad_accumulate_supported rejects makes the op raise before anything is launched."""
    import mpi4torch_b200 as m4t

    ops = _ops()
    Mb, N, K = 128, 128, 256
    gen = _gen(Mb, N, K, 37)
    dy, x = _operands(Mb, N, K, gen)
    dyb, xb = exact_bf16(dy), exact_bf16(x)
    buffers = _rejected_buffers(N, K)
    assert sorted(buffers) == sorted(REJECTED)
    acc = buffers[layout]
    if layout == "transposed":
        assert acc.shape == (N, K) and not acc.is_contiguous()
    assert not ops.wgrad_accumulate_supported(acc, dyb, xb)
    before = acc.clone()
    n0 = dict(m4t._C.kernel_launch_table()).get("wgrad_accumulate", 0)
    with pytest.raises(RuntimeError, match="wgrad_accumulate_"):
        ops.wgrad_accumulate_(acc, dyb, xb)
    torch.cuda.synchronize()
    assert dict(m4t._C.kernel_launch_table()).get("wgrad_accumulate", 0) == n0
    assert torch.equal(acc, before)


def test_rejected_operands_raise():
    """The operand rules of wgrad_bf16_supported: batch % 64, N % 128, K % 128, bf16 operands."""
    ops = _ops()
    cases = {"batch 96": (96, 128, 128), "N 192": (64, 192, 128), "K 200": (64, 128, 200)}
    for what, (Mb, N, K) in cases.items():
        dy = torch.zeros(Mb, N, device="cuda", dtype=torch.bfloat16)
        x = torch.zeros(Mb, K, device="cuda", dtype=torch.bfloat16)
        acc = torch.zeros(N, K, device="cuda")
        assert not ops.wgrad_accumulate_supported(acc, dy, x), what
        with pytest.raises(RuntimeError):
            ops.wgrad_accumulate_(acc, dy, x)
    dy = torch.zeros(64, 128, device="cuda")
    x = torch.zeros(64, 128, device="cuda", dtype=torch.bfloat16)
    assert not ops.wgrad_accumulate_supported(torch.zeros(128, 128, device="cuda"), dy, x)


# ------------------------------------------------------------------------------------------------------------------
# The models at one rank
# ------------------------------------------------------------------------------------------------------------------
def _comm():
    import mpi4torch_b200 as m4t

    comm = m4t.COMM_WORLD
    assert comm.size == 1 and m4t.cuda_backend_ready()
    return comm


def _bits_equal(a, b, what):
    assert_same_bits(a.detach(), b.detach(), what)


def test_dp_linear_model_micro_batches_bitwise():
    """Four micro-batches give the full-batch in-backward step bit for bit, twice in a row (the inputs stay exact)."""
    from mpi4torch_b200.models import DPLinearModel

    B, D, O = 1024, 512, 512
    comm = _comm()
    gen = _gen(B, D, O, 40)
    lr = B / 2.0
    full = DPLinearModel(D, O, comm, device="cuda", lr=lr, seed=3)
    accum = DPLinearModel(D, O, comm, device="cuda", lr=lr, seed=3)
    w = ternary((O, D), 0.25, gen, 2.0 ** -4)
    with torch.no_grad():
        full.weight.copy_(exact_bf16(w))
        accum.weight.copy_(exact_bf16(w))
    for step in range(2):
        x = ternary((B, D), 0.25, gen)
        assert_exact_gemm(x, w.t(), what=f"step {step}")
        t = mse_target(x @ w.t(), gen, 1 / 64)
        w_before = full.weight.detach().clone()
        l_full = full.train_step(exact_bf16(x), t)
        l_acc = accum.train_step(exact_bf16(x), t, micro_batches=4)
        assert not torch.equal(full.weight.detach(), w_before), "the case does not move the weight"
        _bits_equal(l_acc, l_full, f"step {step} loss")
        _bits_equal(accum.weight, full.weight, f"step {step} weight")
        w = full.weight.detach().double()
    assert accum.weight.grad is None and accum.accumulator.updates == 2
    assert all(not bool(b.any()) for _, b in accum.accumulator.buffers())


def _load(model, w1, b1, w2, b2):
    with torch.no_grad():
        for p, v in zip(model.parameters(), (exact_bf16(w1), exact_f32(b1), exact_bf16(w2), exact_f32(b2))):
            p.copy_(v)


def test_dp_mlp_model_micro_batches_bitwise():
    """DPMLPModel (MSE), micro_batches=4: the in-backward full-batch step and the float64 emulation, bit for bit."""
    from mpi4torch_b200.models import DPMLPModel

    shape = (256, 256, 512, 384)
    B, D, H, O = shape
    comm = _comm()
    x, w1, b1, w2, b2, t = mse_case(*shape, _gen(*shape, 41))
    lr = 2.0 ** 2
    full = DPMLPModel(D, H, O, comm, device="cuda", lr=lr)
    accum = DPMLPModel(D, H, O, comm, device="cuda", lr=lr)
    for m in (full, accum):
        _load(m, w1, b1, w2, b2)
    h, z_k = torch.ops.mpi4torch_b200.linear_bias_gelu_forward(exact_bf16(x), full.w1.detach(), full.b1.detach())
    _check_saturation(h, z_k, "mlp accum")
    e = emulate_node(x, w1, b1, w2, b2, ls=1.0 / B, target=t, what="mlp accum")
    want = emulate_sgd_in_backward([w1, b1, w2, b2], e, lr, lr)
    assert all(not torch.equal(a, b) for a, b in zip(want, (w1, b1, w2, b2))), "the case leaves a parameter unchanged"
    l_full = full.train_step(exact_bf16(x), t)
    l_acc = accum.train_step(exact_bf16(x), t, micro_batches=4)
    _bits_equal(l_acc, l_full, "loss")
    _check_params(accum.parameters(), want, "micro_batches=4")
    for p, q in zip(accum.parameters(), full.parameters()):
        _bits_equal(p, q, "accumulated vs in-backward")
    assert len(accum.accumulator.buffers()) == 4
    assert all(b.dtype == torch.float32 and not bool(b.any()) for _, b in accum.accumulator.buffers())


def test_dp_mlp_classifier_micro_batches():
    """DPMLPClassifier with equal logits, micro_batches=4: W1, b1, W2 bit for bit against the emulation of the
    full-batch in-backward step; the loss and b2 within the derived fp32 bounds plus the K-term sums of the chunks."""
    from mpi4torch_b200.models import DPMLPClassifier

    B, D, H, K = 256, 256, 256, 4
    comm = _comm()
    x, w1, b1, w2, b2, labels = xent_case(B, D, H, _gen(B, D, H, 42), XENT_IGNORE)
    lr = 2.0 ** 3
    model = DPMLPClassifier(D, H, 2 * N_REAL, comm, device="cuda", lr=lr, ignore_index=XENT_IGNORE)
    _load(model, w1, b1, w2, b2)
    ls = 1.0 / B
    e = emulate_node(x, w1, b1, w2, b2, ls=ls, labels=labels, ignore_index=XENT_IGNORE, what="classifier accum")
    loss = model.train_step(exact_bf16(x), labels.cuda(), micro_batches=K)
    loss_bound, gb2_bound = _xent_bounds(e, labels, 1.0, ls)
    loss_bound += K * U24 * float(e["loss"])
    assert abs(float(loss) - float(e["loss"])) <= loss_bound, f"loss {float(loss)!r} vs {float(e['loss'])!r}"
    want = emulate_sgd_in_backward([w1, b1, w2, b2], e, lr, lr)
    w1_k, b1_k, w2_k, b2_k = model.parameters()
    _check_params([w1_k, b1_k, w2_k], want[:3], "classifier micro_batches=4")
    chunk_sums = K * U24 * e["dy32"].abs().sum(0)[:N_REAL]
    _check_b2(b2_k.detach(), want[3], lr * (gb2_bound + chunk_sums) + U24 * want[3][:N_REAL].abs(), "classifier b2")


def test_mlp_step_launches():
    """One DPMLPModel step with micro_batches=4 runs 8 accumulating wgrad kernels and no other wgrad."""
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.models import DPMLPModel

    B, D, H, O = 256, 256, 256, 256
    comm = _comm()
    model = DPMLPModel(D, H, O, comm, device="cuda", lr=1e-3)
    g = torch.Generator(device="cuda").manual_seed(43)
    x = torch.randn(B, D, device="cuda", generator=g).to(torch.bfloat16)
    t = torch.randn(B, O, device="cuda", generator=g).to(torch.bfloat16)
    model.train_step(x, t, micro_batches=4)  # warm-up: lazy buffers
    torch.cuda.synchronize()
    before = dict(m4t._C.kernel_launch_table())
    w0 = model.w1.detach().clone()
    model.train_step(x, t, micro_batches=4)
    torch.cuda.synchronize()
    after = dict(m4t._C.kernel_launch_table())
    diff = {k: v - before.get(k, 0) for k, v in after.items() if v != before.get(k, 0)}
    assert diff.get("wgrad_accumulate") == 8, diff
    assert "wgrad_sgd_epilogue" not in diff and "wgrad" not in diff, diff
    assert not torch.equal(model.w1.detach(), w0)
    assert all(p.grad is None for p in model.parameters())
