"""wgmma GEMM numerics against a plain fp32 PyTorch reference."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(x, w):
    return (x.float() @ w.float().t())


def _assert_close_bf16(got, ref, K, what=""):
    """Element-wise check of a bf16 result against the fp32 reference: each element may differ by bf16
    output rounding (2^-8 relative) plus fp32 accumulation-order noise, which scales with the magnitude of
    the K summands rather than with the (possibly cancelled) result.  A dropped K-slice or a wrong tile
    changes elements by O(sqrt(K/BK)) * that floor and fails."""
    got = got.float()
    err = (got - ref).abs()
    floor = 2.0 ** -7 * ref.abs() + 2.0 ** -9 * (float(K) ** 0.5)
    bad = ~(err <= floor)  # NaN fails
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements off, worst {float((err - floor).max()):.4g} (max ref {float(ref.abs().max()):.4g})"


@pytest.mark.parametrize("shape", [(128, 256, 64), (256, 512, 128), (384, 256, 4096), (4096, 4096, 4096),
                                   (8192, 4096, 4096), (130, 264, 72), (1, 8, 8), (1000, 1000, 1000)])
def test_gemm_bf16_tn_matches_fp32_reference(shape):
    import mpi4torch_b200 as m4t  # noqa: F401

    m4t.COMM_WORLD  # bring the backend up
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    assert torch.ops.mpi4torch_b200.gemm_bf16_tn_supported(x, w)
    y = torch.ops.mpi4torch_b200.gemm_bf16_tn(x, w)
    torch.cuda.synchronize()
    ref = _ref(x, w)
    _assert_close_bf16(y, ref, K=K, what=f"gemm {shape}")
    # structured check: identity-like weight reproduces the input exactly
    if N == K:
        eye = torch.eye(N, device="cuda", dtype=torch.bfloat16)
        assert torch.equal(torch.ops.mpi4torch_b200.gemm_bf16_tn(x, eye), x)


def test_gemm_speed_report():
    import mpi4torch_b200 as m4t  # noqa: F401

    m4t.COMM_WORLD
    M, N, K = 8192, 4096, 4096
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    w = torch.randn(N, K, device="cuda").to(torch.bfloat16)
    for name, fn in (("wgmma", lambda: torch.ops.mpi4torch_b200.gemm_bf16_tn(x, w)), ("cublas", lambda: x @ w.t())):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(10):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b) / 10
        print(f"[gemm] {name}: {ms:.3f} ms  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s")


@pytest.mark.parametrize("shape", [(64, 256, 256), (128, 256, 512), (512, 512, 256), (8192, 4096, 4096), (4096, 1024, 2048),
                                   (256, 384, 640)])
def test_wgrad_mn_major_matches_fp32_reference(shape):
    import mpi4torch_b200 as m4t  # noqa: F401

    m4t.COMM_WORLD
    Mb, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(Mb + 3 * N + 7 * K)
    dy = torch.randn(Mb, N, device="cuda", generator=g).to(torch.bfloat16)
    x = torch.randn(Mb, K, device="cuda", generator=g).to(torch.bfloat16)
    assert torch.ops.mpi4torch_b200.wgrad_bf16_supported(dy, x)
    gw = torch.ops.mpi4torch_b200.wgrad_bf16(dy, x)
    torch.cuda.synchronize()
    ref = dy.float().t() @ x.float()
    _assert_close_bf16(gw, ref, K=Mb, what=f"wgrad {shape}")
    # structured check: a one-hot dy row selects rows of x exactly
    sel = torch.zeros(Mb, N, device="cuda", dtype=torch.bfloat16)
    idx = torch.arange(min(Mb, N), device="cuda")
    sel[idx, idx] = 1
    out = torch.ops.mpi4torch_b200.wgrad_bf16(sel, x)
    assert torch.equal(out[: idx.numel()], x[: idx.numel()])


@pytest.mark.parametrize("shape", [(256, 256, 64), (384, 512, 256), (8192, 4096, 4096), (300, 520, 200), (1000, 1000, 1000),
                                   (130, 264, 72)])
def test_linear_mse_epilogue_matches_fp32_reference(shape):
    """GEMM with the fused loss epilogue (dL/dy = g * (x W^T - t), loss = s * sum((x W^T - t)^2)), large
    shapes and ragged tiles."""
    import mpi4torch_b200 as m4t  # noqa: F401

    m4t.COMM_WORLD
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + 5 * N + 11 * K)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    t = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    grad_scale, loss_scale = 2.0 / M, 1.0 / M
    dy, loss, w_avg = torch.ops.mpi4torch_b200.linear_mse_forward(x, w, t, 1.0, loss_scale, grad_scale, True)
    torch.cuda.synchronize()
    d = x.float() @ w.float().t() - t.float()
    ref_dy = grad_scale * d
    err = (dy.float() - ref_dy).abs().max().item()
    assert err <= 2e-2 * ref_dy.abs().max().item() + 1e-6, f"{shape}: dL/dy max abs err {err}"
    ref_loss = loss_scale * d.square().sum().item()
    assert abs(float(loss) - ref_loss) <= 2e-3 * abs(ref_loss), f"{shape}: loss {float(loss)} vs {ref_loss}"
    assert w_avg.data_ptr() == w.data_ptr()  # single rank: nothing to average
    # exact structure: target equal to the bf16 product -> loss and gradient are (almost) zero
    y = torch.ops.mpi4torch_b200.gemm_bf16_tn(x, w)
    dy0, loss0, _ = torch.ops.mpi4torch_b200.linear_mse_forward(x, w, y, 1.0, 1.0, 1.0, True)
    assert dy0.float().abs().max().item() <= 2 ** -7 * y.float().abs().max().item() + 1e-6


@pytest.mark.parametrize("shape", [(256, 256, 64), (512, 768, 256), (8192, 4096, 4096), (300, 520, 200), (1000, 1000, 1000)])
def test_gemm_nn_dgrad_matches_fp32_reference(shape):
    """gy[M,N] @ W[N,K] with the weight read in place as an MN-major wgmma operand (no transposed copy)."""
    import mpi4torch_b200 as m4t  # noqa: F401

    m4t.COMM_WORLD
    M, N, K = shape
    g = torch.Generator(device="cuda").manual_seed(M + 3 * N + 5 * K)
    gy = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(N, K, device="cuda", generator=g).to(torch.bfloat16)
    assert torch.ops.mpi4torch_b200.gemm_bf16_nn_supported(gy, w)
    gx = torch.ops.mpi4torch_b200.gemm_bf16_nn(gy, w)
    torch.cuda.synchronize()
    ref = gy.float() @ w.float()
    _assert_close_bf16(gx, ref, K=N, what=f"dgrad {shape}")
    if M == N:  # identity gy selects the rows of w exactly
        eye = torch.eye(N, device="cuda", dtype=torch.bfloat16)
        assert torch.equal(torch.ops.mpi4torch_b200.gemm_bf16_nn(eye, w), w)


def test_wgrad_grad_scale_and_sgd_epilogue():
    """Device-scalar grad_scale folded into the wgrad epilogue, and the single-rank SGD step as the GEMM's own epilogue."""
    import mpi4torch_b200 as m4t  # noqa: F401

    m4t.COMM_WORLD
    Mb, N, K = 512, 512, 256
    g = torch.Generator(device="cuda").manual_seed(17)
    dy = torch.randn(Mb, N, device="cuda", generator=g).to(torch.bfloat16)
    x = torch.randn(Mb, K, device="cuda", generator=g).to(torch.bfloat16)
    gs = torch.full((1,), 3.0, device="cuda")
    ref = dy.float().t() @ x.float()
    _assert_close_bf16(torch.ops.mpi4torch_b200.wgrad_bf16(dy, x, gs), 3.0 * ref, K=Mb, what="wgrad * grad_scale")
    w0 = (torch.randn(N, K, device="cuda", generator=g) * 4).to(torch.bfloat16)
    w = w0.clone()
    torch.ops.mpi4torch_b200.wgrad_sgd_(w, dy, x, -0.01, gs)
    torch.cuda.synchronize()
    _assert_close_bf16(w, w0.float() - 0.03 * ref, K=Mb, what="wgrad_sgd_")
