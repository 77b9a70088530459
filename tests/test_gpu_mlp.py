"""Two-layer MLP on the wgmma kernels: the bias+GELU, bias+MSE+column-sum and GELU-backward+column-sum GEMM
epilogues and the column-sum reduce against fp32 references, and DPMLPModel at one rank against the fp32 torch
composition."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_gemm import _assert_close_bf16

pytestmark = pytest.mark.gpu

SHAPES = [(130, 264, 72), (1, 8, 8), (1000, 1000, 1000), (8192, 16384, 4096)]


def _ops():
    import mpi4torch_b200 as m4t

    m4t.COMM_WORLD  # bring the backend up
    return torch.ops.mpi4torch_b200


def _gen(*vals):
    return torch.Generator(device="cuda").manual_seed(sum((i + 1) * 7919 * v for i, v in enumerate(vals)))


def _assert_colsum(got, values, what):
    """Column sums against the fp64 sum of fp32 values: the kernel's own fp32 values differ from the reference's
    by accumulation-order noise, so the bound is relative to the sum of magnitudes."""
    ref = values.double().sum(0)
    bound = 1e-5 * values.double().abs().sum(0) + 1e-6
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), f"{what}: column sum off by {float((err - bound).max()):.4g} over the bound"


@pytest.mark.parametrize("shape", SHAPES)
def test_linear_bias_gelu_forward(shape):
    ops = _ops()
    M, N, K = shape
    g = _gen(M, N, K)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g)
    h, z = ops.linear_bias_gelu_forward(x, w, b)
    torch.cuda.synchronize()
    z_ref = x.float() @ w.float().t() + b
    _assert_close_bf16(z, z_ref, K=K, what=f"bias+gelu z {shape}")
    # h comes from the fp32 z: z's error (gelu' <= 1.13) plus the bf16 rounding of h
    h_ref = F.gelu(z_ref, approximate="tanh")
    err = (h.float() - h_ref).abs()
    floor = 1.2 * (2.0 ** -7 * z_ref.abs() + 2.0 ** -9 * K ** 0.5) + 2.0 ** -8 * h_ref.abs()
    assert not bool((err > floor).any()), f"bias+gelu h {shape}: worst {float((err - floor).max()):.4g}"


@pytest.mark.parametrize("shape", SHAPES)
def test_linear_bias_mse_colsum(shape):
    ops = _ops()
    M, N, K = shape
    g = _gen(M, N, K, 1)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    b = torch.randn(N, device="cuda", generator=g)
    t = torch.randn(M, N, device="cuda", generator=g).to(torch.bfloat16)
    loss_scale, grad_scale = 1.0 / M, 2.0 / M
    dy, loss, part = ops.linear_bias_mse_forward_local(x, w, b, t, loss_scale, grad_scale)
    torch.cuda.synchronize()
    assert part.shape == ((M + 15) // 16, N) and part.dtype == torch.float32
    d = x.float() @ w.float().t() + b - t.float()
    ref_dy = grad_scale * d
    err = (dy.float() - ref_dy).abs().max().item()
    assert err <= 2e-2 * ref_dy.abs().max().item() + 1e-6, f"{shape}: dL/dy max abs err {err}"
    ref_loss = loss_scale * d.double().square().sum().item()
    assert abs(float(loss) - ref_loss) <= 2e-3 * abs(ref_loss), f"{shape}: loss {float(loss)} vs {ref_loss}"
    db = ops.column_sum(part)
    _assert_colsum(db, ref_dy, f"dy column sum {shape}")
    gs = torch.full((1,), 3.0, device="cuda")
    _assert_colsum(ops.column_sum(part, gs), 3.0 * ref_dy, f"dy column sum x grad_scale {shape}")
    # deterministic: a second identical call gives the same bits
    dy2, _, part2 = ops.linear_bias_mse_forward_local(x, w, b, t, loss_scale, grad_scale)
    assert torch.equal(dy, dy2) and torch.equal(part, part2) and torch.equal(ops.column_sum(part2), db)


@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_nn_gelu_backward(shape):
    """dz = grad_scale * (dy @ W) * gelu_tanh'(z) against torch autograd of F.gelu(approximate="tanh") in fp32 on
    the stored bf16 z."""
    ops = _ops()
    M, N, K = shape  # dy [M, K] @ W [K, N] -> dz [M, N]
    g = _gen(M, N, K, 2)
    dy = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randn(K, N, device="cuda", generator=g).to(torch.bfloat16)
    z = (2 * torch.randn(M, N, device="cuda", generator=g)).to(torch.bfloat16)
    for scale in (None, 3.0):
        gs = None if scale is None else torch.full((1,), scale, device="cuda")
        dz, part = ops.gemm_nn_gelu_backward(dy, w, z, gs)
        torch.cuda.synchronize()
        zz = z.float().requires_grad_()
        F.gelu(zz, approximate="tanh").backward((scale or 1.0) * (dy.float() @ w.float()))
        ref = zz.grad
        err = (dz.float() - ref).abs()
        floor = 2.0 ** -7 * ref.abs() + 1.2 * (scale or 1.0) * 2.0 ** -9 * K ** 0.5
        assert not bool((err > floor).any()), f"gelu backward {shape} x{scale}: worst {float((err - floor).max()):.4g}"
        db = ops.column_sum(part)
        _assert_colsum(db, ref, f"dz column sum {shape} x{scale}")
        dz2, part2 = ops.gemm_nn_gelu_backward(dy, w, z, gs)
        assert torch.equal(dz, dz2) and torch.equal(ops.column_sum(part2), db)


def _launches():
    import mpi4torch_b200 as m4t

    return dict(m4t._C.kernel_launch_table())


def _reference_steps(params, xs, ts, lr):
    """fp32 torch composition: Linear -> GELU(tanh) -> Linear -> MSE (mean over the batch), SGD."""
    w1, b1, w2, b2 = [p.detach().float().clone().requires_grad_() for p in params]
    losses = []
    for x, t in zip(xs, ts):
        y = F.linear(F.gelu(F.linear(x.float(), w1, b1), approximate="tanh"), w2, b2)
        loss = (y - t.float()).square().sum() / x.shape[0]
        loss.backward()
        with torch.no_grad():
            for p in (w1, b1, w2, b2):
                p -= lr * p.grad
                p.grad = None
        losses.append(float(loss))
    return losses, [p.detach() for p in (w1, b1, w2, b2)]


def _run_model(B, D, H, O, sgd_in_backward, kernels_expected):
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.models import DPMLPModel

    comm = m4t.COMM_WORLD
    lr = 12.8 / O  # the loss sums over the O outputs: a fixed step size would diverge at O = 4096
    model = DPMLPModel(D, H, O, comm, device="cuda", lr=lr, seed=11, sgd_in_backward=sgd_in_backward)
    assert model.b1.dtype == torch.float32 and model.w1.dtype == torch.bfloat16
    init = [p.detach().clone() for p in model.parameters()]
    g = _gen(B, D, H, O)
    xs = [torch.randn(B, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3)]
    ts = [torch.randn(B, O, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3)]
    names = ("gemm_bias_gelu", "gemm_bias_mse_colsum", "gemm_nn_gelu_bwd_colsum")
    losses = []
    for x, t in zip(xs, ts):
        before = _launches()
        if sgd_in_backward and kernels_expected:
            loss = model.loss(x, t)
            loss.backward()
            assert all(p.grad is None for p in model.parameters()), "optimizer-in-backward left a .grad"
            losses.append(float(loss))
        else:
            losses.append(float(model.train_step(x, t)))
        after = _launches()
        for n in names:
            ran = after.get(n, 0) - before.get(n, 0)
            assert ran == (1 if kernels_expected else 0), f"{n} ran {ran} times in one step"
    ref_losses, ref_params = _reference_steps(init, xs, ts, lr)
    what = f"{(B, D, H, O)} sgd_in_backward={sgd_in_backward}"
    for got, ref in zip(losses, ref_losses):
        assert abs(got - ref) <= 1e-2 * abs(ref), f"{what}: loss {got} vs {ref}"
    for name, p, ref in zip(("w1", "b1", "w2", "b2"), model.parameters(), ref_params):
        err = float((p.detach().float() - ref).abs().max())
        assert err <= 2e-2, f"{what}: {name} off by {err}"


@pytest.mark.parametrize("sgd_in_backward", [True, False])
@pytest.mark.parametrize("dims", [(384, 256, 512, 256), (8192, 4096, 16384, 4096)])
def test_dp_mlp_model_single_rank(dims, sgd_in_backward):
    _run_model(*dims, sgd_in_backward=sgd_in_backward, kernels_expected=True)


def test_dp_mlp_model_off_the_kernel_path():
    """H = 200 is not a multiple of 128: the model runs the torch composition and still matches."""
    from mpi4torch_b200.ops import dp_mlp_mse_supported

    _run_model(384, 256, 200, 256, sgd_in_backward=True, kernels_expected=False)
    x = torch.zeros(384, 256, device="cuda", dtype=torch.bfloat16)
    w1 = torch.zeros(200, 256, device="cuda", dtype=torch.bfloat16)
    w2 = torch.zeros(256, 200, device="cuda", dtype=torch.bfloat16)
    b1, b2 = torch.zeros(200, device="cuda"), torch.zeros(256, device="cuda")
    assert not dp_mlp_mse_supported(x, w1, b1, w2, b2, torch.zeros(384, 256, device="cuda", dtype=torch.bfloat16))
