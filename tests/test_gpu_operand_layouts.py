"""The wgmma ops on operands that are not fresh contiguous tensors.

* Every op on interior views of NaN-filled buffers (leading dimension above the width, base offsets that keep the
  documented alignment): the result matches the fp32 reference, is bit-identical to the same op on contiguous
  copies, and no byte outside the views changes.  NaN x 0 is NaN, so a kernel that reads a neighbouring column or
  row (a tensor map with the leading dimension as its extent, a K tail, an epilogue read past N) shows it.
* Layouts the kernels cannot read in place: the ``*_supported`` predicates say so, and the ops raise on the host
  without launching anything.  That includes epilogue operands the kernels read with vector loads (MSE target,
  GELU input z, bias) at a misaligned base or row stride.
* The functional paths (``dp_linear_mse``, ``dp_mlp_mse``) run the torch composition on such inputs.
* Outputs of more than 2^31 elements, checked against references computed in row chunks.
"""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_gemm import _assert_close_bf16
from test_gpu_mlp import _assert_colsum, _gen, _launches, _ops, _reference_steps

pytestmark = pytest.mark.gpu

NAN = float("nan")
BF16 = torch.bfloat16
TN_SHAPES = [(300, 520, 200), (4100, 4104, 1000)]  # (M, N, K): one wave of ragged tiles, then more tiles than SMs
WGRAD_SHAPES = [(192, 384, 640), (1088, 4096, 4224)]  # (batch, N, K) with K % 256 != 0: a half-width last tile
LD_PADS = [16, 64]  # leading dimension = width + pad


def _rand(g, *shape, scale=1.0):
    return torch.randn(*shape, device="cuda", generator=g, dtype=BF16) * scale


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


class _Padded:
    """`data` copied into the interior of a NaN-filled buffer: two NaN rows (elements, for a vector) on each side
    and, for a matrix, 8 NaN columns on the left and a leading dimension of width + ld_pad.  The view keeps the
    alignment the ops document: 16 bytes for a bf16 matrix, 8 bytes for an fp32 vector."""

    def __init__(self, data, ld_pad=16):
        if data.dim() == 1:
            self.buf = torch.full((data.shape[0] + 4,), NAN, dtype=data.dtype, device="cuda")
            region = (slice(2, 2 + data.shape[0]),)
        else:
            rows, cols = data.shape
            self.buf = torch.full((rows + 4, cols + ld_pad), NAN, dtype=data.dtype, device="cuda")
            region = (slice(2, 2 + rows), slice(8, 8 + cols))
        self.view = self.buf[region]
        self.view.copy_(data)
        self._outside = torch.ones(self.buf.shape, dtype=torch.bool, device="cuda")
        self._outside[region] = False
        self._before = _bits(self.buf).clone()  # compared as integers: NaN != NaN

    def fresh(self):
        """A contiguous copy of the view in a new allocation."""
        return self.view.clone(memory_format=torch.contiguous_format)

    def assert_padding_intact(self, what):
        now = _bits(self.buf)
        assert torch.equal(now[self._outside], self._before[self._outside]), f"{what}: padding overwritten"

    def assert_intact(self, what):
        assert torch.equal(_bits(self.buf), self._before), f"{what}: input buffer modified"


def _assert_dy(dy, ref_dy, what):
    err = (dy.float() - ref_dy).abs().max().item()
    assert err <= 2e-2 * ref_dy.abs().max().item() + 1e-6, f"{what}: dL/dy max abs err {err}"


def _assert_loss(loss, ref_loss, what):
    assert abs(float(loss) - ref_loss) <= 2e-3 * abs(ref_loss), f"{what}: loss {float(loss)} vs {ref_loss}"


def _assert_same_loss(loss, loss_contiguous, what):
    """The loss comes from float atomics, whose order differs from call to call."""
    a, b = float(loss), float(loss_contiguous)
    assert abs(a - b) <= 1e-4 * abs(b), f"{what}: loss {a} on views vs {b} on contiguous copies"


def _assert_gelu(h, z_ref, K, what):
    """h = gelu_tanh(z) from the fp32 z: z's error (gelu' <= 1.13) plus the bf16 rounding of h."""
    h_ref = F.gelu(z_ref, approximate="tanh")
    err = (h.float() - h_ref).abs()
    floor = 1.2 * (2.0 ** -7 * z_ref.abs() + 2.0 ** -9 * K ** 0.5) + 2.0 ** -8 * h_ref.abs()
    assert bool((err <= floor).all()), f"{what}: h off by up to {float((err - floor).max()):.4g}"


def _gelu_grad_ref(dy, w, z, scale):
    """scale * (dy @ w) * gelu_tanh'(z) by torch autograd in fp32."""
    zz = z.float().requires_grad_()
    F.gelu(zz, approximate="tanh").backward(scale * (dy.float() @ w.float()))
    return zz.grad


def _assert_gelu_grad(dz, ref, K, scale, what):
    err = (dz.float() - ref).abs()
    floor = 2.0 ** -7 * ref.abs() + 1.2 * scale * 2.0 ** -9 * K ** 0.5
    assert bool((err <= floor).all()), f"{what}: dz off by up to {float((err - floor).max()):.4g}"


# ---- 1. every op on interior views of NaN-filled buffers ---------------------------------------------------------
@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", TN_SHAPES)
def test_gemm_bf16_tn_on_views(shape, ld_pad):
    ops = _ops()
    M, N, K = shape
    what = f"gemm_bf16_tn {shape} ld=width+{ld_pad}"
    g = _gen(M, N, K, ld_pad)
    x, w = _Padded(_rand(g, M, K), ld_pad), _Padded(_rand(g, N, K), ld_pad)
    assert ops.gemm_bf16_tn_supported(x.view, w.view)
    y = ops.gemm_bf16_tn(x.view, w.view)
    _assert_close_bf16(y, x.view.float() @ w.view.float().t(), K=K, what=what)
    assert torch.equal(y, ops.gemm_bf16_tn(x.fresh(), w.fresh())), what
    x.assert_intact(what)
    w.assert_intact(what)


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", TN_SHAPES)
def test_gemm_bf16_nn_on_views(shape, ld_pad):
    ops = _ops()
    M, N, K = shape
    what = f"gemm_bf16_nn {shape} ld=width+{ld_pad}"
    g = _gen(M, N, K, ld_pad, 1)
    a, b = _Padded(_rand(g, M, K), ld_pad), _Padded(_rand(g, K, N), ld_pad)
    assert ops.gemm_bf16_nn_supported(a.view, b.view)
    y = ops.gemm_bf16_nn(a.view, b.view)
    _assert_close_bf16(y, a.view.float() @ b.view.float(), K=K, what=what)
    assert torch.equal(y, ops.gemm_bf16_nn(a.fresh(), b.fresh())), what
    a.assert_intact(what)
    b.assert_intact(what)


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", WGRAD_SHAPES)
def test_wgrad_bf16_on_views(shape, ld_pad):
    ops = _ops()
    Mb, N, K = shape
    what = f"wgrad_bf16 {shape} ld=width+{ld_pad}"
    g = _gen(Mb, N, K, ld_pad, 2)
    dy, x = _Padded(_rand(g, Mb, N), ld_pad), _Padded(_rand(g, Mb, K), ld_pad)
    gs = torch.full((1,), 3.0, device="cuda")
    assert ops.wgrad_bf16_supported(dy.view, x.view)
    gw = ops.wgrad_bf16(dy.view, x.view, gs)
    _assert_close_bf16(gw, 3.0 * (dy.view.float().t() @ x.view.float()), K=Mb, what=what)
    assert torch.equal(gw, ops.wgrad_bf16(dy.fresh(), x.fresh(), gs)), what
    dy.assert_intact(what)
    x.assert_intact(what)


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", WGRAD_SHAPES)
def test_wgrad_sgd_on_views(shape, ld_pad):
    """The in-place update writes w through its own leading dimension (> K) and nothing around it."""
    ops = _ops()
    Mb, N, K = shape
    what = f"wgrad_sgd_ {shape} ld=width+{ld_pad}"
    g = _gen(Mb, N, K, ld_pad, 3)
    dy, x = _Padded(_rand(g, Mb, N), ld_pad), _Padded(_rand(g, Mb, K), ld_pad)
    w0 = _rand(g, N, K, scale=4.0)
    w, w_contiguous = _Padded(w0, ld_pad), w0.clone()
    gs = torch.full((1,), 3.0, device="cuda")
    ops.wgrad_sgd_(w.view, dy.view, x.view, -0.01, gs)
    ops.wgrad_sgd_(w_contiguous, dy.fresh(), x.fresh(), -0.01, gs)
    _assert_close_bf16(w.view, w0.float() - 0.03 * (dy.view.float().t() @ x.view.float()), K=Mb, what=what)
    assert torch.equal(w.view, w_contiguous), what
    w.assert_padding_intact(what)
    dy.assert_intact(what)
    x.assert_intact(what)


@pytest.mark.parametrize("local", [False, True])
@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", TN_SHAPES)
def test_linear_mse_forward_on_views(shape, ld_pad, local):
    """linear_mse_forward at one rank (no average) and linear_mse_forward_local: GEMM + MSE epilogue."""
    ops = _ops()
    M, N, K = shape
    what = f"linear_mse_forward{'_local' if local else ''} {shape} ld=width+{ld_pad}"
    g = _gen(M, N, K, ld_pad, 4 + local)
    x, w, t = _Padded(_rand(g, M, K), ld_pad), _Padded(_rand(g, N, K, scale=K ** -0.5), ld_pad), _Padded(_rand(g, M, N), ld_pad)
    loss_scale, grad_scale = 1.0 / M, 2.0 / M

    def run(*a):
        if local:
            return ops.linear_mse_forward_local(*a, loss_scale, grad_scale)
        return ops.linear_mse_forward(*a, 1.0, loss_scale, grad_scale, True)[:2]

    dy, loss = run(x.view, w.view, t.view)
    d = x.view.float() @ w.view.float().t() - t.view.float()
    _assert_dy(dy, grad_scale * d, what)
    _assert_loss(loss, loss_scale * d.double().square().sum().item(), what)
    dy_c, loss_c = run(x.fresh(), w.fresh(), t.fresh())
    assert torch.equal(dy, dy_c), what
    _assert_same_loss(loss, loss_c, what)
    for p in (x, w, t):
        p.assert_intact(what)


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", TN_SHAPES)
def test_linear_bias_gelu_forward_on_views(shape, ld_pad):
    ops = _ops()
    M, N, K = shape
    what = f"linear_bias_gelu_forward {shape} ld=width+{ld_pad}"
    g = _gen(M, N, K, ld_pad, 6)
    x, w = _Padded(_rand(g, M, K), ld_pad), _Padded(_rand(g, N, K, scale=K ** -0.5), ld_pad)
    b = _Padded(torch.randn(N, device="cuda", generator=g))
    h, z = ops.linear_bias_gelu_forward(x.view, w.view, b.view)
    z_ref = x.view.float() @ w.view.float().t() + b.view
    _assert_close_bf16(z, z_ref, K=K, what=f"{what} z")
    _assert_gelu(h, z_ref, K, what)
    h_c, z_c = ops.linear_bias_gelu_forward(x.fresh(), w.fresh(), b.fresh())
    assert torch.equal(h, h_c) and torch.equal(z, z_c), what
    for p in (x, w, b):
        p.assert_intact(what)


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", TN_SHAPES)
def test_linear_bias_mse_forward_local_on_views(shape, ld_pad):
    ops = _ops()
    M, N, K = shape
    what = f"linear_bias_mse_forward_local {shape} ld=width+{ld_pad}"
    g = _gen(M, N, K, ld_pad, 7)
    x, w = _Padded(_rand(g, M, K), ld_pad), _Padded(_rand(g, N, K, scale=K ** -0.5), ld_pad)
    b, t = _Padded(torch.randn(N, device="cuda", generator=g)), _Padded(_rand(g, M, N), ld_pad)
    loss_scale, grad_scale = 1.0 / M, 2.0 / M
    dy, loss, part = ops.linear_bias_mse_forward_local(x.view, w.view, b.view, t.view, loss_scale, grad_scale)
    d = x.view.float() @ w.view.float().t() + b.view - t.view.float()
    _assert_dy(dy, grad_scale * d, what)
    _assert_loss(loss, loss_scale * d.double().square().sum().item(), what)
    _assert_colsum(ops.column_sum(part), grad_scale * d, f"{what} dy column sum")
    dy_c, loss_c, part_c = ops.linear_bias_mse_forward_local(x.fresh(), w.fresh(), b.fresh(), t.fresh(), loss_scale,
                                                             grad_scale)
    assert torch.equal(dy, dy_c) and torch.equal(part, part_c), what
    _assert_same_loss(loss, loss_c, what)
    for p in (x, w, b, t):
        p.assert_intact(what)


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", TN_SHAPES)
def test_gemm_nn_gelu_backward_on_views(shape, ld_pad):
    ops = _ops()
    M, N, K = shape  # dy [M, K] @ w [K, N] -> dz [M, N]
    what = f"gemm_nn_gelu_backward {shape} ld=width+{ld_pad}"
    g = _gen(M, N, K, ld_pad, 8)
    dy, w, z = _Padded(_rand(g, M, K), ld_pad), _Padded(_rand(g, K, N), ld_pad), _Padded(_rand(g, M, N, scale=2.0), ld_pad)
    gs = torch.full((1,), 3.0, device="cuda")
    dz, part = ops.gemm_nn_gelu_backward(dy.view, w.view, z.view, gs)
    ref = _gelu_grad_ref(dy.view, w.view, z.view, 3.0)
    _assert_gelu_grad(dz, ref, K, 3.0, what)
    _assert_colsum(ops.column_sum(part), ref, f"{what} dz column sum")
    dz_c, part_c = ops.gemm_nn_gelu_backward(dy.fresh(), w.fresh(), z.fresh(), gs)
    assert torch.equal(dz, dz_c) and torch.equal(part, part_c), what
    for p in (dy, w, z):
        p.assert_intact(what)


@pytest.mark.parametrize("shape", [(19, 520), (257, 4104)])
def test_column_sum_on_view(shape):
    """The partials are contiguous by contract: here a contiguous view at an offset inside a NaN-filled buffer."""
    ops = _ops()
    what = f"column_sum {shape}"
    g = _gen(*shape)
    values = torch.randn(*shape, device="cuda", generator=g)
    flat = _Padded(values.flatten())
    part = flat.view.view(shape)
    gs = torch.full((1,), 3.0, device="cuda")
    out = ops.column_sum(part, gs)
    _assert_colsum(out, 3.0 * values, what)
    assert torch.equal(out, ops.column_sum(flat.fresh().view(shape), gs)), what
    flat.assert_intact(what)


# ---- 2. the predicates agree with the ops on layouts the kernels cannot read ---------------------------------------
LAYOUTS = {  # name -> can the wgmma GEMMs read such an operand in place?
    "contiguous": True,
    "column_slice": True,
    "offset_16B": True,
    "offset_2B": False,
    "offset_8B": False,
    "ld_not_multiple_of_8": False,
    "expand": False,
    "overlapping_rows": False,
}
LAYOUT_OPS = {  # op -> operand shapes
    "gemm_bf16_tn": ((130, 72), (264, 72)),
    "gemm_bf16_nn": ((130, 72), (72, 264)),
    "wgrad_bf16": ((192, 256), (192, 384)),
}


def _layout(data, name):
    """`data` [R, C] (or an fp32 vector for the offsets) in the named layout; "expand" and "overlapping_rows"
    derive their values from `data`.  Everything outside the view is NaN."""
    if name == "contiguous":
        return data.clone()
    if name == "expand":
        return data[:1].expand(data.shape)
    if name.startswith("offset_"):
        e = int(name[len("offset_"):-1]) // data.element_size()
        v = torch.full((data.numel() + 16,), NAN, dtype=data.dtype, device="cuda")[e:e + data.numel()].view(data.shape)
    else:
        R, C = data.shape
        if name == "overlapping_rows":  # leading dimension C - 8: aligned, but rows share elements
            return data.flatten()[: (R - 1) * (C - 8) + C].clone().as_strided((R, C), (C - 8, 1))
        off, ld = {"column_slice": (8, C + 24), "ld_not_multiple_of_8": (0, C + 4), "odd_ld": (0, C + 1)}[name]
        v = torch.full((off + R * ld,), NAN, dtype=data.dtype, device="cuda").as_strided((R, C), (ld, 1), off)
    v.copy_(data)
    return v


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("operand", [0, 1])
@pytest.mark.parametrize("op", list(LAYOUT_OPS))
def test_predicate_agrees_with_op(op, operand, layout):
    ops = _ops()
    what = f"{op} operand {operand} {layout}"
    g = _gen(len(op), operand, len(layout))
    args = [_rand(g, *s) for s in LAYOUT_OPS[op]]
    args[operand] = _layout(args[operand], layout)
    supported = bool(getattr(ops, op + "_supported")(*args))
    assert supported == LAYOUTS[layout], f"{what}: the predicate says {supported}"
    if supported:
        fresh = [a.clone(memory_format=torch.contiguous_format) for a in args]
        assert torch.equal(getattr(ops, op)(*args), getattr(ops, op)(*fresh)), what
    else:
        before = _launches()
        with pytest.raises(RuntimeError):
            getattr(ops, op)(*args)
        torch.cuda.synchronize()
        assert _launches() == before, f"{what}: a kernel was launched"


# ---- 3. misaligned epilogue operands are rejected on the host -------------------------------------------------------
EPILOGUE_CASES = [
    ("linear_mse_forward", "target", "offset_2B"),
    ("linear_mse_forward", "target", "odd_ld"),
    ("linear_mse_forward_local", "target", "offset_2B"),
    ("linear_mse_forward_local", "target", "odd_ld"),
    ("linear_bias_mse_forward_local", "target", "offset_2B"),
    ("linear_bias_mse_forward_local", "target", "odd_ld"),
    ("linear_bias_mse_forward_local", "bias", "offset_4B"),
    ("linear_bias_gelu_forward", "bias", "offset_4B"),
    ("gemm_nn_gelu_backward", "z", "offset_2B"),
    ("gemm_nn_gelu_backward", "z", "odd_ld"),
]


@pytest.mark.parametrize("op,operand,layout", EPILOGUE_CASES)
def test_misaligned_epilogue_operand_is_rejected(op, operand, layout):
    ops = _ops()
    M, N, K = 128, 256, 128
    what = f"{op} {operand} {layout}"
    g = _gen(M, N, K, len(what))
    x, w, t, z = _rand(g, M, K), _rand(g, N, K, scale=K ** -0.5), _rand(g, M, N), _rand(g, M, N, scale=2.0)
    b, w_kn = torch.randn(N, device="cuda", generator=g), _rand(g, K, N)
    if op != "gemm_nn_gelu_backward":
        assert ops.gemm_bf16_tn_supported(x, w, t, b)
    if operand == "target":
        t = _layout(t, layout)
        assert not ops.gemm_bf16_tn_supported(x, w, t), f"{what}: the predicate accepts the target"
    elif operand == "bias":
        b = _layout(b, layout)
        assert not ops.gemm_bf16_tn_supported(x, w, None, b), f"{what}: the predicate accepts the bias"
    else:
        z = _layout(z, layout)
    call = {
        "linear_mse_forward": lambda: ops.linear_mse_forward(x, w, t, 1.0, 1.0, 1.0, True),
        "linear_mse_forward_local": lambda: ops.linear_mse_forward_local(x, w, t, 1.0, 1.0),
        "linear_bias_mse_forward_local": lambda: ops.linear_bias_mse_forward_local(x, w, b, t, 1.0, 1.0),
        "linear_bias_gelu_forward": lambda: ops.linear_bias_gelu_forward(x, w, b),
        "gemm_nn_gelu_backward": lambda: ops.gemm_nn_gelu_backward(x, w_kn, z),
    }[op]
    before = _launches()
    with pytest.raises(RuntimeError, match="aligned"):
        call()
    torch.cuda.synchronize()
    assert _launches() == before, f"{what}: a kernel was launched"


# ---- 4. the functional paths fall back instead of raising or faulting -----------------------------------------------
MLP_KERNELS = ("gemm_bias_gelu", "gemm_bias_mse_colsum", "gemm_nn_gelu_bwd_colsum", "column_sum")


def _ran(before, after, name):
    return after.get(name, 0) - before.get(name, 0)


@pytest.mark.parametrize("which,nbytes", [("x", 2), ("target", 2), ("b1", 4)])
def test_dp_mlp_mse_falls_back_on_misaligned_operand(which, nbytes):
    from mpi4torch_b200.ops import dp_mlp_mse, dp_mlp_mse_supported

    _ops()
    B, D, H, O = 128, 128, 256, 128
    what = f"dp_mlp_mse with {which} at a {nbytes}-byte offset"
    g = _gen(B, D, H, O, nbytes)
    args = {"x": _rand(g, B, D), "w1": _rand(g, H, D, scale=D ** -0.5), "b1": 0.1 * torch.randn(H, device="cuda", generator=g),
            "w2": _rand(g, O, H, scale=H ** -0.5), "b2": 0.1 * torch.randn(O, device="cuda", generator=g),
            "target": _rand(g, B, O)}
    assert dp_mlp_mse_supported(*args.values()), f"{what}: the aligned inputs are off the kernel path"
    args[which] = _layout(args[which], f"offset_{nbytes}B")
    assert not dp_mlp_mse_supported(*args.values()), what
    params = [args[k].requires_grad_() for k in ("w1", "b1", "w2", "b2")]
    before = _launches()
    loss = dp_mlp_mse(*args.values(), loss_scale=1.0 / B)
    grads = torch.autograd.grad(loss, params)
    torch.cuda.synchronize()
    after = _launches()
    for n in MLP_KERNELS:
        assert _ran(before, after, n) == 0, f"{what}: {n} ran"
    # one SGD step of lr 1 in the fp32 reference: its gradient is the parameter change
    ref_losses, ref_params = _reference_steps(params, [args["x"]], [args["target"]], 1.0)
    assert abs(float(loss) - ref_losses[0]) <= 1e-2 * abs(ref_losses[0]), f"{what}: loss {float(loss)} vs {ref_losses[0]}"
    for name, p, grad, after_step in zip(("w1", "b1", "w2", "b2"), params, grads, ref_params):
        ref = p.detach().float() - after_step
        err = float((grad.float() - ref).abs().max())
        assert err <= 3e-2 * float(ref.abs().max()), f"{what}: d{name} off by {err}"


def _linear_reference(x, w, t):
    """fp32 loss sum((x w^T - t)^2) / B and its weight gradient."""
    wf = w.detach().float().requires_grad_()
    loss = (x.float() @ wf.t() - t.float()).square().sum() / x.shape[0]
    loss.backward()
    return float(loss), wf.grad


def test_dp_linear_mse_falls_back_on_misaligned_target():
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.ops import dp_linear_mse, dp_linear_mse_supported

    _ops()
    comm = m4t.COMM_WORLD
    B, D, N = 256, 256, 256
    g = _gen(B, D, N, 9)
    x, t = _rand(g, B, D), _rand(g, B, N)
    w = _rand(g, N, D, scale=D ** -0.5).requires_grad_()
    assert dp_linear_mse_supported(x, w, t, comm)
    t_off = _layout(t, "offset_2B")
    assert not dp_linear_mse_supported(x, w, t_off, comm)
    before = _launches()
    loss = dp_linear_mse(x, w, t_off, comm, loss_scale=1.0 / B)
    loss.backward()
    torch.cuda.synchronize()
    after = _launches()
    for n in ("gemm_mse_epilogue", "wgrad", "wgrad_sgd_epilogue"):
        assert _ran(before, after, n) == 0, f"{n} ran on a misaligned target"
    ref_loss, ref_grad = _linear_reference(x, w, t)
    assert abs(float(loss) - ref_loss) <= 1e-2 * ref_loss, (float(loss), ref_loss)
    err = float((w.grad.float() - ref_grad).abs().max())
    assert err <= 2e-2 * float(ref_grad.abs().max()), f"weight gradient off by {err}"


@pytest.mark.parametrize("in_backward_sgd", [False, True])
def test_dp_linear_mse_column_slice_input_stays_on_kernels(in_backward_sgd):
    """x with a leading dimension above D (aligned) runs the MSE-epilogue GEMM forward and the wgrad kernel (plain,
    or with the SGD step as its epilogue) backward, reading x in place."""
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.ops import InBackwardSGD, dp_linear_mse, dp_linear_mse_supported, in_backward_sgd_supported

    _ops()
    comm = m4t.COMM_WORLD
    B, D, N, lr = 256, 256, 256, 0.1
    g = _gen(B, D, N, 10 + in_backward_sgd)
    x, t = _Padded(_rand(g, B, D), 64), _rand(g, B, N)
    w = _rand(g, N, D, scale=D ** -0.5).requires_grad_()
    w0 = w.detach().clone()
    assert x.view.stride(0) > D and dp_linear_mse_supported(x.view, w, t, comm)
    opt = None
    if in_backward_sgd:
        assert in_backward_sgd_supported(x.view, w, comm)
        opt = InBackwardSGD(lr)
    before = _launches()
    loss = dp_linear_mse(x.view, w, t, comm, loss_scale=1.0 / B, optimizer=opt)
    mid = _launches()
    loss.backward()
    torch.cuda.synchronize()
    after = _launches()
    assert _ran(before, mid, "gemm_mse_epilogue") == 1
    assert _ran(mid, after, "wgrad_sgd_epilogue" if in_backward_sgd else "wgrad") == 1
    ref_loss, ref_grad = _linear_reference(x.view, w0, t)
    _assert_loss(loss, ref_loss, "dp_linear_mse on a column slice")
    if in_backward_sgd:
        assert w.grad is None
        ref_w = w0.float() - lr * ref_grad
        err = (w.detach().float() - ref_w).abs()
        bound = 2.0 ** -7 * ref_w.abs() + 2e-2 * lr * ref_grad.abs().max()
        assert bool((err <= bound).all()), f"updated weight off by up to {float((err - bound).max()):.4g}"
    else:
        err = float((w.grad.float() - ref_grad).abs().max())
        assert err <= 2e-2 * float(ref_grad.abs().max()), f"weight gradient off by {err}"
    x.assert_intact("dp_linear_mse x")


# ---- 5. outputs of more than 2^31 elements ----------------------------------------------------------------------
GiB = 1 << 30
BIG_M, BIG_N, BIG_K = 131072, 16392, 64
CHUNK = 8192  # rows of the reference per step (a multiple of 16: whole column-sum partial rows)


@pytest.fixture
def mem():
    """Holds a large case's tensors and frees them, with the allocator's cache, when the case ends, passed or not."""
    store = {}
    yield store
    store.clear()
    torch.cuda.empty_cache()


def _require_free(nbytes):
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    need = nbytes + 6 * GiB  # reference chunks, comparison temporaries and a margin
    if free < need:
        pytest.skip(f"needs {need / GiB:.1f} GiB of free device memory, {free / GiB:.1f} GiB free (the GPU is shared)")


def _chunks(rows, step=CHUNK):
    return [(r, min(rows, r + step)) for r in range(0, rows, step)]


def test_gemm_bf16_tn_output_beyond_2_31_elements(mem):
    assert BIG_M * BIG_N > 2 ** 31
    _require_free(BIG_M * BIG_N * 2)
    ops = _ops()
    g = _gen(BIG_M, BIG_N, BIG_K)
    mem["x"], mem["w"] = _rand(g, BIG_M, BIG_K), _rand(g, BIG_N, BIG_K)
    mem["y"] = ops.gemm_bf16_tn(mem["x"], mem["w"])
    for r0, r1 in _chunks(BIG_M):
        _assert_close_bf16(mem["y"][r0:r1], mem["x"][r0:r1].float() @ mem["w"].float().t(), K=BIG_K,
                           what=f"gemm_bf16_tn rows {r0}:{r1}")


def test_linear_bias_gelu_forward_output_beyond_2_31_elements(mem):
    _require_free(2 * BIG_M * BIG_N * 2)
    ops = _ops()
    g = _gen(BIG_M, BIG_N, BIG_K, 1)
    mem["x"], mem["w"] = _rand(g, BIG_M, BIG_K), _rand(g, BIG_N, BIG_K, scale=BIG_K ** -0.5)
    mem["b"] = torch.randn(BIG_N, device="cuda", generator=g)
    mem["h"], mem["z"] = ops.linear_bias_gelu_forward(mem["x"], mem["w"], mem["b"])
    for r0, r1 in _chunks(BIG_M):
        z_ref = mem["x"][r0:r1].float() @ mem["w"].float().t() + mem["b"]
        what = f"linear_bias_gelu_forward rows {r0}:{r1}"
        _assert_close_bf16(mem["z"][r0:r1], z_ref, K=BIG_K, what=what)
        _assert_gelu(mem["h"][r0:r1], z_ref, BIG_K, what)


def test_linear_bias_mse_forward_local_output_beyond_2_31_elements(mem):
    _require_free(2 * BIG_M * BIG_N * 2 + (BIG_M // 16) * BIG_N * 4)
    ops = _ops()
    g = _gen(BIG_M, BIG_N, BIG_K, 2)
    mem["x"], mem["w"] = _rand(g, BIG_M, BIG_K), _rand(g, BIG_N, BIG_K, scale=BIG_K ** -0.5)
    mem["b"], mem["t"] = torch.randn(BIG_N, device="cuda", generator=g), _rand(g, BIG_M, BIG_N)
    loss_scale, grad_scale = 1.0 / BIG_M, 2.0 / BIG_M
    mem["dy"], loss, mem["part"] = ops.linear_bias_mse_forward_local(mem["x"], mem["w"], mem["b"], mem["t"], loss_scale,
                                                                      grad_scale)
    ref_loss = 0.0
    for r0, r1 in _chunks(BIG_M):
        d = mem["x"][r0:r1].float() @ mem["w"].float().t() + mem["b"] - mem["t"][r0:r1].float()
        what = f"linear_bias_mse_forward_local rows {r0}:{r1}"
        _assert_dy(mem["dy"][r0:r1], grad_scale * d, what)
        _assert_colsum(ops.column_sum(mem["part"][r0 // 16:r1 // 16]), grad_scale * d, f"{what} column sum")
        ref_loss += loss_scale * d.double().square().sum().item()
    _assert_loss(loss, ref_loss, "linear_bias_mse_forward_local beyond 2^31")


def test_gemm_nn_gelu_backward_output_beyond_2_31_elements(mem):
    _require_free(2 * BIG_M * BIG_N * 2 + (BIG_M // 16) * BIG_N * 4)
    ops = _ops()
    g = _gen(BIG_M, BIG_N, BIG_K, 3)
    mem["dy"], mem["w"], mem["z"] = _rand(g, BIG_M, BIG_K), _rand(g, BIG_K, BIG_N), _rand(g, BIG_M, BIG_N, scale=2.0)
    gs = torch.full((1,), 3.0, device="cuda")
    mem["dz"], mem["part"] = ops.gemm_nn_gelu_backward(mem["dy"], mem["w"], mem["z"], gs)
    for r0, r1 in _chunks(BIG_M):
        ref = _gelu_grad_ref(mem["dy"][r0:r1], mem["w"], mem["z"][r0:r1], 3.0)
        what = f"gemm_nn_gelu_backward rows {r0}:{r1}"
        _assert_gelu_grad(mem["dz"][r0:r1], ref, BIG_K, 3.0, what)
        _assert_colsum(ops.column_sum(mem["part"][r0 // 16:r1 // 16]), ref, f"{what} column sum")


def test_wgrad_bf16_output_beyond_2_31_elements(mem):
    Mb, N = 64, 46464  # N x N > 2^31, N % 128 == 0
    assert N * N > 2 ** 31
    _require_free(N * N * 2)
    ops = _ops()
    g = _gen(Mb, N, 4)
    mem["dy"], mem["x"] = _rand(g, Mb, N), _rand(g, Mb, N)
    mem["gw"] = ops.wgrad_bf16(mem["dy"], mem["x"])
    for r0, r1 in _chunks(N, 4096):
        _assert_close_bf16(mem["gw"][r0:r1], mem["dy"][:, r0:r1].float().t() @ mem["x"].float(), K=Mb,
                           what=f"wgrad_bf16 rows {r0}:{r1}")
