"""The MLP autograd nodes (``dp_mlp_mse``, ``dp_mlp_cross_entropy``) and ``DPMLPModel`` bit for bit, at one rank,
against a float64 emulation of one node that rounds exactly where the kernels round.

test_gpu_exact_arithmetic.py checks each kernel alone.  This file checks the Python that wires them together: which
saved tensor each kernel reads, where the upstream gradient ``g`` is folded in, which ``needs_input_grad`` flags are
honoured, and the order of the reads and the in-place updates.  The tolerance tests in test_gpu_mlp.py and
test_gpu_xent.py cannot see a dropped ``g`` or a weight read after its own update; these tests can.

Exact inputs.  As in test_gpu_exact_arithmetic.py, every input is a small integer times a power of two, and every
premise is checked with its quanta bounds at every step: each GEMM, the loss, the column sums and the fp32 updates.
GELU is the one non-exact step, so every pre-activation z is either exactly 0 or has |z| >= 16 (a large |b1| plus a
small x W1^T).  There the tanh argument is over 150, ``tanhf`` is +-1, and the kernel's gelu_tanh / gelu_tanh_grad
give exactly h = z, gelu' = 1 (z > 0); h = -0, gelu' = +0 (z < 0); h = 0, gelu' = 1/2 (z = 0).  Each test checks
that premise on the kernel's own h first.  A "zero unit" reads a column of x that is 1 in every row, with W1 = 1/2
there and b1 = -1/2: z = 0 exactly, and its nonzero W1 entry carries dz into the gradient of x.

Cross-entropy.  All 256 real classes get equal logits (equal columns of W2 at the live units, equal biases), and 256
padded classes have bias -inf, a whole 256-column tile of them.  Then dy = ls (1/256 - onehot) exactly in bf16, and
everything downstream of dy is exact again.  The columns of W2 differ at the zero units (h = 0), so dy W2 is not zero
there.  The loss and the bias gradient of the output layer come from fp32 exp/log and are held to the derived bounds
of test_gpu_xent.py instead.
"""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_exact_arithmetic import (U24, _gen, assert_exact_gemm, assert_exact_loss, assert_loss_exact,
                                       assert_same_bits, exact_bf16, exact_f32, ints, mse_target, rne_bf16, ternary)

pytestmark = pytest.mark.gpu

SAT = 16.0        # |z| at or above which the kernel's tanhf is exactly +-1
N_REAL = 256      # real classes of the cross-entropy cases; as many padded ones follow
SMALL, RAGGED, BIG = (128, 256, 256, 256), (192, 256, 512, 384), (4096, 512, 2048, 1024)
SHAPES = [SMALL, RAGGED, BIG]  # BIG: the first GEMM has 32 x 8 = 256 tiles, more than an H100's SMs


# ------------------------------------------------------------------------------------------------------------------
# The float64 emulation (no GPU state: tests/test_exact_helpers.py runs it on the CPU)
# ------------------------------------------------------------------------------------------------------------------
def _no_check(*args, **kwargs):
    pass


def _exact_f32_or_skip(check):
    return exact_f32 if check else (lambda v: v)


def gelu_saturated(z, what=""):
    """h and gelu'(z) of the kernel for pre-activations that are 0 or have |z| >= 16 (asserted)."""
    ok = (z == 0) | (z.abs() >= SAT)
    assert bool(ok.all()), f"{what}: {int((~ok).sum())} pre-activations are neither 0 nor at least {SAT} in magnitude"
    h = torch.where(z > 0, z, torch.zeros_like(z))
    gp = torch.where(z > 0, torch.ones_like(z), torch.where(z == 0, torch.full_like(z, 0.5), torch.zeros_like(z)))
    return h, gp


def emulate_node(x, w1, b1, w2, b2, *, ls, g=1.0, target=None, labels=None, ignore_index=-100, rnd=rne_bf16,
                 check=True, what=""):
    """One node's forward and backward in float64.  ``rnd`` is the kernels' fp32 -> bf16 store (pass the identity to
    turn rounding off); with ``check`` every exactness premise is asserted.  Gives a dict with
      z, h, dy (as stored), dy32 (the fp32 dy the column sums add), loss, dz, dz32, gx,
      G1 = dz^T x and G2 = g dy^T h (unrounded), gw1, gw2 (rounded as wgrad_bf16 stores them), gb1, gb2.
    MSE with ``target``; softmax cross-entropy (sum over rows, ``ignore_index``) with ``labels``."""
    r = lambda v: rnd(v).double()  # noqa: E731
    chk = assert_exact_gemm if check else _no_check
    B = x.shape[0]
    chk(x, w1.t(), b1.expand(B, -1), what=f"{what} z")
    z32 = x @ w1.t() + b1
    gelu_saturated(z32, f"{what} z")
    z = r(z32)
    h, gp = gelu_saturated(z, f"{what} bf16 z")  # the kernel's h is gelu(fp32 z) = bf16 z, its gelu' is of bf16 z
    out = {"z": z, "h": h}
    if target is not None:
        chk(h, w2.t(), b2.expand(B, -1), target, what=f"{what} y - t")
        d = h @ w2.t() + b2 - target
        if check:
            assert_exact_loss(d, f"{what} loss")
        dy32 = 2.0 * ls * d
        loss = ls * d.square().sum()
    else:
        finite_b2 = torch.where(torch.isfinite(b2), b2, torch.zeros_like(b2))
        chk(h, w2.t(), finite_b2.expand(B, -1), what=f"{what} logits")
        logits = r(h @ w2.t() + b2)
        C = logits.shape[1]
        keep = (labels != ignore_index).double()
        onehot = F.one_hot(labels.clamp(0, C - 1), C).double()
        dy32 = ls * (torch.softmax(logits, 1) - onehot) * keep[:, None]
        picked = logits.gather(1, labels.clamp(0, C - 1)[:, None])[:, 0]
        loss = ls * (keep * (torch.logsumexp(logits, 1) - picked)).sum()
        out["logits"] = logits
    dy = r(dy32)
    chk(g * dy, w2, what=f"{what} dz")
    dz32 = g * (dy @ w2) * gp
    dz = r(dz32)
    chk(dz, w1, what=f"{what} gx")
    chk(g * dy.t(), h, what=f"{what} G2")
    chk(dz.t(), x, what=f"{what} G1")
    ones = torch.ones(1, B, dtype=x.dtype, device=x.device)
    chk(ones, g * dy32, what=f"{what} db2")
    chk(ones, dz32, what=f"{what} db1")
    G1, G2 = dz.t() @ x, g * (dy.t() @ h)
    out.update(dy=dy, dy32=dy32, loss=loss, dz=dz, dz32=dz32, gx=r(dz @ w1), G1=G1, G2=G2, gw1=r(G1), gw2=r(G2),
               gb1=dz32.sum(0), gb2=g * dy32.sum(0))
    return out


def emulate_sgd_in_backward(params, e, lr1, lr2, frozen=(), rnd=rne_bf16, check=True):
    """The in-backward update of one node: W <- bf16(W - lr G) from the unrounded G (one rounding, in the wgrad
    epilogue), b <- b - lr gb in fp32.  ``frozen``: indices into (w1, b1, w2, b2) left unchanged.  With ``check``,
    lr G and W - lr G (lr gb and b - lr gb) must be exact in fp32."""
    f32 = _exact_f32_or_skip(check)
    steps = (lr1 * e["G1"], lr1 * e["gb1"], lr2 * e["G2"], lr2 * e["gb2"])
    new = []
    for i, (p, s) in enumerate(zip(params, steps)):
        v = p if i in frozen else f32(p - f32(s))
        new.append(rnd(v).double() if i % 2 == 0 and i not in frozen else v)
    return new


def emulate_sgd_plain(params, grads, lr, rnd=rne_bf16, check=True):
    """``train_step``'s update: W <- bf16(fp32(W - lr gW)) (torch's bf16 add_) and b <- b - lr gb in fp32."""
    f32 = _exact_f32_or_skip(check)
    w1, b1, w2, b2 = params
    gw1, gb1, gw2, gb2 = grads
    return [rnd(f32(w1 - lr * gw1)).double(), f32(b1 - lr * gb1), rnd(f32(w2 - lr * gw2)).double(), f32(b2 - lr * gb2)]


# ------------------------------------------------------------------------------------------------------------------
# Exact cases
# ------------------------------------------------------------------------------------------------------------------
def hidden_layer(B, D, H, gen, zero_units=True):
    """x (ternary, column 0 all ones), W1 and b1 with every z = 0 or |z| in [16, 32]: positive units (b1 in
    [20, 28]), negative units (b1 in [-28, -20]) and, with ``zero_units``, zero units.  W1 of a live unit is
    ternary / 4 with about 8 nonzeros, so |x W1^T| <= 4."""
    x = ternary((B, D), 0.25, gen)
    x[:, 0] = 1.0
    k = ints((H,), 3, gen)
    kind = torch.where(k >= 1, 1.0, torch.where(k <= -2, -1.0, 0.0 if zero_units else 1.0))
    live = kind != 0
    w1 = ternary((H, D), min(1.0, 8.0 / D), gen, 0.25) * live.double()[:, None]
    w1[:, 0] = torch.where(live, 0.0, 0.5)
    b1 = torch.where(live, kind * (20.0 + ints((H,), 8, gen).abs()), torch.full_like(kind, -0.5))
    return x, w1, b1, kind


def output_weights(O, kind, gen, live_nnz):
    """W2 [O, H] in {-1/8, 0, 1/8}: about ``live_nnz`` nonzeros per row at the positive units (few, so most y are
    exact in bf16 and the target can match them), denser at the units with h = 0."""
    n_pos = max(1, int((kind > 0).sum()))
    dens = torch.where(kind > 0, min(1.0, live_nnz / n_pos), 0.25)
    keep = torch.rand((O, kind.shape[0]), generator=gen, device=gen.device, dtype=torch.float64) < dens
    return ternary((O, kind.shape[0]), 1.0, gen, 0.125) * keep


def mse_case(B, D, H, O, gen, zero_units=True):
    big = B * O > 2 ** 20
    x, w1, b1, kind = hidden_layer(B, D, H, gen, zero_units)
    w2 = output_weights(O, kind, gen, 1.0 if big else 2.0)
    b2 = ints((O,), 16, gen, 2.0 ** -5)
    z = x @ w1.t() + b1
    v = torch.where(z > 0, z, 0.0) @ w2.t() + b2
    t = mse_target(v, gen, 1 / 64 if big else 1 / 8)
    return x, w1, b1, w2, b2, t


def xent_case(B, D, H, gen, ignore_index):
    """256 real classes with equal logits in every row, then 256 padded classes with bias -inf.  W2 is equal across
    the real classes at the positive units and differs at the zero and negative units (h = 0)."""
    C = 2 * N_REAL
    x, w1, b1, kind = hidden_layer(B, D, H, gen)
    w2 = output_weights(C, kind, gen, 4.0)
    pos = kind > 0
    w2[:N_REAL, pos] = w2[0, pos]
    b2 = torch.cat([torch.full((N_REAL,), 0.25, dtype=torch.float64, device=x.device),
                    torch.full((C - N_REAL,), float("-inf"), dtype=torch.float64, device=x.device)])
    labels = torch.randint(0, N_REAL, (B,), generator=gen, device=gen.device)
    labels[::5] = ignore_index
    labels[-1] = N_REAL - 1
    return x, w1, b1, w2, b2, labels


# ------------------------------------------------------------------------------------------------------------------
# GPU side
# ------------------------------------------------------------------------------------------------------------------
def _comm():
    import mpi4torch_b200 as m4t

    comm = m4t.COMM_WORLD
    assert comm.size == 1 and m4t.cuda_backend_ready()
    return comm


def _device_params(x, w1, b1, w2, b2, requires=(True,) * 5):
    ts = [exact_bf16(x), exact_bf16(w1), exact_f32(b1), exact_bf16(w2), exact_f32(b2)]
    return [t.requires_grad_(q) for t, q in zip(ts, requires)]


def _check_saturation(h, z, what):
    """The premise on the kernel's own output: h equals the saturated rule of its own z, by value."""
    z64 = z.double()
    gelu_saturated(z64, what)
    assert_same_bits(h, torch.where(z64 > 0, z64, 0.0).to(torch.bfloat16), f"{what}: saturated GELU")


def _check_saved(local, e, what):
    """z, h and dy from the node's saved tensors (x, h, z, dy, w1_avg, w2_avg, dy_part)."""
    _, h, z, dy, _, _, _ = local.grad_fn.saved_tensors
    _check_saturation(h, z, what)
    assert_same_bits(z, exact_bf16(e["z"]), f"{what} z")
    assert_same_bits(h, exact_bf16(e["h"]), f"{what} h")
    assert_same_bits(dy, exact_bf16(e["dy"]), f"{what} dy")


def _check_grads(grads, e, what, names=("x", "w1", "b1", "w2", "b2")):
    keys = {"x": "gx", "w1": "gw1", "b1": "gb1", "w2": "gw2", "b2": "gb2"}
    for name, got in zip(names, grads):
        want = e[keys[name]]
        want = exact_f32(want) if name.startswith("b") else exact_bf16(want)
        assert got is not None, f"{what}: no gradient for {name}"
        assert_same_bits(got, want, f"{what} grad {name}")


def _check_params(got, want, what):
    for name, p, w in zip(("w1", "b1", "w2", "b2"), got, want):
        assert p.grad is None, f"{what}: in-backward mode left a .grad on {name}"
        assert_same_bits(p.detach(), exact_f32(w) if name.startswith("b") else exact_bf16(w), f"{what} {name}")


def _mse_node(x, w1, b1, w2, b2, t, ls, opts=None):
    from mpi4torch_b200.ops import dp_mlp_mse, dp_mlp_mse_supported

    comm = _comm()
    assert dp_mlp_mse_supported(x, w1, b1, w2, b2, t, comm)
    return dp_mlp_mse(x, w1, b1, w2, b2, t, comm, loss_scale=ls, optimizers=opts)


G_VALUES = [1.0, 2.0 ** -3, 3.0]
LS = 2.0 ** -3


@pytest.mark.parametrize("g", G_VALUES, ids=["g1", "g2^-3", "g3"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_mse_node_plain(shape, g):
    """loss, the saved z / h / dy, and the gradients of all five inputs under an upstream gradient g."""
    B, D, H, O = shape
    gen = _gen(*shape, int(8 * g), 1)
    x, w1, b1, w2, b2, t = mse_case(*shape, gen)
    what = f"{shape} g={g}"
    e = emulate_node(x, w1, b1, w2, b2, ls=LS, g=g, target=t, what=what)
    assert bool((e["dz"] != 0).any()) and bool((e["gx"] != 0).any()), "the case leaves dz or gx all zero"
    ins = _device_params(x, w1, b1, w2, b2)
    local = _mse_node(*ins, t, LS)
    _check_saved(local, e, what)
    assert_loss_exact(local.detach(), float(e["loss"]), f"{what} loss")
    grads = torch.autograd.grad(local, ins, grad_outputs=torch.full((1,), g, device="cuda"))
    _check_grads(grads, e, what)


PARTIAL = {"x": (True, False, False, False, False), "w2_b2": (False, False, False, True, True),
           "w1": (False, True, False, False, False), "biases": (False, False, True, False, True)}


@pytest.mark.parametrize("subset", list(PARTIAL))
def test_mse_node_partial_requires_grad(subset):
    """Only the requested gradients are returned, bit-identical to the full case; the others are None."""
    shape, g = RAGGED, 3.0
    x, w1, b1, w2, b2, t = mse_case(*shape, _gen(*shape, 2))
    e = emulate_node(x, w1, b1, w2, b2, ls=LS, g=g, target=t, what=subset)
    req = PARTIAL[subset]
    ins = _device_params(x, w1, b1, w2, b2, req)
    local = _mse_node(*ins, t, LS)
    local.backward(torch.full((1,), g, device="cuda"))
    names = ("x", "w1", "b1", "w2", "b2")
    for name, p, q in zip(names, ins, req):
        if q:
            _check_grads([p.grad], e, subset, (name,))
        else:
            assert p.grad is None, f"{subset}: {name} got a gradient"


def _opts(lr1, lr2):
    from mpi4torch_b200.ops import InBackwardSGD

    return (InBackwardSGD(lr1), InBackwardSGD(lr2))


LR1, LR2 = 2.0 ** 2, 2.0 ** 2  # large enough that most updates move the bf16 weights


@pytest.mark.parametrize("g", [1.0, 3.0], ids=["g1", "g3"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_mse_node_in_backward(shape, g):
    """Optimizer-in-backward with x.requires_grad: the four parameters updated bit for bit, no .grad left, and
    x's gradient from W1 as it was before its update."""
    gen = _gen(*shape, int(g), 3)
    x, w1, b1, w2, b2, t = mse_case(*shape, gen)
    what = f"{shape} g={g} in-backward"
    e = emulate_node(x, w1, b1, w2, b2, ls=LS, g=g, target=t, what=what)
    want = emulate_sgd_in_backward([w1, b1, w2, b2], e, LR1, LR2)
    for i, name in enumerate(("w1", "b1", "w2", "b2")):
        assert not torch.equal(want[i], [w1, b1, w2, b2][i]), f"{what}: the case does not move {name}"
    ins = _device_params(x, w1, b1, w2, b2)
    local = _mse_node(*ins, t, LS, _opts(LR1, LR2))
    _check_saved(local, e, what)
    (gx,) = torch.autograd.grad(local, [ins[0]], grad_outputs=torch.full((1,), g, device="cuda"))
    _check_grads([gx], e, what, ("x",))
    _check_params(ins[1:], want, what)


@pytest.mark.parametrize("frozen", range(4), ids=["w1", "b1", "w2", "b2"])
def test_mse_in_backward_frozen_parameter(frozen):
    """A parameter with requires_grad=False stays unchanged bit for bit; the other three take their update."""
    shape, g = RAGGED, 2.0 ** -1
    x, w1, b1, w2, b2, t = mse_case(*shape, _gen(*shape, 4))
    e = emulate_node(x, w1, b1, w2, b2, ls=LS, g=g, target=t)
    want = emulate_sgd_in_backward([w1, b1, w2, b2], e, LR1, LR2, frozen=(frozen,))
    req = [True] * 5
    req[1 + frozen] = False
    ins = _device_params(x, w1, b1, w2, b2, req)
    local = _mse_node(*ins, t, LS, _opts(LR1, LR2))
    local.backward(torch.full((1,), g, device="cuda"))
    _check_params(ins[1:], want, f"frozen {('w1', 'b1', 'w2', 'b2')[frozen]}")


def _two_batches(shape, seed):
    gen = _gen(*shape, seed)
    x, w1, b1, w2, b2, ta = mse_case(*shape, gen)
    xb = ternary(x.shape, 0.25, gen)
    xb[:, 0] = 1.0
    z = xb @ w1.t() + b1
    tb = mse_target(torch.where(z > 0, z, 0.0) @ w2.t() + b2, gen, 1 / 8)
    return (w1, b1, w2, b2), (x, ta), (xb, tb)


def test_stacked_forwards_plain():
    """Two forwards, one backward of the sum: .grad is the sum of both nodes' gradients, rounded once more where it
    is accumulated (bf16 for the weights, fp32 for the biases)."""
    params, (xa, ta), (xb, tb) = _two_batches(SMALL, 5)
    ea = emulate_node(xa, *params, ls=LS, target=ta, what="node a")
    eb = emulate_node(xb, *params, ls=LS, target=tb, what="node b")
    w1, b1, w2, b2 = _device_params(xa, *params)[1:]
    xa_d, xb_d = exact_bf16(xa).requires_grad_(), exact_bf16(xb).requires_grad_()
    la = _mse_node(xa_d, w1, b1, w2, b2, ta, LS)
    lb = _mse_node(xb_d, w1, b1, w2, b2, tb, LS)
    (la + lb).backward()
    _check_grads([xa_d.grad], ea, "node a", ("x",))
    _check_grads([xb_d.grad], eb, "node b", ("x",))
    for name, p in (("w1", w1), ("w2", w2)):
        k = "g" + name
        want = rne_bf16(exact_bf16(ea[k]).double() + exact_bf16(eb[k]).double())
        assert_same_bits(p.grad, want, f"accumulated grad {name}")
    for name, p in (("b1", b1), ("b2", b2)):
        k = "g" + name
        want = exact_f32(exact_f32(ea[k]).double() + exact_f32(eb[k]).double())
        assert_same_bits(p.grad, want, f"accumulated grad {name}")


def test_stacked_forwards_in_backward_raise():
    """Two forwards, one backward, with InBackwardSGD: the second node to run raises, naming the cause, and the
    parameters hold exactly one node's update (either order)."""
    params, (xa, ta), (xb, tb) = _two_batches(SMALL, 6)
    wants = []
    for x, t in ((xa, ta), (xb, tb)):
        e = emulate_node(x, *params, ls=LS, target=t)
        wants.append(emulate_sgd_in_backward(list(params), e, LR1, LR2))
    ins = _device_params(xa, *params)[1:]
    opts = _opts(LR1, LR2)
    la = _mse_node(exact_bf16(xa), *ins, ta, LS, opts)
    lb = _mse_node(exact_bf16(xb), *ins, tb, LS, opts)
    with pytest.raises(RuntimeError, match="one backward per forward"):
        (la + lb).backward()
    torch.cuda.synchronize()
    errors = []
    for name, want in zip(("node a", "node b"), wants):
        try:
            _check_params(ins, want, f"update of {name}")
            return
        except AssertionError as err:
            errors.append(str(err))
    raise AssertionError("the parameters hold neither node's update alone: " + "; ".join(errors))


def test_in_backward_sequential_forwards_still_run():
    """The stale-weight check does not fire in the normal pattern: forward, backward, forward, backward.  The first
    step is checked bit for bit; the second must run and move the weights (its inputs are no longer exact)."""
    params, (xa, ta), (xb, tb) = _two_batches(SMALL, 7)
    want = emulate_sgd_in_backward(list(params), emulate_node(xa, *params, ls=LS, target=ta), LR1, LR2)
    ins = _device_params(xa, *params)[1:]
    opts = _opts(LR1, LR2)
    _mse_node(exact_bf16(xa), *ins, ta, LS, opts).backward()
    _check_params(ins, want, "first step")
    before = [p.detach().clone() for p in ins]
    _mse_node(exact_bf16(xb), *ins, tb, LS, opts).backward()
    assert not torch.equal(ins[2].detach(), before[2]), "the second step did not update w2"
    assert opts[0].updates == opts[1].updates == 2


@pytest.mark.parametrize("sgd_in_backward", [True, False])
@pytest.mark.parametrize("shape", [SMALL, (256, 256, 512, 384)], ids=lambda s: "x".join(map(str, s)))
def test_dp_mlp_model_step_bitwise(shape, sgd_in_backward):
    """One DPMLPModel step at one rank (loss_scale = 1/B, g = 1) in each optimizer mode, checking the saturation
    premise on the kernel's h first.  Only one step is exact: the update gives the bf16 weights and the fp32 b1
    (about 24) fine low bits, and the second step's sums then exceed the exact bound."""
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.models import DPMLPModel

    B, D, H, O = shape
    x, w1, b1, w2, b2, t = mse_case(*shape, _gen(*shape, int(sgd_in_backward), 8))
    lr = 2.0 ** 2
    model = DPMLPModel(D, H, O, m4t.COMM_WORLD, device="cuda", lr=lr, sgd_in_backward=sgd_in_backward)
    with torch.no_grad():
        for p, v in zip(model.parameters(), (exact_bf16(w1), exact_f32(b1), exact_bf16(w2), exact_f32(b2))):
            p.copy_(v)
    params = [w1, b1, w2, b2]
    what = f"{shape} sgd_in_backward={sgd_in_backward}"
    e = emulate_node(x, *params, ls=1.0 / B, target=t, what=what)
    if sgd_in_backward:
        new = emulate_sgd_in_backward(params, e, lr, lr)
    else:
        new = emulate_sgd_plain(params, [e["gw1"], e["gb1"], e["gw2"], e["gb2"]], lr)
    assert all(not torch.equal(a, b) for a, b in zip(new, params)), f"{what}: the case leaves a parameter unchanged"
    h, z_k = torch.ops.mpi4torch_b200.linear_bias_gelu_forward(exact_bf16(x), model.w1.detach(), model.b1.detach())
    _check_saturation(h, z_k, what)
    loss = model.train_step(exact_bf16(x), t)
    assert_loss_exact(loss.reshape(1), float(e["loss"]), f"{what} loss")
    _check_params(model.parameters(), new, what)


# ------------------------------------------------------------------------------------------------------------------
# Cross-entropy
# ------------------------------------------------------------------------------------------------------------------
XENT_IGNORE = 3  # a real class: its rows add nothing


def _xent_bounds(e, labels, g, ls):
    """Derived bounds of test_gpu_xent.py on the fp32 loss and g * column sums of dy (real classes)."""
    from test_gpu_xent import _fp32_bounds, _reference

    logits = e["logits"][:, :N_REAL]
    p, lse, dy_ref, row = _reference(logits, labels, ls, ls, XENT_IGNORE)
    _, loss_err, colsum_err = _fp32_bounds(logits, p, lse, dy_ref, row, ls)
    return ls * loss_err, abs(g) * colsum_err + U24 * e["gb2"][:N_REAL].abs()


def _check_xent_forward(local, e, labels, g, ls, what):
    _check_saved(local, e, what)
    logits = e["logits"]
    assert bool((logits[:, :N_REAL] == logits[:, :1]).all()), f"{what}: the real logits of a row differ"
    loss_bound, _ = _xent_bounds(e, labels, g, ls)
    assert abs(float(local) - float(e["loss"])) <= loss_bound, f"{what}: loss {float(local)!r} vs {float(e['loss'])!r}"


def _check_b2(got, want, bound, what):
    """b2 (or its gradient) within the bound at the real classes, and bit for bit at the padded ones."""
    err = (got[:N_REAL].double() - want[:N_REAL]).abs()
    assert bool((err <= bound).all()), f"{what}: off by {float((err - bound).max()):.4g} over the bound"
    assert_same_bits(got[N_REAL:], want[N_REAL:].float(), f"{what} padded classes")


@pytest.mark.parametrize("sgd_in_backward", [False, True])
@pytest.mark.parametrize("shape", [SMALL[:3], BIG[:3]], ids=lambda s: "x".join(map(str, s)))
def test_xent_node(shape, sgd_in_backward):
    """The cross-entropy node with g = 3 and ignore_index = 3: the saved z / h / dy, gx, and the weight gradients
    (or updates) bit for bit; the loss and b2 within the derived fp32 bounds."""
    from mpi4torch_b200.ops import dp_mlp_cross_entropy, dp_mlp_cross_entropy_supported

    B, D, H = shape
    g, ls = 3.0, 2.0 ** -2
    x, w1, b1, w2, b2, labels = xent_case(B, D, H, _gen(*shape, 9), XENT_IGNORE)
    what = f"{shape} cross-entropy sgd_in_backward={sgd_in_backward}"
    e = emulate_node(x, w1, b1, w2, b2, ls=ls, g=g, labels=labels, ignore_index=XENT_IGNORE, what=what)
    for k in ("dz", "gx", "gw1", "gb1", "gw2"):
        assert bool((e[k] != 0).any()), f"{what}: the case leaves {k} all zero"
    ins = _device_params(x, w1, b1, w2, b2)
    comm = _comm()
    assert dp_mlp_cross_entropy_supported(*ins, labels, comm)
    opts = _opts(LR1, LR2) if sgd_in_backward else None
    local = dp_mlp_cross_entropy(*ins, labels, comm, loss_scale=ls, ignore_index=XENT_IGNORE, optimizers=opts)
    _check_xent_forward(local, e, labels, g, ls, what)
    _, gb2_bound = _xent_bounds(e, labels, g, ls)
    if not sgd_in_backward:
        grads = torch.autograd.grad(local, ins, grad_outputs=torch.full((1,), g, device="cuda"))
        _check_grads(grads[:4], e, what, ("x", "w1", "b1", "w2"))
        _check_b2(grads[4], e["gb2"], gb2_bound, f"{what} grad b2")
        return
    want = emulate_sgd_in_backward([w1, b1, w2, b2], e, LR1, LR2)
    (gx,) = torch.autograd.grad(local, [ins[0]], grad_outputs=torch.full((1,), g, device="cuda"))
    _check_grads([gx], e, what, ("x",))
    _check_params(ins[1:4], want[:3], what)
    _check_b2(ins[4].detach(), want[3], LR2 * gb2_bound + U24 * want[3][:N_REAL].abs(), f"{what} b2")


@pytest.mark.parametrize("sgd_in_backward", [False, True])
def test_dp_mlp_classifier_ignore_index(sgd_in_backward):
    """DPMLPClassifier(ignore_index=3): one step through the model with an upstream gradient of 3."""
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.models import DPMLPClassifier

    B, D, H = SMALL[:3]
    x, w1, b1, w2, b2, labels = xent_case(B, D, H, _gen(B, D, H, 10), XENT_IGNORE)
    lr, g = 2.0 ** 3, 3.0
    model = DPMLPClassifier(D, H, 2 * N_REAL, m4t.COMM_WORLD, device="cuda", lr=lr, sgd_in_backward=sgd_in_backward,
                            ignore_index=XENT_IGNORE)
    with torch.no_grad():
        for p, v in zip(model.parameters(), (exact_bf16(w1), exact_f32(b1), exact_bf16(w2), exact_f32(b2))):
            p.copy_(v)
    what = f"classifier sgd_in_backward={sgd_in_backward}"
    ls = 1.0 / B
    e = emulate_node(x, w1, b1, w2, b2, ls=ls, g=g, labels=labels, ignore_index=XENT_IGNORE, what=what)
    loss = model.loss(exact_bf16(x), labels)
    loss_bound, gb2_bound = _xent_bounds(e, labels, g, ls)
    assert abs(float(loss) - float(e["loss"])) <= loss_bound, f"{what}: loss {float(loss)!r} vs {float(e['loss'])!r}"
    (g * loss).backward()
    w1_k, b1_k, w2_k, b2_k = model.parameters()
    if sgd_in_backward:
        want = emulate_sgd_in_backward([w1, b1, w2, b2], e, lr, lr)
        _check_params([w1_k, b1_k, w2_k], want[:3], what)
        _check_b2(b2_k.detach(), want[3], lr * gb2_bound + U24 * want[3][:N_REAL].abs(), f"{what} b2")
    else:
        _check_grads([w1_k.grad, b1_k.grad, w2_k.grad], e, what, ("w1", "b1", "w2"))
        _check_b2(b2_k.grad, e["gb2"], gb2_bound, f"{what} grad b2")
