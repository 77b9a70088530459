"""Softmax cross-entropy output layer of the MLP (``linear_bias_xent_forward_local``: the ``gemm_bias_xent`` GEMM
epilogue and ``xent_finish``) and ``DPMLPClassifier`` on one GPU.

Op level, the reference is float64 ``F.cross_entropy`` / softmax on the kernel's own bf16 logits.  With the exact
inputs of test_gpu_exact_arithmetic.py those logits are known bit for bit: ``rne_bf16(x @ w^T + b)`` of the float64
product.  What is left is fp32 arithmetic on them, bounded term by term (``_fp32_bounds``):
  * the row's ``lse``: every ``exp`` is off by <= 2 ulp (CUDA ``expf``), the sum of exps is added in at most
    ``n_add`` = 64 (a thread's values) + 2 (the quad) + ceil(C/256) (the tiles) + 16 (xent_finish's slots) steps,
    each rounding by <= u24 of the partial sum, and ``M + log(sum)`` rounds twice more; so
    |lse - lse_ref| <= (n_add + 8) u24 + 2 u24 |lse|.
  * ``p = exp(logit - lse)``: the argument carries the lse error plus one rounding (u24 |logit - lse|), exp adds
    2 ulp, so |p - p_ref| <= p_ref (lse_err + u24 |logit - lse| + 3 u24) (first order; the terms are < 1e-4).
  * ``dy = gs (p - onehot)`` (gs a power of two) rounds once in fp32 and once to bf16.
  * the row loss ``lse - logit[label]`` rounds once, and the fixed-order sum of M of them adds
    <= (M / 256 + 8) u24 sum |row loss|; the column sums of dy likewise add (16 + rows / 8 + 8) u24 sum |dy|.
  * a p below fp32's smallest normal (2^-126) may be lost outright: an absolute 2^-126 per element.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from test_gpu_exact_arithmetic import (U24, _gen, _rounded_bound, assert_exact_gemm, assert_same_bits, exact_bf16,
                                       exact_f32, ints, rne_bf16)

pytestmark = pytest.mark.gpu

IGNORE = -100
TILE_C = 256


def _ops():
    import mpi4torch_b200 as m4t

    m4t.COMM_WORLD  # bring the backend up
    return torch.ops.mpi4torch_b200


def _launches():
    import mpi4torch_b200 as m4t

    return dict(m4t._C.kernel_launch_table())


def _reference(logits, labels, ls, gs, ignore_index=IGNORE):
    """float64 reference on the bf16 logits: p, lse, dy, per-row loss (0 for ignored rows)."""
    z = logits.double()
    lse = torch.logsumexp(z, dim=1)
    p = torch.softmax(z, dim=1)
    C = z.shape[1]
    ignored = labels == ignore_index
    onehot = F.one_hot(labels.clamp(0, C - 1), C).double() * (~ignored).double()[:, None]
    dy = gs * (p - onehot) * (~ignored).double()[:, None]
    row = F.cross_entropy(z, labels, reduction="none", ignore_index=ignore_index)
    return p, lse, dy, row


def _fp32_bounds(logits, p, lse, dy, row, gs):
    M, C = logits.shape
    n_add = 64 + 2 + math.ceil(C / TILE_C) + 16
    z = logits.double()
    lse_err = (n_add + 8) * U24 + 2 * U24 * lse.abs()
    p_err = p * (lse_err[:, None] + U24 * (z - lse[:, None]).abs() + 3 * U24)
    # + 2^-126: a p below fp32's normal range may come out as 0 or subnormal
    dy32_err = abs(gs) * (p_err + U24 * (dy.abs() / abs(gs)) + 2.0 ** -126)
    loss_err = (lse_err + U24 * row.abs()).sum() + (M / 256 + 8) * U24 * row.abs().sum()
    colsum_err = dy32_err.sum(0) + (16 + math.ceil(M / 16) / 8 + 8) * U24 * dy.abs().sum(0) + M * 2.0 ** -126
    return dy32_err, float(loss_err), colsum_err


def _check_against_reference(ops, logits, labels, dy, loss, part, ls, gs, what):
    p, lse, dy_ref, row = _reference(logits, labels, ls, gs)
    dy32_err, loss_err, colsum_err = _fp32_bounds(logits, p, lse, dy_ref, row, gs)
    err = (dy.double() - dy_ref).abs()
    bound = _rounded_bound(dy_ref, dy32_err)
    assert bool((err <= bound).all()), f"{what}: dy off by {float((err - bound).max()):.4g} over the bound"
    ref_loss = ls * float(row.sum())
    assert abs(float(loss) - ref_loss) <= abs(ls) * loss_err, f"{what}: loss {float(loss)!r} vs {ref_loss!r}"
    assert part.shape == ((logits.shape[0] + 15) // 16, logits.shape[1]) and part.dtype == torch.float32
    db = ops.column_sum(part).double()
    cerr = (db - dy_ref.sum(0)).abs()
    assert bool((cerr <= colsum_err).all()), f"{what}: db off by {float((cerr - colsum_err).max()):.4g} over the bound"


def _exact_case(M, C, K, seed):
    """Exact inputs: x ints in [-3, 3], w ints in [-3, 3] / 8, bias ints in [-8, 8] / 4; logits below ~2^7."""
    g = _gen(M, C, K, seed)
    x = ints((M, K), 3, g)
    w = ints((C, K), 3, g, 2.0 ** -3)
    b = ints((C,), 8, g, 2.0 ** -2)
    assert_exact_gemm(x, w.t(), b[None, :].expand(M, C), what=f"{(M, C, K)}")
    logits = rne_bf16(x @ w.t() + b)
    labels = torch.randint(0, C, (M,), generator=g, device="cuda")
    labels[-1] = C - 1  # a label in the last (possibly ragged) tile
    return exact_bf16(x), exact_bf16(w), exact_f32(b), logits, labels


TILE_M = (1, 127, 128, 129)
TILE_C_EDGES = (8, 248, 256, 264, 384, 520)
TILE_K = (8, 72, 136)
EXACT_SHAPES = [(M, C, TILE_K[(i + j) % len(TILE_K)]) for i, M in enumerate(TILE_M) for j, C in enumerate(TILE_C_EDGES)]
# more tiles than SMs: 35 x 5 = 175 tiles of 128 x 256 (ragged in M and C) on a 132-SM H100
EXACT_SHAPES += [(128 * 35 - 3, 1032, 72)]


@pytest.mark.parametrize("shape", EXACT_SHAPES)
def test_xent_op_exact_inputs(shape):
    ops = _ops()
    M, C, K = shape
    x, w, b, logits, labels = _exact_case(M, C, K, 1)
    ls, gs = 2.0 ** -5, 2.0 ** -3
    dy, loss, part = ops.linear_bias_xent_forward_local(x, w, b, labels, ls, gs)
    torch.cuda.synchronize()
    assert dy.dtype == torch.bfloat16 and dy.shape == (M, C) and loss.shape == (1,)
    _check_against_reference(ops, logits, labels, dy, loss, part, ls, gs, f"{shape}")


@pytest.mark.parametrize("shape", [(129, 520, 72), (128 * 35 - 3, 1032, 72)])
def test_xent_determinism(shape):
    ops = _ops()
    x, w, b, _, labels = _exact_case(*shape, 2)
    labels[::7] = IGNORE
    a = ops.linear_bias_xent_forward_local(x, w, b, labels, 2.0 ** -5, 2.0 ** -5)
    c = ops.linear_bias_xent_forward_local(x, w, b, labels, 2.0 ** -5, 2.0 ** -5)
    for u, v, name in zip(a, c, ("dy", "loss", "partials")):
        assert torch.equal(u.view(torch.int16) if u.dtype == torch.bfloat16 else u.view(torch.int32),
                           v.view(torch.int16) if v.dtype == torch.bfloat16 else v.view(torch.int32)), name


def test_xent_ignore_index():
    """Ignored rows: a zero dy row bit for bit, and the loss and db equal those of the batch without them."""
    ops = _ops()
    M, C, K = 129, 264, 72
    x, w, b, logits, labels = _exact_case(M, C, K, 3)
    ls, gs = 2.0 ** -4, 2.0 ** -4
    lab = labels.clone()
    ign = torch.zeros(M, dtype=torch.bool, device="cuda")
    ign[::3] = True
    ign[-1] = False
    lab[ign] = IGNORE
    dy, loss, part = ops.linear_bias_xent_forward_local(x, w, b, lab, ls, gs)
    torch.cuda.synchronize()
    assert_same_bits(dy[ign], torch.zeros_like(dy[ign]), "ignored dy rows")
    _check_against_reference(ops, logits, lab, dy, loss, part, ls, gs, "ignore_index")
    # the same loss and db as the kept rows alone (fp32 sums of fewer terms: within the same bounds)
    keep = ~ign
    dy_k, loss_k, part_k = ops.linear_bias_xent_forward_local(x[keep].contiguous(), w, b, lab[keep].contiguous(), ls, gs)
    assert_same_bits(dy[keep], dy_k, "kept rows")
    _check_against_reference(ops, logits[keep], lab[keep], dy_k, loss_k, part_k, ls, gs, "kept rows alone")
    assert abs(float(loss) - float(loss_k)) <= 1e-6 * abs(float(loss_k))
    db, db_k = ops.column_sum(part), ops.column_sum(part_k)
    assert bool(((db - db_k).abs() <= 1e-6 * dy_k.float().abs().sum(0) + 1e-12).all())
    # a user-chosen ignore_index inside [0, C) ignores that class, as F.cross_entropy does
    dy2, loss2, _ = ops.linear_bias_xent_forward_local(x, w, b, labels, ls, gs, 5)
    ref = F.cross_entropy(logits.double(), labels, reduction="sum", ignore_index=5) * ls
    assert abs(float(loss2) - float(ref)) <= 1e-5 * abs(float(ref))
    assert_same_bits(dy2[labels == 5], torch.zeros_like(dy2[labels == 5]), "rows of ignored class 5")


def test_xent_out_of_range_labels():
    """Labels C, -1 and 2^40: that row's dy and the loss are NaN; every other row is unchanged bit for bit."""
    ops = _ops()
    M, C, K = 129, 264, 72
    x, w, b, _, labels = _exact_case(M, C, K, 4)
    ls, gs = 2.0 ** -5, 2.0 ** -5
    dy0, loss0, _ = ops.linear_bias_xent_forward_local(x, w, b, labels, ls, gs)
    assert not torch.isnan(loss0).any()
    for i, bad in enumerate((C, -1, 2 ** 40)):
        r = (17 * i + 5) % M
        lab = labels.clone()
        lab[r] = bad
        dy, loss, _ = ops.linear_bias_xent_forward_local(x, w, b, lab, ls, gs)
        torch.cuda.synchronize()
        assert torch.isnan(loss).all(), f"label {bad}: loss {float(loss)}"
        assert torch.isnan(dy[r]).all(), f"label {bad}: row {r} not NaN"
        others = torch.arange(M, device="cuda") != r
        assert_same_bits(dy[others], dy0[others], f"label {bad}: other rows")


def _pattern_case(L, idx, bias):
    """x = one-hot rows picking a row of L (bf16 [P, C]), w = L^T: logit[r] = L[idx[r]] + bias exactly (one nonzero
    product per output)."""
    P, C = L.shape
    K = max(8, (P + 7) // 8 * 8)
    x = torch.zeros(len(idx), K, device="cuda", dtype=torch.bfloat16)
    x[torch.arange(len(idx), device="cuda"), idx] = 1
    w = torch.zeros(C, K, device="cuda", dtype=torch.bfloat16)
    w[:, :P] = L.t()
    return x, w, bias.float().contiguous()


def test_xent_large_logits():
    """Logits near +-3e4: exp overflows without the max subtraction; the loss must stay finite and match."""
    ops = _ops()
    g = _gen(5)
    C, M = 384, 130
    base = torch.tensor([30000.0, -30000.0, 29952.0], device="cuda", dtype=torch.float64)
    L = (base[:, None] + ints((3, C), 4, g, 128.0)).to(torch.bfloat16)
    idx = torch.arange(M, device="cuda") % 3
    x, w, b = _pattern_case(L, idx, torch.zeros(C, device="cuda"))
    labels = torch.randint(0, C, (M,), generator=g, device="cuda")
    logits = L[idx]
    dy, loss, part = ops.linear_bias_xent_forward_local(x, w, b, labels, 2.0 ** -7, 2.0 ** -7)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all() and torch.isfinite(dy).all()
    _check_against_reference(ops, logits, labels, dy, loss, part, 2.0 ** -7, 2.0 ** -7, "logits near 3e4")


def test_xent_equal_logits_row():
    """A row of equal logits: p = 1/C everywhere, loss log C."""
    ops = _ops()
    M, C, K = 64, 520, 72
    x, w, b, logits, labels = _exact_case(M, C, K, 6)
    x[3] = 0
    b = torch.zeros_like(b)
    logits = rne_bf16(x.double() @ w.double().t())
    assert bool((logits[3] == 0).all())
    dy, loss, part = ops.linear_bias_xent_forward_local(x, w, b, labels, 1.0, 1.0)
    torch.cuda.synchronize()
    _check_against_reference(ops, logits, labels, dy, loss, part, 1.0, 1.0, "equal-logit row")
    want = torch.full((C,), 1.0 / C, device="cuda", dtype=torch.float64)
    want[labels[3]] -= 1.0
    assert_same_bits(dy[3], rne_bf16(want), "equal-logit row dy")


def test_xent_padded_classes_all_inf_tile():
    """200 real classes padded to 512 with bias -inf: the second 256-column tile is all -inf.  Padded dy is exactly 0
    and loss and dy match F.cross_entropy on the 200 real classes."""
    ops = _ops()
    M, C, K, n = 129, 512, 72, 200
    x, w, b, _, _ = _exact_case(M, C, K, 7)
    b[n:] = float("-inf")
    g = _gen(7, 1)
    labels = torch.randint(0, n, (M,), generator=g, device="cuda")
    logits = rne_bf16(x.double() @ w.double().t() + b.double())
    dy, loss, part = ops.linear_bias_xent_forward_local(x, w, b, labels, 2.0 ** -5, 2.0 ** -5)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    assert_same_bits(dy[:, n:], torch.zeros_like(dy[:, n:]), "padded classes' dy")
    _check_against_reference(ops, logits[:, :n], labels, dy[:, :n].contiguous(), loss,
                             part[:, :n].contiguous(), 2.0 ** -5, 2.0 ** -5, "200 of 512 classes")
    assert_same_bits(ops.column_sum(part)[n:], torch.zeros(C - n, device="cuda"), "padded classes' db")


def test_xent_nan_and_inf_logits_match_torch():
    """A NaN row of x, and a +inf bias (a +inf logit in every row): NaN wherever F.cross_entropy gives NaN."""
    ops = _ops()
    M, C, K = 129, 264, 72
    x, w, b, _, labels = _exact_case(M, C, K, 8)
    x[5] = float("nan")
    logits = rne_bf16(x.double() @ w.double().t() + b.double())
    dy, loss, _ = ops.linear_bias_xent_forward_local(x, w, b, labels, 1.0, 1.0)
    torch.cuda.synchronize()
    z = logits.double().requires_grad_()
    ref_row = F.cross_entropy(z, labels, reduction="none")
    ref_row.sum().backward()
    assert torch.isnan(loss).all() and bool(torch.isnan(ref_row).any())
    assert torch.equal(torch.isnan(dy), torch.isnan(z.grad)), "NaN positions of dy differ from torch's gradient"
    assert bool(torch.isnan(dy[5]).all()) and not bool(torch.isnan(dy[6]).any())
    # +inf logits: torch's log_softmax is NaN in every such row
    x, w, b, _, labels = _exact_case(M, C, K, 9)
    b[C - 3] = float("inf")
    logits = rne_bf16(x.double() @ w.double().t() + b.double())
    dy, loss, _ = ops.linear_bias_xent_forward_local(x, w, b, labels, 1.0, 1.0)
    torch.cuda.synchronize()
    z = logits.double().requires_grad_()
    ref_row = F.cross_entropy(z, labels, reduction="none")
    ref_row.sum().backward()
    assert torch.isnan(loss).all() == torch.isnan(ref_row.sum()).all()
    assert torch.equal(torch.isnan(dy), torch.isnan(z.grad))


def test_xent_random_inputs_at_scale():
    """randn inputs at M x C x K = 8192 x 32768 x 4096 against an fp32 reference on the bf16-rounded fp32 logits."""
    ops = _ops()
    M, C, K = 8192, 32768, 4096
    g = _gen(M, C, K)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (3 * torch.randn(C, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    b = torch.randn(C, device="cuda", generator=g)
    labels = torch.randint(0, C, (M,), generator=g, device="cuda")
    ls = gs = 1.0 / M
    dy, loss, part = ops.linear_bias_xent_forward_local(x, w, b, labels, ls, gs)
    torch.cuda.synchronize()
    z32 = torch.addmm(b, x.float(), w.float().t())
    zb = z32.to(torch.bfloat16).float()  # the kernel rounds its fp32 logits the same way; order noise can flip an ulp
    del z32
    p = torch.softmax(zb, dim=1)
    ref_row = torch.logsumexp(zb, 1) - zb.gather(1, labels[:, None])[:, 0]
    ref_loss = ls * float(ref_row.double().sum())
    assert abs(float(loss) - ref_loss) <= 1e-3 * abs(ref_loss), f"loss {float(loss)} vs {ref_loss}"
    # accumulation-order noise can flip the bf16 rounding of a logit by one ulp (<= 2^-7 of it): that moves
    # logit - lse by at most 2^-7 (|logit| + max |logit| of the row), and p by that factor
    p.scatter_add_(1, labels[:, None], -torch.ones(M, 1, device="cuda"))
    ref_dy = gs * p
    zmax = zb.abs().amax(1, keepdim=True)
    tol = gs * (p.abs() + 1e-6) * (2.0 ** -6 * (zb.abs() + zmax)) + 2.0 ** -8 * ref_dy.abs()
    del zb
    err = (dy.float() - ref_dy).abs()
    assert bool((err <= tol).all()), f"dy off by {float((err - tol).max()):.4g} over the bound"
    db_tol = tol.sum(0) + 1e-4 * ref_dy.abs().sum(0)  # the per-element bound summed over the rows, plus fp32 sums
    del err, tol
    db = ops.column_sum(part)
    db_err = (db - ref_dy.sum(0)).abs()
    assert bool((db_err <= db_tol).all()), f"db off by {float((db_err - db_tol).max()):.4g} over the bound"


# ------------------------------------------------------------------------------------------------------------------
# DPMLPClassifier at one rank
# ------------------------------------------------------------------------------------------------------------------
def _reference_steps(params, xs, ls_, lr, ignore_index=IGNORE):
    """fp32 torch composition: Linear -> GELU(tanh) -> Linear -> cross-entropy (sum / B), SGD."""
    w1, b1, w2, b2 = [p.detach().float().clone().requires_grad_() for p in params]
    losses = []
    for x, lab in zip(xs, ls_):
        y = F.linear(F.gelu(F.linear(x.float(), w1, b1), approximate="tanh"), w2, b2)
        loss = F.cross_entropy(y, lab, reduction="sum", ignore_index=ignore_index) / x.shape[0]
        loss.backward()
        with torch.no_grad():
            for p in (w1, b1, w2, b2):
                p -= lr * p.grad
                p.grad = None
        losses.append(float(loss))
    return losses, [p.detach() for p in (w1, b1, w2, b2)]


XENT_NAMES = ("gemm_bias_gelu", "gemm_bias_xent", "xent_finish", "gemm_nn_gelu_bwd_colsum")
MSE_NAMES = ("gemm_bias_mse_colsum", "gemm_mse_epilogue")


def _run_classifier(B, D, H, C, sgd_in_backward, kernels_expected, n_real=None):
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.models import DPMLPClassifier

    comm = m4t.COMM_WORLD
    lr = 1.0
    n = C if n_real is None else n_real
    model = DPMLPClassifier(D, H, C, comm, device="cuda", lr=lr, seed=13, sgd_in_backward=sgd_in_backward)
    if n < C:  # the padded-class recipe
        model.b2.data[n:] = float("-inf")
    init = [p.detach().clone() for p in model.parameters()]
    g = _gen(B, D, H, C)
    xs = [torch.randn(B, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(3)]
    labs = [torch.randint(0, n, (B,), generator=g, device="cuda") for _ in range(3)]
    labs[1][::5] = IGNORE
    losses = []
    for x, lab in zip(xs, labs):
        before = _launches()
        if sgd_in_backward and kernels_expected:
            loss = model.loss(x, lab)
            loss.backward()
            assert all(p.grad is None for p in model.parameters()), "optimizer-in-backward left a .grad"
            losses.append(float(loss))
        else:
            losses.append(float(model.train_step(x, lab)))
        after = _launches()
        for name in XENT_NAMES:
            ran = after.get(name, 0) - before.get(name, 0)
            assert ran == (1 if kernels_expected else 0), f"{name} ran {ran} times in one step"
        for name in MSE_NAMES:
            assert after.get(name, 0) == before.get(name, 0), f"{name} ran in a cross-entropy step"
    # the reference runs the unpadded model: the padded classes must not change anything
    ref_init = [init[0], init[1], init[2][:n], init[3][:n]]
    ref_losses, ref_params = _reference_steps(ref_init, xs, labs, lr)
    what = f"{(B, D, H, C)} n={n} sgd_in_backward={sgd_in_backward}"
    for got, ref in zip(losses, ref_losses):
        assert abs(got - ref) <= 1e-2 * abs(ref), f"{what}: loss {got} vs {ref}"
    # parameters: the bf16 weights round each step's update (<= half an ulp, 2^-8 of the weight, per step), and the
    # bf16 dy / h / dz of the kernels put a relative error of about 1 % on the updates themselves
    w1, b1, w2, b2 = [p.detach().float() for p in model.parameters()]
    for name, p, ref, p0 in zip(("w1", "b1", "w2", "b2"), (w1, b1, w2[:n], b2[:n]), ref_params, ref_init):
        moved = float((ref - p0.float()).abs().max())
        assert moved > 0, f"{what}: {name} did not move in the reference"
        err = (p - ref).abs()
        bound = 3e-2 * moved + 3 * 2.0 ** -8 * ref.abs() + 1e-7
        assert bool((err <= bound).all()), f"{what}: {name} off by {float((err - bound).max()):.4g} over the bound"
    if n < C:
        assert bool(torch.isneginf(b2[n:]).all()), f"{what}: a padded bias left -inf"
        assert torch.equal(w2[n:], init[2][n:].float()), f"{what}: padded weight rows moved"
    probe = model.logits(xs[0])
    assert probe.shape == (B, C) and bool(torch.isfinite(probe[:, :n]).all())


@pytest.mark.parametrize("sgd_in_backward", [True, False])
@pytest.mark.parametrize("dims", [(384, 256, 512, 256), (8192, 4096, 16384, 4096)])
def test_dp_mlp_classifier_single_rank(dims, sgd_in_backward):
    _run_classifier(*dims, sgd_in_backward=sgd_in_backward, kernels_expected=True)


@pytest.mark.parametrize("sgd_in_backward", [True, False])
def test_dp_mlp_classifier_padded_classes(sgd_in_backward):
    """200 classes padded to 256 with bias -inf stay on the kernels and train as the 200-class model."""
    _run_classifier(384, 256, 512, 256, sgd_in_backward=sgd_in_backward, kernels_expected=True, n_real=200)


def test_dp_mlp_classifier_off_the_kernel_path():
    """C = 200 without padding is not a multiple of 128: the torch composition runs and still matches."""
    from mpi4torch_b200.ops import dp_mlp_cross_entropy_supported

    _run_classifier(384, 256, 512, 200, sgd_in_backward=True, kernels_expected=False)
    x = torch.zeros(384, 256, device="cuda", dtype=torch.bfloat16)
    w1 = torch.zeros(512, 256, device="cuda", dtype=torch.bfloat16)
    w2 = torch.zeros(200, 512, device="cuda", dtype=torch.bfloat16)
    b1, b2 = torch.zeros(512, device="cuda"), torch.zeros(200, device="cuda")
    labels = torch.zeros(384, dtype=torch.int64, device="cuda")
    assert not dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels)
    w2, b2 = torch.zeros(256, 512, device="cuda", dtype=torch.bfloat16), torch.zeros(256, device="cuda")
    assert dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels)
    assert not dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels.int())
    assert not dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels[:-1])
    assert not dp_mlp_cross_entropy_supported(x, w1, b1, w2, b2, labels.cpu())


def test_xent_op_rejects_bad_labels():
    ops = _ops()
    x = torch.zeros(64, 64, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(128, 64, device="cuda", dtype=torch.bfloat16)
    b = torch.zeros(128, device="cuda")
    good = torch.zeros(64, dtype=torch.int64, device="cuda")
    before = _launches()
    for bad in (good.int(), good[:-1], good.cpu(), good.reshape(8, 8), torch.zeros(128, dtype=torch.int64, device="cuda")[::2]):
        with pytest.raises(RuntimeError, match="labels"):
            ops.linear_bias_xent_forward_local(x, w, b, bad, 1.0, 1.0)
    assert _launches() == before
