"""FP8 training of the data-parallel linear layer on the GPU (DESIGN §4.4).

* ``quantize_fp8``: both layouts bit for bit against the CPU recipe (``quantize_fp8_reference``, itself checked
  against numpy in test_fp8_cpu.py) at odd shapes, the transposed copy against the row-major one, a supplied amax,
  non-finite inputs.
* The accumulator probe: how many bits one k-block of fp8 wgmma keeps on this card, and that the kernel's split
  accumulation keeps a sum across k-blocks that one block cannot hold.
* The three GEMM epilogues bit for bit on exact inputs: small integers whose per-k-block partial sums stay below 2^11
  quanta (well inside what the probe measures), at tile, wave and k-block edges, both A formats, non-unit scales,
  g != 1.
* Random normal inputs at 8192 x 4096 x 4096 against float64 on the dequantized operands and against
  ``torch._scaled_mm`` on the same fp8 operands.
* ``dp_linear_mse(fp8=True)`` in each optimizer mode bit for bit against a float64 emulation, the model, graph capture
  and the launch table; rejected layouts.
"""
import math

import pytest
import torch

from test_gpu_exact_arithmetic import _gen, _ops, _sm_count, assert_exact_loss, assert_same_bits, exact_bf16, ints, \
    ternary, wave_tile_counts

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPLinearModel
from mpi4torch_b200.ops import InBackwardSGD, dp_linear_mse
from mpi4torch_b200.ops.fp8 import E4M3, E5M2, dequantize, quantize_fp8_reference

pytestmark = pytest.mark.gpu

TILE = 128
PROBE_MIN_BITS = 12  # the exact tests below need 11 bits per k-block (plus the sign)


def _launches():
    return dict(m4t._C.kernel_launch_table())


def _q(x, fmt, rowwise=True, transposed=False, amax=None):
    return _ops().quantize_fp8(x, fmt, rowwise, transposed, amax)


def _bits(q):
    return q.view(torch.uint8)


# ---- quantize -------------------------------------------------------------------------------------------------------
QSHAPES = [(1, 8), (1, 1), (37, 53), (64, 64), (130, 264), (257, 129), (512, 4096)]


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
@pytest.mark.parametrize("shape", QSHAPES, ids=lambda s: "x".join(map(str, s)))
def test_quantize_bitwise(fmt, shape):
    g = torch.Generator().manual_seed(shape[0] * 1000 + shape[1])
    x = (torch.randn(shape, generator=g) * 3.0).to(torch.bfloat16)
    q, qt, si = _q(x.cuda(), fmt, True, True)
    rq, rsi = quantize_fp8_reference(x, fmt)
    assert torch.equal(si.cpu(), rsi), (float(si), float(rsi))
    assert torch.equal(_bits(q).cpu(), _bits(rq)), "row-major copy"
    assert torch.equal(_bits(qt), _bits(q).t()), "transposed copy is not the transpose of the row-major one"
    # each layout alone gives the same bytes
    q1, none1, _ = _q(x.cuda(), fmt, True, False)
    none2, qt2, _ = _q(x.cuda(), fmt, False, True)
    assert none1 is None and none2 is None
    assert torch.equal(_bits(q1), _bits(q)) and torch.equal(_bits(qt2), _bits(qt))


def test_quantize_strided_input():
    """A row stride above the width (and an odd one) takes the scalar path: same bytes."""
    g = torch.Generator().manual_seed(9)
    base = (torch.randn(70, 101, generator=g) * 0.01).to(torch.bfloat16)
    for cols in (96, 53):
        x = base.cuda()[:, :cols]
        assert x.stride(0) == 101
        q, qt, si = _q(x, E4M3, True, True)
        rq, rsi = quantize_fp8_reference(x.cpu(), E4M3)
        assert torch.equal(si.cpu(), rsi) and torch.equal(_bits(q).cpu(), _bits(rq))
        assert torch.equal(_bits(qt), _bits(q).t())


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
def test_quantize_supplied_amax(fmt):
    x = (torch.randn(96, 160) * 5).to(torch.bfloat16)
    amax = torch.tensor([float(x.float().abs().max()) * 37.0])
    q, qt, si = _q(x.cuda(), fmt, True, True, amax.cuda())
    rq, rsi = quantize_fp8_reference(x, fmt, amax)
    assert torch.equal(si.cpu(), rsi) and torch.equal(_bits(q).cpu(), _bits(rq))
    assert torch.equal(_bits(qt), _bits(q).t())
    _, own = quantize_fp8_reference(x, fmt)
    assert float(si) != float(own), "the supplied amax was ignored"


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_quantize_non_finite(fmt, bad):
    x = torch.randn(128, 256, device="cuda").to(torch.bfloat16)
    x[77, 201] = bad
    _, _, si = _q(x, fmt, True, True)
    assert math.isnan(float(si))


def test_quantize_zero():
    q, qt, si = _q(torch.zeros(64, 128, device="cuda", dtype=torch.bfloat16), E4M3, True, True)
    assert float(si) == 1.0 and not bool(_bits(q).any()) and not bool(_bits(qt).any())


# ---- accumulator probe ----------------------------------------------------------------------------------------------
def _raw_gemm(a64, b64, a_fmt=E4M3):
    """gemm_fp8_tn with unit scales on float64 matrices whose values are exact in fp8."""
    one = torch.ones(1, device="cuda")
    dt = torch.float8_e5m2 if a_fmt == E5M2 else torch.float8_e4m3fn
    a, b = a64.to(dt), b64.to(torch.float8_e4m3fn)
    assert torch.equal(a.double(), a64) and torch.equal(b.double(), b64)
    return _ops().gemm_fp8_tn(a, b, one, one)


def fp8_block_bits():
    """Bits one k-block of fp8 wgmma keeps below the leading bit of its largest product: block 0 sums 2^16 and
    2^(16 - t), block 1 adds -2^16 in the kernel's fp32 accumulator, and the bf16 output reads what is left of the
    small term (2^(16 - t) when the block kept it).  The largest t kept is returned; the smallest fp8 product,
    2^-18, caps the probe at 34 bits."""
    for t in range(1, 40):
        K = 256
        a = torch.zeros(8, K, dtype=torch.float64, device="cuda")
        b = torch.zeros(TILE, K, dtype=torch.float64, device="cuda")
        a[:, 0] = 2.0 ** 8   # 2^16 in block 0
        b[:, 0] = 2.0 ** 8
        lo = 16 - t          # the small term 2^lo in the same block
        la = max(-9, lo - 8)
        if lo - la < -9:
            return t - 1
        a[:, 1] = 2.0 ** la
        b[:, 1] = 2.0 ** (lo - la)
        a[:, 128] = -(2.0 ** 8)  # block 1 takes the 2^16 away again, in the fp32 accumulator
        b[:, 128] = 2.0 ** 8
        c = _raw_gemm(a, b)
        if float(c[0, 0]) != 2.0 ** lo:
            return t - 1
    return 39


def test_block_precision_and_split_accumulation(capsys):
    bits = fp8_block_bits()
    with capsys.disabled():
        print(f"\n[fp8 probe] one k-block keeps {bits} bits below the leading bit of its largest product")
    assert bits >= PROBE_MIN_BITS, bits
    # split accumulation: 2^16 in block 0 and 2^(16 - bits - 2) in block 1 survive in the fp32 accumulator; the same
    # two terms in one block lose the small one.  The big term is taken away again by block 2.
    lo = 16 - bits - 2
    if lo < -18:
        pytest.skip(f"the block keeps {bits} bits: no fp8 product lies below them")
    la = max(-9, lo - 8)
    a = torch.zeros(8, 384, dtype=torch.float64, device="cuda")
    b = torch.zeros(TILE, 384, dtype=torch.float64, device="cuda")
    a[:, 0], b[:, 0] = 2.0 ** 8, 2.0 ** 8
    a[:, 256], b[:, 256] = -(2.0 ** 8), 2.0 ** 8
    split = a.clone()
    split[:, 128], b[:, 128] = 2.0 ** la, 2.0 ** (lo - la)
    one = a.clone()
    one[:, 1], b[:, 1] = 2.0 ** la, 2.0 ** (lo - la)
    assert float(_raw_gemm(split, b)[0, 0]) == 2.0 ** lo, "split accumulation lost the small block"
    assert float(_raw_gemm(one, b)[0, 0]) != 2.0 ** lo, "one k-block kept what the probe says it cannot"


# ---- GEMM epilogues on exact inputs -----------------------------------------------------------------------------------
def exact_operand(shape, gen, fmt, scale):
    """bf16 integers in [-4, 4] (E4M3) or [-3, 3] (E5M2) times a power of two: exact after quantization."""
    r = 4 if fmt == E4M3 else 3
    return exact_bf16(ints(shape, r, gen, scale))


def quantized(v, fmt):
    q, _, si = _q(v, fmt)
    d = dequantize(q, si, torch.float64)
    assert torch.equal(d, v.double()), "operand not exact in fp8"
    return q, si, d


def check_plain(M, N, K, gen, a_fmt=E4M3, g=None, scales=(2.0 ** -3, 2.0 ** -4)):
    a, sa, ad = quantized(exact_operand((M, K), gen, a_fmt, scales[0]), a_fmt)
    b, sb, bd = quantized(exact_operand((N, K), gen, E4M3, scales[1]), E4M3)
    gs = None if g is None else torch.full((1,), g, device="cuda")
    c = _ops().gemm_fp8_tn(a, b, sa, sb, gs)
    v = ad @ bd.t()
    ref = (v.float() * (1.0 if g is None else g)).to(torch.bfloat16) if g is not None else v.float().to(torch.bfloat16)
    assert_same_bits(c, ref, f"gemm_fp8_tn {(M, N, K)} {a_fmt} g={g}")


def check_mse(M, N, K, gen):
    x, sx, xd = quantized(exact_bf16(ternary((M, K), 0.25, gen, 2.0 ** -3)), E4M3)
    w, sw, wd = quantized(exact_bf16(ternary((N, K), 0.25, gen, 2.0 ** -5)), E4M3)
    y = xd @ wd.t()
    # d in [-3, 3] quanta, sparser on large outputs so that sum d^2 stays inside the exact range of the fp32 loss
    d = ints((M, N), 3, gen, 2.0 ** -8) if 9 * M * N < 2 ** 21 else ternary((M, N), 2.0 ** 21 / (M * N), gen, 2.0 ** -8)
    t = exact_bf16(y - d)
    ls, gsc = 2.0 ** -9, 2.0 ** -3
    assert_exact_loss(d)
    dy, loss, amax = _ops().linear_mse_forward_fp8_local(x, w, sx, sw, t, ls, gsc)
    ref = (d * gsc).float().to(torch.bfloat16)
    assert_same_bits(dy, ref, f"fp8 mse dy {(M, N, K)}")
    assert float(loss) == ls * float(d.square().sum())
    assert float(amax) == float(ref.float().abs().max())


def check_sgd(M, N, K, gen, a_fmt=E5M2, g=3.0, lr=2.0 ** -2):
    a, sa, ad = quantized(exact_operand((M, K), gen, a_fmt, 2.0 ** -6), a_fmt)
    b, sb, bd = quantized(exact_operand((N, K), gen, E4M3, 2.0 ** -2), E4M3)
    w0 = exact_bf16(ints((M, N), 200, gen, 2.0 ** -7))
    w = w0.clone()
    gs = torch.full((1,), g, device="cuda")
    _ops().gemm_fp8_tn_sgd_(w, a, b, sa, sb, -lr, gs)
    step = torch.tensor(g, dtype=torch.float32) * torch.tensor(-lr, dtype=torch.float32)
    ref = ((ad @ bd.t()).float() * step.cuda() + w0.float()).to(torch.bfloat16)
    assert_same_bits(w, ref, f"gemm_fp8_tn_sgd_ {(M, N, K)} {a_fmt}")


EDGE_SHAPES = [(1, 8, 16), (127, 120, 112), (128, 128, 128), (129, 136, 144), (257, 264, 400), (64, 1024, 272),
               (300, 8, 1040)]
CHECKS = {"plain": lambda M, N, K, gen: check_plain(M, N, K, gen),
          "plain_e5m2_g": lambda M, N, K, gen: check_plain(M, N, K, gen, E5M2, g=3.0),
          "plain_scaled": lambda M, N, K, gen: check_plain(M, N, K, gen, g=2.0 ** -3, scales=(2.0 ** 9, 2.0 ** -20)),
          "mse": check_mse,
          "sgd_e5m2": check_sgd,
          "sgd_e4m3": lambda M, N, K, gen: check_sgd(M, N, K, gen, E4M3, g=0.75)}


@pytest.mark.parametrize("op", list(CHECKS))
@pytest.mark.parametrize("shape", EDGE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_epilogue_tile_edges_bitwise(op, shape):
    CHECKS[op](*shape, _gen(*shape, len(op)))


@pytest.mark.parametrize("op", ["plain_e5m2_g", "mse", "sgd_e5m2"])
@pytest.mark.parametrize("wave", range(4), ids=["S-1", "S", "S+1", "2S+1"])
def test_epilogue_wave_edges_bitwise(op, wave):
    T = wave_tile_counts(_sm_count())[wave]
    n_t = max(d for d in range(1, 6) if T % d == 0)
    M, N, K = TILE * (T // n_t) - 24, TILE * n_t - 16, 3 * 128 - 16
    assert -(-M // TILE) * -(-N // TILE) == T
    CHECKS[op](M, N, K, _gen(M, N, K, wave))


@pytest.mark.parametrize("op", ["plain", "sgd_e5m2"])
def test_epilogue_many_kblocks_bitwise(op):
    CHECKS[op](256, 256, 128 * 40 + 48, _gen(40, len(op)))


def test_nan_scale_poisons_output():
    gen = _gen(1, 2, 3)
    x = exact_operand((128, 256), gen, E4M3, 1.0)
    x[5, 7] = float("inf")
    a, _, sa = _q(x, E4M3)
    b, _, sb = _q(exact_operand((128, 256), gen, E4M3, 1.0), E4M3)
    assert bool(_ops().gemm_fp8_tn(a, b, sa, sb).float().isnan().all())


# ---- realistic inputs ---------------------------------------------------------------------------------------------
def test_randn_against_float64_and_scaled_mm(capsys):
    M, N, K = 8192, 4096, 4096
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn(N, K, device="cuda", generator=g) * K ** -0.5).to(torch.bfloat16)
    xq, _, sx = _q(x, E4M3)
    wq, _, sw = _q(w, E4M3)
    c = _ops().gemm_fp8_tn(xq, wq, sx, sw)
    ref = dequantize(xq, sx, torch.float64) @ dequantize(wq, sw, torch.float64).t()
    mm = torch._scaled_mm(xq, wq.t(), scale_a=sx, scale_b=sw, out_dtype=torch.bfloat16)
    err = (c.double() - ref).abs()
    err_mm = (mm.double() - ref).abs()
    # bound: a bf16 ulp (2^-8 relative) plus 2^-9 of the sum of |products| (fp8 accumulation within a k-block)
    mag = dequantize(xq, sx, torch.float64).abs() @ dequantize(wq, sw, torch.float64).abs().t()
    assert bool((err <= 2.0 ** -8 * ref.abs() + 2.0 ** -9 * mag).all()), float((err - 2.0 ** -8 * ref.abs()).max())
    rel, rel_mm = float(err.norm() / ref.norm()), float(err_mm.norm() / ref.norm())
    with capsys.disabled():
        print(f"\n[fp8 randn] relative error: gemm_fp8_tn {rel:.3e}, torch._scaled_mm {rel_mm:.3e}, "
              f"max |diff| to _scaled_mm {float((c.double() - mm.double()).abs().max()):.3e}")
    assert rel <= max(1.5 * rel_mm, 3e-3)


# ---- the node and the model ----------------------------------------------------------------------------------------
def node_case(B, D, O, gen):
    """Ternary bf16 x and W (exact after E4M3 quantization, y small), t = y - d with d in [-3, 3] quanta: dy is exact
    in E5M2, and the fp8 wgrad sums stay far below the probe's range."""
    x = exact_bf16(ternary((B, D), 0.25, gen, 2.0 ** -3))
    w = exact_bf16(ternary((O, D), 0.25, gen, 2.0 ** -4))
    d = ints((B, O), 3, gen, 2.0 ** -7)
    t = exact_bf16(x.double() @ w.double().t() - d)
    return x, w, t, d


def emulate(x, w, t, d, ls, g):
    """(loss, dy, G = bf16(g dy^T x), x.grad = bf16(bf16(dy @ W) * g)) of the kernel path, float64 (all exact)."""
    dy = (d * 2.0 * ls).float().to(torch.bfloat16)
    dyq, dys = quantize_fp8_reference(dy.cpu(), E5M2)
    assert torch.equal(dequantize(dyq, dys, torch.float64).cuda(), dy.double()), "dy not exact in E5M2"
    G = ((dy.double().t() @ x.double()).float() * g).to(torch.bfloat16)
    gx = ((dy.double() @ w.double()).float().to(torch.bfloat16).float() * g).to(torch.bfloat16)
    return ls * float(d.square().sum()), G, gx


@pytest.mark.parametrize("mode", ["plain", "in_backward"])
@pytest.mark.parametrize("frozen", [False, True])
@pytest.mark.parametrize("g", [1.0, 3.0])
def test_node_bitwise(mode, frozen, g):
    B, D, O = 256, 384, 128
    gen = _gen(B, D, O, 5 + frozen)
    x, w, t, d = node_case(B, D, O, gen)
    ls, lr = 1.0 / B, 2.0 ** -3
    xr = x.clone().requires_grad_()
    wr = w.clone().requires_grad_(not frozen)
    opt = InBackwardSGD(lr) if mode == "in_backward" else None
    loss = dp_linear_mse(xr, wr, t, m4t.COMM_WORLD, loss_scale=ls, optimizer=opt, fp8=True)
    (loss * g).sum().backward()
    l_ref, G, gx = emulate(x, w, t, d, ls, g)
    assert float(loss) == l_ref
    assert_same_bits(xr.grad, gx, "x.grad")
    if frozen:
        assert wr.grad is None and torch.equal(wr.detach(), w)
    elif mode == "plain":
        assert_same_bits(wr.grad, G, "W.grad")
    else:
        assert wr.grad is None and opt.updates == 1
        step = torch.tensor(g, dtype=torch.float32) * torch.tensor(-lr, dtype=torch.float32)
        acc = (d * 2.0 * ls).t() @ x.double()
        ref = (acc.float() * step.cuda() + w.float()).to(torch.bfloat16)
        assert_same_bits(wr.detach(), ref, "W after the in-backward step")


def _regression(B, D, O, steps, fp8, lr):
    g = torch.Generator(device="cuda").manual_seed(3)
    teacher = torch.randn(O, D, device="cuda", generator=g) * D ** -0.5
    model = DPLinearModel(D, O, m4t.COMM_WORLD, device="cuda", dtype=torch.bfloat16, lr=lr, seed=1, fp8=fp8)
    losses = []
    for _ in range(steps):
        x = torch.randn(B, D, device="cuda", generator=g)
        losses.append(float(model.train_step(x.to(torch.bfloat16), (x @ teacher.t()).to(torch.bfloat16))))
    return losses


def test_model_learns_like_bf16(capsys):
    l8 = _regression(1024, 512, 512, 60, True, 0.5)
    l16 = _regression(1024, 512, 512, 60, False, 0.5)
    with capsys.disabled():
        print(f"\n[fp8 model] loss {l8[0]:.4f} -> {l8[-1]:.4f} (bf16: {l16[0]:.4f} -> {l16[-1]:.4f})")
    assert l8[-1] < 0.2 * l8[0]
    assert l8[-1] <= 1.5 * l16[-1] + 0.01 * l16[0]


def test_graph_capture_replays_like_eager():
    B, D, O = 512, 256, 384
    g = torch.Generator(device="cuda").manual_seed(4)
    xs = [torch.randn(B, D, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4)]
    ts = [torch.randn(B, O, device="cuda", generator=g).to(torch.bfloat16) for _ in range(4)]
    eager = DPLinearModel(D, O, m4t.COMM_WORLD, device="cuda", lr=0.05, seed=2, fp8=True)
    graphed = DPLinearModel(D, O, m4t.COMM_WORLD, device="cuda", lr=0.05, seed=2, fp8=True)
    replay, sx, st, gl = graphed.make_graphed_step(xs[0], ts[0], warmup=3)
    for _ in range(3):
        eager.train_step(xs[0], ts[0])  # the warm-up steps of the capture (capturing runs nothing)
    for x, t in zip(xs, ts):
        le = eager.train_step(x, t)
        sx.copy_(x)
        st.copy_(t)
        replay()
        torch.cuda.synchronize()
        assert abs(float(gl) - float(le)) <= 1e-5 * abs(float(le))
        assert torch.equal(graphed.weight.detach().view(torch.int16), eager.weight.detach().view(torch.int16))


def test_launch_table_per_step():
    B, D, O = 256, 256, 256
    model = DPLinearModel(D, O, m4t.COMM_WORLD, device="cuda", lr=0.01, seed=2, fp8=True)
    x = torch.randn(B, D, device="cuda").to(torch.bfloat16)
    t = torch.randn(B, O, device="cuda").to(torch.bfloat16)
    model.train_step(x, t)
    before = _launches()
    model.train_step(x, t)
    after = _launches()
    diff = {k: after.get(k, 0) - before.get(k, 0) for k in after if after.get(k, 0) != before.get(k, 0)}
    assert diff.get("quantize_fp8_amax") == 2 and diff.get("quantize_fp8_cast") == 3, diff
    assert diff.get("gemm_fp8_mse") == 1 and diff.get("gemm_fp8_sgd") == 1, diff
    assert "gemm_fp8_tn" not in diff and "gemm_mse_epilogue" not in diff and "wgrad_sgd_epilogue" not in diff, diff
    plain = DPLinearModel(D, O, m4t.COMM_WORLD, device="cuda", lr=0.01, seed=2, fp8=True, sgd_in_backward=False)
    before = _launches()
    plain.train_step(x, t)
    after = _launches()
    assert after.get("gemm_fp8_tn", 0) - before.get("gemm_fp8_tn", 0) == 1


# ---- rejected layouts -------------------------------------------------------------------------------------------------
def test_rejected_layouts_raise_before_launching():
    ops = _ops()
    a, _, sa = _q(torch.randn(256, 256, device="cuda").to(torch.bfloat16), E4M3)
    b, _, sb = _q(torch.randn(128, 256, device="cuda").to(torch.bfloat16), E4M3)
    a5, _, _ = _q(torch.randn(128, 256, device="cuda").to(torch.bfloat16), E5M2)
    cases = [
        (a[:, 8:], b[:, 8:], sa, sb),                  # base not 16-byte aligned, K = 248 % 16 != 0
        (a[:, :120], b[:, :120], sa, sb),              # K % 16 != 0
        (a, a5, sa, sb),                               # B must be E4M3
        (a, b.t().contiguous().t(), sa, sb),           # B not K-major
        (a, b, sa.cpu(), sb),                          # scale on the CPU
        (a, b, torch.ones(2, device="cuda"), sb),      # scale with two elements
        (a.view(torch.uint8), b, sa, sb),              # not an fp8 dtype
        (a, b[:124], sa, sb),                          # N % 8 != 0
    ]
    before = _launches()
    for args in cases:
        assert not ops.gemm_fp8_tn_supported(*args)
        with pytest.raises(RuntimeError):
            ops.gemm_fp8_tn(*args)
    t = torch.zeros(256, 128, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(RuntimeError):
        ops.linear_mse_forward_fp8_local(a, b, sa, sb, t[:, :127], 1.0, 1.0)  # target shape
    with pytest.raises(RuntimeError):
        ops.linear_mse_forward_fp8_local(a, b, sa, sb, torch.zeros(256, 129, device="cuda",
                                                                   dtype=torch.bfloat16)[:, 1:], 1.0, 1.0)  # odd base
    with pytest.raises(RuntimeError):
        ops.gemm_fp8_tn_sgd_(torch.zeros(256, 128, device="cuda"), a, b, sa, sb, -1.0)  # fp32 weight
    with pytest.raises(RuntimeError):
        ops.quantize_fp8(torch.zeros(4, 4, device="cuda"), E4M3, True, False)  # fp32 input
    with pytest.raises(RuntimeError):
        ops.quantize_fp8(torch.zeros(4, 4, device="cuda", dtype=torch.bfloat16), "e3m4", True, False)
    after = _launches()
    fp8_names = ("gemm_fp8_tn", "gemm_fp8_mse", "gemm_fp8_sgd", "quantize_fp8_amax", "quantize_fp8_cast")
    assert all(after.get(k, 0) == before.get(k, 0) for k in fp8_names)
