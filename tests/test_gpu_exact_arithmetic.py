"""The wgmma ops bit for bit, on inputs for which the fp32 accumulation is exact.

Every input is a small integer times a power of two, and every scale is a power of two.  When, in units of the
common quantum, each output's sum of |addends| stays below 2^22, every partial sum is an integer below 2^24: it is
exact in fp32 in whatever order the tensor cores, the warp shuffles or the float atomics add.  The float64
reference of such an input is then exact too, and rounding it once to fp32 and once to bf16 at the points where
the kernel rounds gives the kernel's output exactly.  So a truncating or ties-away bf16 store, a bias rounded
before it is added, a tile lost or added twice in the loss, or the wrong GELU show up as bit differences at any
shape, where the tolerance tests in test_gpu_gemm.py, test_gpu_mlp.py and test_gpu_operand_layouts.py cannot see
them.  The only non-exact values are GELU and its derivative, computed by the kernel in fp32 with ``tanhf``; they
are bounded by half a bf16 ulp plus a derived fp32 term (tests/test_exact_helpers.py checks on the CPU that these
bounds accept torch's fp32 tanh-GELU and reject erf-GELU and truncation).

The shapes sweep the tile edges (128 x 256 tiles, 64-deep k-blocks), the wave edges (S - 1, S, S + 1 and 2S + 1
tiles for S SMs) and the 4-stage smem ring: with 3 or 5 k-blocks per tile a CTA's second tile starts part-way
round the ring, with 5 also on the flipped barrier parity (tests/test_protocol_models.py models the ring).

Measured on one H100 80GB HBM3 (700 W power limit): every bitwise case holds with the 2^22 bound, so the tensor
cores add such sums exactly.  The file's 324 cases take about 5 s and peak at 0.9 GiB of device memory.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EXACT_UNITS = 2 ** 22    # bound on sum(|addend|) per output, and on sum(d^2) per loss, in units of the quantum
BM, BN, BK = 128, 256, 64  # GEMM tile of the single-GPU kernels
WGRAD_BM, WGRAD_BN = 128, 256
WAVE_KBLOCKS = (3, 5)    # k-blocks per tile of the wave sweep: second tiles start at ring stage 3 / stage 1, parity 1

GELU_BETA = math.sqrt(2.0 / math.pi)
GELU_KAPPA = 0.044715
U24 = 2.0 ** -24         # unit roundoff of fp32


# ------------------------------------------------------------------------------------------------------------------
# Shapes (plain Python: tests/test_protocol_models.py replays them through its model of the smem ring)
# ------------------------------------------------------------------------------------------------------------------
TILE_M = (1, 64, 65, 127, 128, 129, 257)
TILE_N = (8, 248, 256, 264, 520)
TILE_K = (8, 64, 72, 136, 200, 264, 328)  # 1, 1, 2, 3, 4, 5, 6 k-blocks


def tile_edge_shapes():
    """Every (M, N) pair once, K cycling through the k-block counts: each K meets five Ms and every N."""
    return [(M, N, TILE_K[(i * len(TILE_N) + j) % len(TILE_K)]) for i, M in enumerate(TILE_M) for j, N in enumerate(TILE_N)]


def wave_tile_counts(S):
    """One SM idle (S - 1), exactly one wave (S), a last wave of one tile (S + 1: one CTA runs two tiles; 2S + 1:
    one CTA runs three).  The grid is min(tiles, S), so no CTA is ever left without a tile."""
    return (S - 1, S, S + 1, 2 * S + 1)


def _divisor_at_most(T, d_max):
    return max(d for d in range(1, d_max + 1) if T % d == 0)


def gemm_wave_shape(T, kblocks):
    """(M, N, K) with exactly T tiles of 128 x 256, ragged in M, N and K, and `kblocks` k-blocks per tile."""
    n_t = _divisor_at_most(T, 5)
    return BM * (T // n_t) - 24, BN * n_t - 16, BK * kblocks - 8


def wgrad_wave_shape(T, kblocks):
    """(Mb, N, K) of wgrad with exactly T tiles of 128 x 256; odd T gets a half-width (K % 256 == 128) last tile."""
    k_t = _divisor_at_most(T, 8)
    return BK * kblocks, WGRAD_BM * (T // k_t), WGRAD_BN * k_t - (128 if T % 2 else 0)


WGRAD_EDGE_SHAPES = [(64, 128, 128), (64, 256, 896), (128, 384, 256), (192, 128, 640), (192, 512, 384),
                     (320, 256, 128), (320, 640, 1152), (384, 128, 512)]


# ------------------------------------------------------------------------------------------------------------------
# Exact inputs
# ------------------------------------------------------------------------------------------------------------------
def _gen(*vals, device="cuda"):
    return torch.Generator(device=device).manual_seed(sum((i + 1) * 7919 * int(v) for i, v in enumerate(vals)) % (2 ** 62))


def ints(shape, r, gen, scale=1.0):
    """float64 integers uniform in [-r, r], times `scale` (a power of two), on the generator's device."""
    return torch.randint(-r, r + 1, shape, generator=gen, device=gen.device, dtype=torch.int64).double() * scale


def ternary(shape, density, gen, scale=1.0):
    """float64 values in {-1, 0, 1} (nonzero with probability `density`), times `scale`, on the generator's device."""
    sign = torch.randint(0, 2, shape, generator=gen, device=gen.device, dtype=torch.int64).double() * 2 - 1
    keep = torch.rand(shape, generator=gen, device=gen.device, dtype=torch.float64) < density
    return sign * keep * scale


def exact_bf16(v):
    """v (float64) as bf16; v must be representable."""
    b = v.to(torch.bfloat16)
    assert torch.equal(b.double(), v), "input not representable in bf16"
    return b


def exact_f32(v):
    f = v.float()
    assert torch.equal(f.double(), v), "input not representable in fp32"
    return f


def rne_bf16(v):
    """The kernel's store: float64 value -> fp32 (round to nearest even) -> bf16 (round to nearest even)."""
    return v.float().to(torch.bfloat16)


def trunc_bf16(v):
    """float64 value (exact in fp32) -> bf16 rounded toward zero: a target one ulp-fraction off its value."""
    f = exact_f32(v)
    return (f.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def quantum(v):
    """Largest power of two q such that v / q is an integer for every finite element (1.0 for all zeros)."""
    v = v.double()
    v = v[torch.isfinite(v) & (v != 0)]
    if v.numel() == 0:
        return 1.0
    m, e = torch.frexp(v)
    n = (m.abs() * 2.0 ** 53).long()
    low = torch.log2((n & -n).double())
    return 2.0 ** int((e.double() - 53 + low).min())


def assert_exact_gemm(a, b, *addends, what=""):
    """Exactness precondition of a @ b (+ addends): per output, sum |addend| < 2^22 quanta."""
    q = min([quantum(a) * quantum(b)] + [quantum(t) for t in addends])
    s = a.double().abs() @ b.double().abs()
    for t in addends:
        s = s + t.double().abs()
    units = float(s.max()) / q
    assert units < EXACT_UNITS, f"{what}: sum |addend| reaches {units:.4g} quanta, above the exact bound 2^22"


def assert_exact_loss(d, what=""):
    """Exactness precondition of sum(d^2) in any order: below 2^22 squared quanta of d."""
    q = quantum(d)
    units = float((d / q).square().sum())
    assert units < EXACT_UNITS, f"{what}: sum d^2 reaches {units:.4g} squared quanta, above the exact bound 2^22"


def _first_mismatch(bad):
    idx = bad.nonzero()[0].tolist()
    return tuple(idx)


def assert_same_bits(got, ref, what=""):
    """Bitwise equality (bf16 or fp32), up to the sign of zero; NaN must sit exactly where the reference has NaN."""
    assert got.dtype == ref.dtype and got.shape == ref.shape, f"{what}: {got.dtype}{tuple(got.shape)} vs {ref.dtype}{tuple(ref.shape)}"
    ig = torch.int16 if got.dtype == torch.bfloat16 else torch.int32
    g0, r0 = got + 0.0, ref + 0.0  # -0 -> +0
    nan_g, nan_r = torch.isnan(got), torch.isnan(ref)
    bad = (nan_g != nan_r) | (~nan_r & (g0.view(ig) != r0.view(ig)))
    if bool(bad.any()):
        at = _first_mismatch(bad)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at {at}: "
                             f"got {float(got[at])!r}, expected {float(ref[at])!r}")


def assert_loss_exact(loss, ref, what=""):
    """The fp32 loss equals the exact value (which is representable: checked)."""
    want = torch.tensor([ref], dtype=torch.float64, device=loss.device)
    assert_same_bits(loss.reshape(1), exact_f32(want), what)


# ------------------------------------------------------------------------------------------------------------------
# GELU references and bounds (float64)
# ------------------------------------------------------------------------------------------------------------------
def gelu_tanh64(z):
    return 0.5 * z * (1.0 + torch.tanh(GELU_BETA * (z + GELU_KAPPA * z ** 3)))


def gelu_tanh_grad64(z):
    t = torch.tanh(GELU_BETA * (z + GELU_KAPPA * z ** 3))
    return 0.5 * (1.0 + t) + 0.5 * z * (1.0 - t * t) * GELU_BETA * (1.0 + 3.0 * GELU_KAPPA * z * z)


def bf16_ulp(m):
    """bf16 ulp at magnitude m (float64, m >= 0); subnormal fp32 magnitudes take the smallest normal's ulp."""
    e = torch.floor(torch.log2(m.clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def _rounded_bound(ref, fp32_err):
    """|bf16(v32) - ref| <= fp32_err + half a bf16 ulp of v32, and |v32| <= |ref| + fp32_err."""
    return 0.5 * bf16_ulp(ref.abs() + fp32_err) + fp32_err


# fp32 error of the kernel's gelu_tanh(v) = 0.5 v (1 + tanhf(beta * fmaf(kappa v, v^2, v))), |v| = |z|:
#   the tanh argument u carries <= 6 u24 relative error (three roundings of the polynomial, the product with beta,
#   the fp32 constants beta and kappa), which moves tanh by <= |u| sech^2(u) * 6 u24 <= 0.45 * 6 u24 = 2.7 u24;
#   tanhf itself is off by <= 2 ulp <= 2 u24, so |dt| <= 4.7 u24 in absolute terms.  1 + t rounds once (<= u24:
#   it is below 2), and 0.5 v (1 + t) once more (<= u24 |v|, since |1 + t| <= 2).  For negative z, 1 + t cancels:
#   the absolute error of t is not reduced with it, so the bound must be relative to |z|, not to |h|:
#   |dh| <= 0.5 |z| (4.7 + 1) u24 + |z| u24 = 3.85 u24 |z|  ->  4 u24 |z|.
GELU_FP32_C = 4.0


def gelu_h_violations(h, z):
    """Elements of the bf16 `h` farther from gelu_tanh(z) (z: float64, the kernel's exact fp32 z) than the bound."""
    ref = gelu_tanh64(z)
    bound = _rounded_bound(ref, GELU_FP32_C * U24 * z.abs())
    return ~((h.double() - ref).abs() <= bound)


def gelu_grad_fp32_units(z):
    """Bound on the fp32 error of gelu_tanh_grad(z) in units of u24 (the kernel's formula, torch's GeluBackward):
      A = 0.5 (1 + t):  0.5 (|dt| + u24)                                    <= 3 u24
      B = 0.5 z (1 - t t) beta (1 + 3 kappa z^2), P = 0.5 |z| beta (1 + 3 kappa z^2):
          1 - t t moves by <= 2 |dt| + u24 (t t and the difference round once each, both below 1) <= 11 u24,
          times P; five more roundings and the constants beta, 3 kappa: <= 7 u24 |B| <= 7 u24 P      -> 18 P u24
      A + B and the product (gs acc) * g' round once each                     <= 2 u24 |g'|
    with |dt| <= 5 u24 (see GELU_FP32_C)."""
    P = 0.5 * z.abs() * GELU_BETA * (1.0 + 3.0 * GELU_KAPPA * z * z)
    return 3.0 + 18.0 * P + 2.0 * gelu_tanh_grad64(z).abs()


def gelu_dz_violations(dz, a, z):
    """Elements of the bf16 dz = bf16(a * gelu_tanh'(z)) out of bound; `a` = gs * acc (exact), z the bf16 input."""
    ref = a * gelu_tanh_grad64(z)
    return ~((dz.double() - ref).abs() <= _rounded_bound(ref, U24 * a.abs() * gelu_grad_fp32_units(z)))


def _gamma(n):
    return n * U24 / (1.0 - n * U24)


def colsum_rows(M):
    return (M + 15) // 16


def colsum_partials64(v):
    """Column sums of each group of 16 rows (the warp's rows in the epilogue), float64."""
    M, N = v.shape
    R = colsum_rows(M)
    pad = torch.zeros(R * 16, N, dtype=v.dtype, device=v.device)
    pad[:M] = v
    return pad.view(R, 16, N).sum(1)


# ------------------------------------------------------------------------------------------------------------------
# per-op checks
# ------------------------------------------------------------------------------------------------------------------
def _ops():
    import mpi4torch_b200 as m4t

    m4t.COMM_WORLD  # bring the backend up
    return torch.ops.mpi4torch_b200


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dense_operands(M, N, K, gen, r):
    """x [M, K] in [-r, r] * 2^-3 and w [N, K] in [-r, r] * 2^-4: products on a 2^-7 grid."""
    return ints((M, K), r, gen, 2.0 ** -3), ints((N, K), r, gen, 2.0 ** -4)


def sparse_operands(M, N, K, gen):
    """Ternary x and w of density 1/4: |acc| stays far below 256 quanta, so acc is exact in bf16."""
    return ternary((M, K), 0.25, gen, 2.0 ** -3), ternary((N, K), 0.25, gen, 2.0 ** -4)


def mse_target(v, gen, density):
    """A bf16 target near the exact fp32 value v: v + e with sparse e in {-1, 0, 1} quanta, rounded toward zero.
    d = v - t is then a few quanta: sum d^2 stays small, and d differs from bf16(v) - t wherever v is not a bf16."""
    return trunc_bf16(v + ternary(v.shape, density, gen, quantum(v)))


def check_gemm_tn(M, N, K, gen, sparse=False):
    ops = _ops()
    x, w = sparse_operands(M, N, K, gen) if sparse else dense_operands(M, N, K, gen, 16)
    assert_exact_gemm(x, w.t(), what="gemm_bf16_tn")
    y = ops.gemm_bf16_tn(exact_bf16(x), exact_bf16(w))
    assert_same_bits(y, rne_bf16(x @ w.t()), f"gemm_bf16_tn {(M, N, K)}")


def check_gemm_nn(M, N, K, gen, sparse=False):
    ops = _ops()
    a, bt = sparse_operands(M, N, K, gen) if sparse else dense_operands(M, N, K, gen, 16)
    b = bt.t().contiguous()  # [K, N]
    assert_exact_gemm(a, b, what="gemm_bf16_nn")
    c = ops.gemm_bf16_nn(exact_bf16(a), exact_bf16(b))
    assert_same_bits(c, rne_bf16(a @ b), f"gemm_bf16_nn {(M, N, K)}")


def check_linear_mse(M, N, K, gen, sparse=False, local=True):
    """dy = bf16(gs * (acc - t)) bitwise and loss = ls * sum((acc - t)^2) exactly."""
    ops = _ops()
    x, w = sparse_operands(M, N, K, gen) if sparse else dense_operands(M, N, K, gen, 4)
    acc = x @ w.t()
    assert_exact_gemm(x, w.t(), what="linear_mse")
    t = mse_target(acc, gen, 1 / 64 if sparse else 1 / 8)
    d = acc - t.double()
    assert_exact_loss(d, "linear_mse")
    ls, gs = 2.0 ** -3, 2.0 ** -2
    xb, wb = exact_bf16(x), exact_bf16(w)
    if local:
        dy, loss = ops.linear_mse_forward_local(xb, wb, t, ls, gs)
    else:
        dy, loss, _ = ops.linear_mse_forward(xb, wb, t, 1.0, ls, gs, True)
    shape = (M, N, K)
    assert_same_bits(dy, rne_bf16(gs * d), f"linear_mse dy {shape}")
    assert_loss_exact(loss, ls * float(d.square().sum()), f"linear_mse loss {shape}")


def bias_operands(M, N, K, gen, sparse):
    """x, w and an fp32 bias on the products' 2^-7 grid.  Dense: |b| up to 8 (z covers [-8, 8] densely, and most
    bias values need more than bf16's 8 bits); sparse: |b| <= 64 quanta, so acc + b stays exact in bf16."""
    x, w = sparse_operands(M, N, K, gen) if sparse else dense_operands(M, N, K, gen, 4)
    b = ints((N,), 64 if sparse else 1024, gen, 2.0 ** -7)
    return x, w, b


def check_bias_gelu(M, N, K, gen, sparse=False):
    """z = bf16(acc + b) bitwise; h within half a bf16 ulp (+ the fp32 term) of float64 gelu_tanh(acc + b)."""
    ops = _ops()
    x, w, b = bias_operands(M, N, K, gen, sparse)
    assert_exact_gemm(x, w.t(), b, what="bias_gelu")
    z = x @ w.t() + b
    h, zk = ops.linear_bias_gelu_forward(exact_bf16(x), exact_bf16(w), exact_f32(b))
    shape = (M, N, K)
    assert_same_bits(zk, rne_bf16(z), f"bias_gelu z {shape}")
    bad = gelu_h_violations(h, z)
    if bool(bad.any()):
        at = _first_mismatch(bad)
        raise AssertionError(f"bias_gelu h {shape}: {int(bad.sum())} elements out of bound; first at {at}: z {float(z[at])!r}, "
                             f"h {float(h[at])!r}, gelu_tanh {float(gelu_tanh64(z[at]))!r}")


def check_bias_mse(M, N, K, gen, sparse=False):
    """dy, loss, the column-sum partials and column_sum (with and without grad_scale) all exact."""
    ops = _ops()
    x, w, b = bias_operands(M, N, K, gen, sparse)
    assert_exact_gemm(x, w.t(), b, what="bias_mse")
    v = x @ w.t() + b
    t = mse_target(v, gen, 1 / 64 if sparse else 1 / 8)
    d = v - t.double()
    assert_exact_loss(d, "bias_mse")
    ls, gs = 2.0 ** -4, 2.0 ** -1
    dy, loss, part = ops.linear_bias_mse_forward_local(exact_bf16(x), exact_bf16(w), exact_f32(b), t, ls, gs)
    shape = (M, N, K)
    assert_same_bits(dy, rne_bf16(gs * d), f"bias_mse dy {shape}")
    assert_loss_exact(loss, ls * float(d.square().sum()), f"bias_mse loss {shape}")
    # the epilogue sums the fp32 values gs * d (not the bf16 dy): integers in quanta, so every sum is exact
    p64 = colsum_partials64(gs * d)
    assert_exact_gemm(torch.ones(1, M, device="cuda", dtype=torch.float64), gs * d, what="bias_mse column sums")
    assert_same_bits(part, exact_f32(p64), f"bias_mse column-sum partials {shape}")
    assert_same_bits(ops.column_sum(part), exact_f32(p64.sum(0)), f"column_sum {shape}")
    g2 = torch.full((1,), 2.0 ** -3, device="cuda")
    assert_same_bits(ops.column_sum(part, g2), exact_f32(2.0 ** -3 * p64.sum(0)), f"column_sum x grad_scale {shape}")


def check_gelu_backward(M, N, K, gen, sparse=False, scales=(None, 2.0 ** -1)):
    """dz = bf16(gs * acc * gelu_tanh'(z)): gs * acc exact, dz within half a bf16 ulp plus the fp32 term of the float64
    value; column sums within the fp32 summation bound of the kernel's order."""
    ops = _ops()
    dy, wt = sparse_operands(M, N, K, gen) if sparse else dense_operands(M, N, K, gen, 16)
    w = wt.t().contiguous()  # [K, N]
    assert_exact_gemm(dy, w, what="gelu_backward")
    acc = dy @ w
    z = rne_bf16(ints((M, N), 1024, gen, 2.0 ** -7))  # bf16 z densely covering [-8, 8]
    z64 = z.double()
    shape = (M, N, K)
    for scale in scales:
        gs = None if scale is None else torch.full((1,), scale, device="cuda")
        dz, part = ops.gemm_nn_gelu_backward(exact_bf16(dy), exact_bf16(w), z, gs)
        a = (scale or 1.0) * acc
        bad = gelu_dz_violations(dz, a, z64)
        if bool(bad.any()):
            at = _first_mismatch(bad)
            raise AssertionError(f"gelu backward dz {shape} x{scale}: {int(bad.sum())} out of bound; first at {at}: "
                                 f"z {float(z64[at])!r}, gs*acc {float(a[at])!r}, dz {float(dz[at])!r}, "
                                 f"exact {float(a[at] * gelu_tanh_grad64(z64[at]))!r}")
        ref = a * gelu_tanh_grad64(z64)
        err = U24 * a.abs() * gelu_grad_fp32_units(z64)  # per element: kernel fp32 value vs ref
        mag = ref.abs() + err
        # partials: 16 rows; a thread adds its two rows, then three shuffle levels: <= 4 roundings on any path
        p_bound = colsum_partials64(err) + _gamma(4) * colsum_partials64(mag)
        p_err = (part.double() - colsum_partials64(ref)).abs()
        assert bool((p_err <= p_bound).all()), f"gelu backward partials {shape} x{scale}: worst {float((p_err - p_bound).max()):.4g}"
        # column_sum: each of 8 row groups adds every 8th partial in order, then the 8 results in order
        R = colsum_rows(M)
        D = 4 + math.ceil(R / 8) + 7
        c_bound = err.sum(0) + _gamma(D) * mag.sum(0)
        c_err = (ops.column_sum(part).double() - ref.sum(0)).abs()
        assert bool((c_err <= c_bound).all()), f"gelu backward column_sum {shape} x{scale}: worst {float((c_err - c_bound).max()):.4g}"


def check_wgrad(Mb, N, K, gen):
    """G = bf16(gs * dy^T x) with and without the device grad_scale, and the SGD epilogue w <- bf16(fp32(s gs acc + w))."""
    ops = _ops()
    dy, x = ints((Mb, N), 16, gen, 2.0 ** -3), ints((Mb, K), 16, gen, 2.0 ** -4)
    assert_exact_gemm(dy.t(), x, what="wgrad")
    acc = dy.t() @ x
    dyb, xb = exact_bf16(dy), exact_bf16(x)
    shape = (Mb, N, K)
    assert_same_bits(ops.wgrad_bf16(dyb, xb), rne_bf16(acc), f"wgrad {shape}")
    gs = torch.full((1,), 2.0 ** 3, device="cuda")
    assert_same_bits(ops.wgrad_bf16(dyb, xb, gs), rne_bf16(8.0 * acc), f"wgrad x grad_scale {shape}")
    # SGD epilogue: w on a grid a few bits coarser than the update, so some sums round, ties included
    w0 = ints((N, K), 255, gen, quantum(acc) * 2.0 ** -2)
    w = exact_bf16(w0)
    scale = -(2.0 ** -5)
    ops.wgrad_sgd_(w, dyb, xb, scale, gs)
    assert_same_bits(w, rne_bf16(scale * 8.0 * acc + w0), f"wgrad_sgd_ {shape}")


# ------------------------------------------------------------------------------------------------------------------
# B + C: every op over the tile-edge and wave-edge shapes
# ------------------------------------------------------------------------------------------------------------------
GEMM_CHECKS = {
    "gemm_bf16_tn": check_gemm_tn,
    "gemm_bf16_nn": check_gemm_nn,
    "linear_mse_forward_local": lambda M, N, K, g, sparse=False: check_linear_mse(M, N, K, g, sparse, local=True),
    "linear_mse_forward": lambda M, N, K, g, sparse=False: check_linear_mse(M, N, K, g, sparse, local=False),
    "linear_bias_gelu_forward": check_bias_gelu,
    "linear_bias_mse_forward_local": check_bias_mse,
    "gemm_nn_gelu_backward": check_gelu_backward,
}

# the kernel instantiation behind each op (linear_mse_forward at one rank runs gemm_mse_epilogue as well)
WAVE_OPS = ["gemm_bf16_tn", "linear_mse_forward_local", "gemm_bf16_nn", "linear_bias_gelu_forward",
            "linear_bias_mse_forward_local", "gemm_nn_gelu_backward"]


@pytest.mark.parametrize("shape", tile_edge_shapes(), ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("op", list(GEMM_CHECKS))
def test_tile_edges_bitwise(op, shape):
    GEMM_CHECKS[op](*shape, _gen(*shape, len(op)))


@pytest.mark.parametrize("kblocks", WAVE_KBLOCKS)
@pytest.mark.parametrize("wave", range(4), ids=["S-1", "S", "S+1", "2S+1"])
@pytest.mark.parametrize("op", WAVE_OPS)
def test_wave_edges_bitwise(op, wave, kblocks):
    T = wave_tile_counts(_sm_count())[wave]
    M, N, K = gemm_wave_shape(T, kblocks)
    assert -(-M // BM) * -(-N // BN) == T
    # above 2^18 outputs the loss ops use the sparse inputs, whose sum of d^2 stays below 2^22 quanta
    sparse = op in ("linear_mse_forward_local", "linear_bias_mse_forward_local") and M * N > 2 ** 18
    kwargs = {"scales": (2.0 ** -1,)} if op == "gemm_nn_gelu_backward" else {}
    GEMM_CHECKS[op](M, N, K, _gen(M, N, K, len(op)), sparse=sparse, **kwargs)


@pytest.mark.parametrize("shape", WGRAD_EDGE_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_wgrad_tile_edges_bitwise(shape):
    check_wgrad(*shape, _gen(*shape, 3))


@pytest.mark.parametrize("kblocks", (1, 3, 5))
@pytest.mark.parametrize("wave", range(4), ids=["S-1", "S", "S+1", "2S+1"])
def test_wgrad_wave_edges_bitwise(wave, kblocks):
    T = wave_tile_counts(_sm_count())[wave]
    Mb, N, K = wgrad_wave_shape(T, kblocks)
    assert (N // WGRAD_BM) * -(-K // WGRAD_BN) == T
    check_wgrad(Mb, N, K, _gen(Mb, N, K, 5))


def test_wgrad_sgd_below_half_an_ulp():
    """The realistic SGD regime: |scale * g| below half a bf16 ulp of w.  w must stay unchanged, except where the
    step is exactly half an ulp: there it rounds to the even neighbour."""
    ops = _ops()
    Mb, N, K = 320, 384, 640
    gen = _gen(Mb, N, K, 11)
    # about one nonzero product per output: acc mostly in {-2 .. 2}
    dy, x = ternary((Mb, N), 0.06, gen), ternary((Mb, K), 0.06, gen)
    acc = dy.t() @ x
    assert_exact_gemm(dy.t(), x, what="wgrad_sgd_ small step")
    step = 2.0 ** -12  # |scale * gs|: acc = +-1 moves w by a quarter ulp, acc = +-2 by exactly half an ulp
    ulp = 4 * step
    mant = ints((N, K), 62, gen).abs() + 129  # 129 .. 191: even and odd bf16 significands, off the binade edge
    w0 = mant * ulp * torch.where(ints((N, K), 1, gen) < 0, -1.0, 1.0)
    w = exact_bf16(w0)
    gs = torch.full((1,), 2.0 ** -2, device="cuda")
    ops.wgrad_sgd_(w, exact_bf16(dy), exact_bf16(x), -(2.0 ** -10), gs)
    ref = rne_bf16(w0 - step * acc)
    assert_same_bits(w, ref, "wgrad_sgd_ below half an ulp")
    small, tie = acc.abs() == 1, acc.abs() == 2
    assert int(small.sum()) > 1000 and int(tie.sum()) > 100, "the inputs do not exercise the sub-ulp regime"
    assert torch.equal(w[small], exact_bf16(w0)[small]), "a step below half an ulp changed w"
    odd = (mant % 2 == 1)
    assert torch.equal(w[tie & ~odd], exact_bf16(w0)[tie & ~odd]), "a tie moved an even significand"
    assert bool((w[tie & odd].double() != w0[tie & odd]).all()), "a tie left an odd significand in place"


# ------------------------------------------------------------------------------------------------------------------
# B: NaN and Inf stay where they belong
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(257, 520, 200), (65, 264, 328)], ids=lambda s: "x".join(map(str, s)))
def test_nan_in_x_poisons_exactly_its_row(shape):
    ops = _ops()
    M, N, K = shape
    gen = _gen(M, N, K, 21)
    x, w = dense_operands(M, N, K, gen, 4)
    assert_exact_gemm(x, w.t(), what="NaN in x")
    i0, k0 = M - 2, K - 3
    xb = exact_bf16(x)
    xb[i0, k0] = float("nan")
    ref = rne_bf16(x @ w.t())
    ref[i0] = float("nan")
    assert_same_bits(ops.gemm_bf16_tn(xb, exact_bf16(w)), ref, "gemm_bf16_tn with a NaN in x")
    t = mse_target(x @ w.t(), gen, 1 / 8)
    assert_exact_loss(x @ w.t() - t.double(), "NaN in x")
    dy, loss, _ = ops.linear_mse_forward(xb, exact_bf16(w), t, 1.0, 1.0, 1.0, True)
    d_ref = rne_bf16(x @ w.t() - t.double())
    d_ref[i0] = float("nan")
    assert_same_bits(dy, d_ref, "linear_mse_forward dy with a NaN in x")
    assert bool(torch.isnan(loss).all()), "a NaN in x must make the loss NaN"


@pytest.mark.parametrize("shape", [(257, 520, 200), (129, 248, 72)], ids=lambda s: "x".join(map(str, s)))
def test_inf_in_w_reaches_only_its_column(shape):
    ops = _ops()
    M, N, K = shape
    gen = _gen(M, N, K, 22)
    x, w = dense_operands(M, N, K, gen, 4)
    assert_exact_gemm(x, w.t(), what="Inf in w")
    j0, k0 = N - 5, 1
    wb = exact_bf16(w)
    wb[j0, k0] = float("inf")
    ref = rne_bf16(x @ w.t())
    # column j0: x[i, k0] * inf is +-inf, or NaN where x[i, k0] == 0
    xs = x[:, k0]
    col = torch.where(xs > 0, float("inf"), torch.where(xs < 0, -float("inf"), float("nan")))
    ref[:, j0] = col.to(torch.bfloat16)
    assert bool((xs == 0).any()) and bool((xs != 0).any())
    assert_same_bits(ops.gemm_bf16_tn(exact_bf16(x), wb), ref, "gemm_bf16_tn with an Inf in w")


@pytest.mark.parametrize("local", [False, True])
def test_nan_target_poisons_the_loss_and_one_dy(local):
    ops = _ops()
    M, N, K = 257, 520, 200
    gen = _gen(M, N, K, 23)
    x, w = dense_operands(M, N, K, gen, 4)
    assert_exact_gemm(x, w.t(), what="NaN target")
    acc = x @ w.t()
    t = mse_target(acc, gen, 1 / 8)
    assert_exact_loss(acc - t.double(), "NaN target")
    i0, j0 = 130, 263
    tn = t.clone()
    tn[i0, j0] = float("nan")
    xb, wb = exact_bf16(x), exact_bf16(w)
    if local:
        dy, loss = ops.linear_mse_forward_local(xb, wb, tn, 2.0 ** -3, 2.0 ** -2)
    else:
        dy, loss, _ = ops.linear_mse_forward(xb, wb, tn, 1.0, 2.0 ** -3, 2.0 ** -2, True)
    ref = rne_bf16(2.0 ** -2 * (acc - t.double()))
    ref[i0, j0] = float("nan")
    assert_same_bits(dy, ref, "linear_mse dy with a NaN target")
    assert bool(torch.isnan(loss).all()), "a NaN target must make the loss NaN"


# ------------------------------------------------------------------------------------------------------------------
# D: the flagship step at one rank, bit for bit against a float64 emulation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sgd_in_backward", [True, False])
@pytest.mark.parametrize("dims", [(256, 512, 512), (2048, 768, 4096)], ids=lambda d: "x".join(map(str, d)))
def test_dp_linear_model_steps_bitwise(dims, sgd_in_backward):
    """Three DPLinearModel steps at one rank.  Forward: dy = bf16((2/B) (acc - t)), loss = (1/B) sum (acc - t)^2.
    Backward with the in-backward optimizer: w <- bf16(fp32(w - lr * g * dy^T x)) with g = 1; plain mode:
    grad = bf16(dy^T x) (wgrad_bf16), then torch's bf16 add_: w <- bf16(fp32(w - lr * grad)).
    x is ternary (quantum 1) and w sits on a 2^-4 grid; lr = B / 2 makes one step move w by whole grid units,
    so the inputs of every step stay exact."""
    import mpi4torch_b200 as m4t
    from mpi4torch_b200.models import DPLinearModel

    B, D, O = dims
    comm = m4t.COMM_WORLD
    assert comm.size == 1
    gen = _gen(B, D, O, int(sgd_in_backward))
    lr = B / 2.0
    model = DPLinearModel(D, O, comm, device="cuda", lr=lr, seed=3, sgd_in_backward=sgd_in_backward)
    w = ternary((O, D), 0.25, gen, 2.0 ** -4)
    with torch.no_grad():
        model.weight.copy_(exact_bf16(w))
    what = f"{dims} sgd_in_backward={sgd_in_backward}"
    for step in range(3):
        x = ternary((B, D), 0.25, gen)
        acc = x @ w.t()
        assert_exact_gemm(x, w.t(), what=f"{what} step {step} forward")
        t = mse_target(acc, gen, 1 / 64)
        d = acc - t.double()
        assert_exact_loss(d, f"{what} step {step}")
        dy = rne_bf16((2.0 / B) * d).double()
        assert_exact_gemm(dy.t(), x, what=f"{what} step {step} wgrad")
        G = dy.t() @ x
        if sgd_in_backward:
            w = rne_bf16(w - lr * G).double()
        else:
            w = rne_bf16(w - lr * rne_bf16(G).double()).double()
        loss = model.train_step(exact_bf16(x), t)
        assert_loss_exact(loss.reshape(1), float(d.square().sum()) / B, f"{what} step {step} loss")
        assert_same_bits(model.weight.detach(), exact_bf16(w), f"{what} step {step} weight")
    assert model.weight.grad is None
