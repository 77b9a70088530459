"""The fp8 GEMMs and the batched / grouped expert GEMMs on operands that are not fresh contiguous tensors, and at
their size limits.

* fp8 (``gemm_fp8_tn`` with and without ``grad_scale``, ``linear_mse_forward_fp8_local``, ``gemm_fp8_tn_sgd_``) on
  interior views of buffers filled with the byte 0x7F, which is NaN in E4M3 and in E5M2: the exact-input recipes of
  test_gpu_fp8.py give the float64 reference bit for bit, the same bits as contiguous copies, and no byte outside
  the views changes.  A tensor map or an epilogue that uses the width instead of the row stride reads NaN or
  writes into the padding.
* ``gemm_fp8_tn_supported`` against its ops over a table of layouts of each fp8 operand, the MSE target and the SGD
  weight: accepted layouts give the bits of contiguous copies, rejected ones raise on the host and launch nothing.
* The batched and grouped expert ops on contiguous views at aligned non-zero storage offsets give the bits of fresh
  tensors; misaligned bases (bf16, fp32 bias, int32 counts) are rejected by the predicates and the ops.
* ``expert_mlp`` and ``grouped_expert_mlp`` take an upstream gradient that is contiguous but misaligned.
* Limits: 1024 groups (the size of the kernels' shared-memory group table) against the single-expert ops, 1025
  groups and empty counts rejected, 1024 batched experts, and outputs of more than 2^31 elements.
"""
import pytest
import torch

from test_gpu_exact_arithmetic import _gen, assert_exact_loss, assert_same_bits, exact_bf16, ints, ternary
from test_gpu_fp8 import exact_operand, quantized
from test_gpu_gemm import _assert_close_bf16
from test_gpu_grouped_moe import _assert_zero_padding, _counts, _grouped, _rows, _starts
from test_gpu_moe import _launches, _m4t, _ops, _randn
from test_gpu_operand_layouts import _chunks, _layout, _Padded, _require_free, mem  # noqa: F401 (mem: fixture)

from mpi4torch_b200.ops.fp8 import E4M3, E5M2

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
NAN = float("nan")
FP8_NAN = 0x7F  # NaN in float8_e4m3fn and in float8_e5m2
FP8_SHAPES = [(300, 136, 272), (4100, 4104, 400)]  # (M, N, K): ragged, then more 128 x 128 tiles than SMs
LD_PADS = [16, 64]  # leading dimension = K + pad


def _launch_count():
    return _m4t()._C.kernel_launch_count()


def _assert_raises_without_launch(call, what):
    before = _launch_count()
    with pytest.raises(RuntimeError):
        call()
    torch.cuda.synchronize()
    assert _launch_count() == before, f"{what}: a kernel was launched"


class _Fp8Padded:
    """An fp8 matrix [rows, K] inside a buffer of 0x7F bytes: two rows above and below, 16 columns on the left and a
    leading dimension of K + ld_pad.  The view's base stays 16-byte aligned."""

    def __init__(self, q, ld_pad):
        rows, K = q.shape
        self.buf = torch.full((rows + 4, K + ld_pad), FP8_NAN, dtype=torch.uint8, device="cuda")
        region = (slice(2, 2 + rows), slice(16, 16 + K))
        self.buf[region].copy_(q.view(torch.uint8))
        self.view = self.buf.view(q.dtype)[region]
        self._before = self.buf.clone()

    def assert_intact(self, what):
        assert torch.equal(self.buf, self._before), f"{what}: fp8 operand buffer modified"


# ---- 1. the fp8 ops on interior views, bit for bit ----------------------------------------------------------------
@pytest.mark.parametrize("a_fmt,g", [(E4M3, None), (E5M2, 3.0)], ids=["e4m3", "e5m2_g3"])
@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", FP8_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_fp8_tn_on_views(shape, ld_pad, a_fmt, g):
    """check_plain's inputs (test_gpu_fp8.py) read through row strides above K."""
    ops = _ops()
    M, N, K = shape
    what = f"gemm_fp8_tn {shape} {a_fmt} g={g} ld=K+{ld_pad}"
    gen = _gen(M, N, K, ld_pad, g is None)
    a, sa, ad = quantized(exact_operand((M, K), gen, a_fmt, 2.0 ** -3), a_fmt)
    b, sb, bd = quantized(exact_operand((N, K), gen, E4M3, 2.0 ** -4), E4M3)
    gs = None if g is None else torch.full((1,), g, device="cuda")
    pa, pb = _Fp8Padded(a, ld_pad), _Fp8Padded(b, ld_pad)
    assert pa.view.stride(0) == K + ld_pad and ops.gemm_fp8_tn_supported(pa.view, pb.view, sa, sb)
    c = ops.gemm_fp8_tn(pa.view, pb.view, sa, sb, gs)
    acc = (ad @ bd.t()).float()
    assert_same_bits(c, (acc if g is None else acc * g).to(BF16), f"{what} vs float64")
    assert_same_bits(c, ops.gemm_fp8_tn(a, b, sa, sb, gs), f"{what} vs contiguous copies")
    pa.assert_intact(what)
    pb.assert_intact(what)


def _mse_case(M, N, K, gen):
    """check_mse's inputs: ternary x and w exact in E4M3, t = x w^T - d with d a few quanta (sparser on large outputs)
    so that sum d^2 is exact in the fp32 loss."""
    x, sx, xd = quantized(exact_bf16(ternary((M, K), 0.25, gen, 2.0 ** -3)), E4M3)
    w, sw, wd = quantized(exact_bf16(ternary((N, K), 0.25, gen, 2.0 ** -5)), E4M3)
    d = ints((M, N), 3, gen, 2.0 ** -8) if 9 * M * N < 2 ** 21 else ternary((M, N), 2.0 ** 21 / (M * N), gen, 2.0 ** -8)
    assert_exact_loss(d)
    return x, sx, w, sw, exact_bf16(xd @ wd.t() - d), d


MSE_SCALES = (2.0 ** -9, 2.0 ** -3)  # loss_scale, grad_scale


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", FP8_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_linear_mse_forward_fp8_local_on_views(shape, ld_pad):
    ops = _ops()
    M, N, K = shape
    what = f"linear_mse_forward_fp8_local {shape} ld=width+{ld_pad}"
    x, sx, w, sw, t, d = _mse_case(M, N, K, _gen(M, N, K, ld_pad, 7))
    px, pw, pt = _Fp8Padded(x, ld_pad), _Fp8Padded(w, ld_pad), _Padded(t, ld_pad)
    ls, gsc = MSE_SCALES
    assert ops.gemm_fp8_tn_supported(px.view, pw.view, sx, sw, pt.view)
    dy, loss, amax = ops.linear_mse_forward_fp8_local(px.view, pw.view, sx, sw, pt.view, ls, gsc)
    ref = (d * gsc).float().to(BF16)
    assert_same_bits(dy, ref, f"{what} dy vs float64")
    assert float(loss) == ls * float(d.square().sum()), what
    assert float(amax) == float(ref.float().abs().max()), what
    dy_c, loss_c, amax_c = ops.linear_mse_forward_fp8_local(x, w, sx, sw, pt.fresh(), ls, gsc)
    assert_same_bits(dy, dy_c, f"{what} vs contiguous copies")
    assert float(loss) == float(loss_c) and float(amax) == float(amax_c), what
    px.assert_intact(what)
    pw.assert_intact(what)
    pt.assert_intact(what)


def _sgd_operands(M, N, K, gen):
    """check_sgd's inputs: E5M2 a, E4M3 b, and a bf16 weight of integers on a 2^-7 grid."""
    a, sa, ad = quantized(exact_operand((M, K), gen, E5M2, 2.0 ** -6), E5M2)
    b, sb, bd = quantized(exact_operand((N, K), gen, E4M3, 2.0 ** -2), E4M3)
    return a, sa, ad, b, sb, bd, exact_bf16(ints((M, N), 200, gen, 2.0 ** -7))


@pytest.mark.parametrize("ld_pad", LD_PADS)
@pytest.mark.parametrize("shape", FP8_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_gemm_fp8_tn_sgd_on_views(shape, ld_pad):
    """The in-place update reads and writes the weight through its own row stride, and nothing around it."""
    ops = _ops()
    M, N, K = shape
    what = f"gemm_fp8_tn_sgd_ {shape} ld=width+{ld_pad}"
    a, sa, ad, b, sb, bd, w0 = _sgd_operands(M, N, K, _gen(M, N, K, ld_pad, 8))
    g, lr = 3.0, 2.0 ** -2
    gs = torch.full((1,), g, device="cuda")
    pa, pb, pw = _Fp8Padded(a, ld_pad), _Fp8Padded(b, ld_pad), _Padded(w0, ld_pad)
    w_contiguous = w0.clone()
    assert ops.gemm_fp8_tn_supported(pa.view, pb.view, sa, sb, None, pw.view)
    ops.gemm_fp8_tn_sgd_(pw.view, pa.view, pb.view, sa, sb, -lr, gs)
    ops.gemm_fp8_tn_sgd_(w_contiguous, a, b, sa, sb, -lr, gs)
    step = torch.tensor(g, dtype=F32) * torch.tensor(-lr, dtype=F32)
    ref = ((ad @ bd.t()).float() * step.cuda() + w0.float()).to(BF16)
    assert_same_bits(pw.view, ref, f"{what} vs float64")
    assert_same_bits(pw.view, w_contiguous, f"{what} vs a contiguous weight")
    pw.assert_padding_intact(what)
    pa.assert_intact(what)
    pb.assert_intact(what)


# ---- 2. gemm_fp8_tn_supported agrees with the ops -------------------------------------------------------------------
FP8_LAYOUTS = {  # name -> can the fp8 GEMMs read an fp8 operand in this layout in place?
    "contiguous": True,
    "column_slice": True,  # 16-byte offset, ld = K + 32
    "offset_16B": True,
    "offset_1B": False,
    "offset_8B": False,
    "offset_15B": False,
    "ld_not_multiple_of_16": False,
    "expand": False,
    "overlapping_rows": False,
}
TARGET_LAYOUTS = {  # the MSE target is read as bf16 pairs: a 4-byte-aligned base and an even row stride
    "contiguous": True,
    "column_slice": True,
    "offset_4B": True,
    "offset_16B": True,
    "expand": True,            # row stride 0: every row reads the same target row
    "overlapping_rows": True,  # read only: rows may share elements
    "offset_2B": False,
    "odd_ld": False,
}
WEIGHT_LAYOUTS = {  # the SGD weight is updated in place: a 16-byte-aligned base and a row stride % 8 == 0, >= N
    "contiguous": True,
    "column_slice": True,
    "offset_16B": True,
    "offset_2B": False,
    "offset_8B": False,
    "ld_not_multiple_of_8": False,
    "expand": False,
    "overlapping_rows": False,
}
PM, PN, PK = 130, 136, 96  # the predicate cases' shape


def _fp8_layout(q, name):
    """fp8 `q` [R, C] in the named layout, every byte outside the view 0x7F; "expand" and "overlapping_rows" derive
    their values from `q`."""
    if name == "contiguous":
        return q.clone()
    if name == "expand":
        return q[:1].expand(q.shape)
    u = q.view(torch.uint8)
    R, C = u.shape
    if name == "overlapping_rows":  # leading dimension C - 16: aligned, but rows share elements
        return u.flatten()[: (R - 1) * (C - 16) + C].clone().as_strided((R, C), (C - 16, 1)).view(q.dtype)
    if name.startswith("offset_"):
        off = int(name[len("offset_"):-1])
        v = torch.full((R * C + 32,), FP8_NAN, dtype=torch.uint8, device="cuda")[off:off + R * C].view(R, C)
    else:
        off, ld = {"column_slice": (16, C + 32), "ld_not_multiple_of_16": (0, C + 8)}[name]
        v = torch.full((off + R * ld,), FP8_NAN, dtype=torch.uint8, device="cuda").as_strided((R, C), (ld, 1), off)
    v.copy_(u)
    return v.view(q.dtype)


def _fresh(t):
    return t.clone(memory_format=torch.contiguous_format)


@pytest.mark.parametrize("layout", list(FP8_LAYOUTS))
@pytest.mark.parametrize("operand", ["a", "b"])
def test_fp8_predicate_agrees_with_gemm(operand, layout):
    ops = _ops()
    what = f"gemm_fp8_tn {operand} {layout}"
    gen = _gen(PM, PN, PK, len(layout), operand == "a")
    args = {"a": quantized(exact_operand((PM, PK), gen, E5M2, 2.0 ** -3), E5M2),
            "b": quantized(exact_operand((PN, PK), gen, E4M3, 2.0 ** -4), E4M3)}
    (a, sa, _), (b, sb, _) = args["a"], args["b"]
    if operand == "a":
        a = _fp8_layout(a, layout)
    else:
        b = _fp8_layout(b, layout)
    gs = torch.full((1,), 3.0, device="cuda")
    supported = bool(ops.gemm_fp8_tn_supported(a, b, sa, sb))
    assert supported == FP8_LAYOUTS[layout], f"{what}: the predicate says {supported}"
    if supported:
        assert_same_bits(ops.gemm_fp8_tn(a, b, sa, sb, gs), ops.gemm_fp8_tn(_fresh(a), _fresh(b), sa, sb, gs), what)
    else:
        _assert_raises_without_launch(lambda: ops.gemm_fp8_tn(a, b, sa, sb, gs), what)


@pytest.mark.parametrize("layout", list(TARGET_LAYOUTS))
def test_fp8_predicate_agrees_with_mse_target(layout):
    ops = _ops()
    what = f"linear_mse_forward_fp8_local target {layout}"
    x, sx, w, sw, t, _ = _mse_case(PM, PN, PK, _gen(PM, PN, PK, len(layout), 2))
    t = _layout(t, layout)
    supported = bool(ops.gemm_fp8_tn_supported(x, w, sx, sw, t))
    assert supported == TARGET_LAYOUTS[layout], f"{what}: the predicate says {supported}"
    run = lambda tt: ops.linear_mse_forward_fp8_local(x, w, sx, sw, tt, *MSE_SCALES)  # noqa: E731
    if supported:
        dy, loss, amax = run(t)
        dy_c, loss_c, amax_c = run(_fresh(t))
        assert_exact_loss(dy_c.double() / MSE_SCALES[1], what)  # the loss is exact, whatever order the atomics add
        assert_same_bits(dy, dy_c, what)
        assert float(loss) == float(loss_c) and float(amax) == float(amax_c), what
    else:
        _assert_raises_without_launch(lambda: run(t), what)


@pytest.mark.parametrize("layout", list(WEIGHT_LAYOUTS))
def test_fp8_predicate_agrees_with_sgd_weight(layout):
    ops = _ops()
    what = f"gemm_fp8_tn_sgd_ weight {layout}"
    a, sa, _, b, sb, _, w0 = _sgd_operands(PM, PN, PK, _gen(PM, PN, PK, len(layout), 3))
    w = _layout(w0, layout)
    gs = torch.full((1,), 3.0, device="cuda")
    supported = bool(ops.gemm_fp8_tn_supported(a, b, sa, sb, None, w))
    assert supported == WEIGHT_LAYOUTS[layout], f"{what}: the predicate says {supported}"
    before = _fresh(w)
    if supported:
        ops.gemm_fp8_tn_sgd_(w, a, b, sa, sb, -0.25, gs)
        ops.gemm_fp8_tn_sgd_(before, a, b, sa, sb, -0.25, gs)
        assert_same_bits(w, before, what)
    else:
        _assert_raises_without_launch(lambda: ops.gemm_fp8_tn_sgd_(w, a, b, sa, sb, -0.25, gs), what)
        assert_same_bits(w, before, f"{what}: the rejected weight changed")


# ---- 3. the batched and grouped expert ops on offset views --------------------------------------------------------
# (op, its operands, its predicate, the predicate's operands); the operands are named as in _expert_operands
BATCHED_OPS = [
    ("batched_linear_bias_gelu_forward", ("x", "w", "b"), "batched_gemm_tn_supported", ("x", "w", "b")),
    ("batched_linear_bias_forward", ("x", "w", "b"), "batched_gemm_tn_supported", ("x", "w", "b")),
    ("batched_gemm_nn_gelu_backward", ("dy", "wn", "z", "gs"), "batched_gemm_nn_supported", ("dy", "wn")),
    ("batched_gemm_nn", ("dy", "wn"), "batched_gemm_nn_supported", ("dy", "wn")),
    ("batched_wgrad_bf16", ("dyw", "x", "gs"), "batched_wgrad_bf16_supported", ("dyw", "x")),
    ("batched_column_sum", ("part", "gs"), None, ()),
]
GROUPED_OPS = [
    ("grouped_linear_bias_gelu_forward", ("x", "w", "b", "counts"), "grouped_gemm_tn_supported",
     ("x", "w", "counts", "b")),
    ("grouped_linear_bias_forward", ("x", "w", "b", "counts"), "grouped_gemm_tn_supported", ("x", "w", "counts", "b")),
    ("grouped_gemm_nn_gelu_backward", ("dy", "wn", "z", "counts"), "grouped_gemm_nn_supported", ("dy", "wn", "counts")),
    ("grouped_gemm_nn", ("dy", "wn", "counts"), "grouped_gemm_nn_supported", ("dy", "wn", "counts")),
    ("grouped_wgrad_bf16", ("dyw", "x", "counts", "gs"), "grouped_wgrad_bf16_supported", ("dyw", "x", "counts")),
    ("grouped_column_sum", ("part", "counts"), None, ()),
    ("grouped_column_sum", ("dyw", "counts"), None, ()),
]
OFFSET_COUNTS = [0, 1, 129, 300]  # an empty group, a one-row group, a partial second tile, a partial third tile


def _expert_operands(family, E=2, M=256, N=256, K=128, counts=OFFSET_COUNTS):
    """x, w [E, N, K], b [E, N] fp32, wn [E, K, N], z, dy, dyw (the wgrad's upstream gradient) and the column-sum
    partials of one family; the grouped rows hold NaN outside every group."""
    E = E if family == "batched" else len(counts)
    t = {"w": _randn(E, N, K, seed=2), "b": _randn(E, N, dtype=F32, seed=3), "wn": _randn(E, K, N, seed=4),
         "gs": torch.full((1,), 0.375, device="cuda")}
    if family == "batched":
        t.update(x=_randn(E, M, K, seed=1), dy=_randn(E, M, K, seed=5), z=_randn(E, M, N, seed=6),
                 dyw=_randn(E, M, N, seed=7), part=_randn(E, M // 16, N, dtype=F32, seed=8))
    else:
        R = _rows(counts)
        t.update(x=_grouped(counts, K, 1), dy=_grouped(counts, K, 5), z=_grouped(counts, N, 6),
                 dyw=_grouped(counts, N, 7), part=_randn(R // 16, N, dtype=F32, seed=8), counts=_counts(counts))
    return t


def _at_offset(t, nbytes, fill):
    """A contiguous copy of `t` whose base lies `nbytes` past the start of a fresh allocation filled with `fill`."""
    e, rem = divmod(nbytes, t.element_size())
    assert rem == 0
    v = torch.full((t.numel() + e + 16,), fill, dtype=t.dtype, device="cuda")[e:e + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 == nbytes % 16
    return v


class _CudaArray:
    """`__cuda_array_interface__` of a raw device pointer inside `owner`, which it keeps alive."""

    def __init__(self, owner, ptr, shape, typestr):
        self.owner = owner
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 3,
                                         "strides": None}


def _int32_at_2_bytes(counts):
    """A contiguous int32 tensor two bytes into an int8 buffer that holds the bytes of `counts` (torch cannot view one
    at that offset).  No device code may read it: an int32 load from it is a misaligned access.  Only the host-side
    checks of the ops look at it."""
    buf = torch.zeros(4 * counts.numel() + 16, dtype=torch.int8, device="cuda")
    buf[2:2 + 4 * counts.numel()].copy_(counts.view(torch.int8))
    v = torch.as_tensor(_CudaArray(buf, buf.data_ptr() + 2, tuple(counts.shape), "<i4"), device="cuda")
    ok = v.dtype == torch.int32 and v.is_contiguous() and v.data_ptr() == buf.data_ptr() + 2
    assert ok, "no int32 view two bytes into the buffer"
    return v


def _call(ops, name, names, t):
    return getattr(ops, name)(*(t[n] for n in names))


def _group_partials(part, counts):
    """The column-sum partial rows of the groups' rows (the kernel leaves those of the zero tiles unwritten)."""
    return torch.cat([part[s // 16:s // 16 + -(-c // 16)] for s, c in zip(_starts(counts), counts)])


def _same_outputs(op, got, want, counts, what):
    got, want = (got, want) if isinstance(got, tuple) else ((got,), (want,))
    if op == "grouped_gemm_nn_gelu_backward":
        got, want = (got[0], _group_partials(got[1], counts)), (want[0], _group_partials(want[1], counts))
    for i, (g, w) in enumerate(zip(got, want)):
        assert_same_bits(g, w, f"{what} output {i}")


@pytest.mark.parametrize("family", ["batched", "grouped"])
def test_expert_ops_on_offset_views(family):
    """Every operand a contiguous view at a 16-byte-aligned non-zero offset (the counts at 4 bytes), NaN around it."""
    ops = _ops()
    fresh = _expert_operands(family)
    views = {}
    for i, (n, t) in enumerate(sorted(fresh.items())):
        views[n] = _at_offset(t, 4, 1 << 30) if n == "counts" else _at_offset(t, 16 * (i + 1), NAN)
    for op, names, pred, pred_names in BATCHED_OPS if family == "batched" else GROUPED_OPS:
        what = f"{op}({', '.join(names)}) on offset views"
        if pred is not None:
            assert getattr(ops, pred)(*(views[n] for n in pred_names)), f"{what}: {pred} rejects them"
        _same_outputs(op, _call(ops, op, names, views), _call(ops, op, names, fresh), OFFSET_COUNTS, what)


REJECTED = [("batched", "x", 2), ("batched", "w", 2), ("batched", "wn", 2), ("batched", "b", 4), ("batched", "z", 2),
            ("batched", "dyw", 2), ("grouped", "x", 2), ("grouped", "w", 2), ("grouped", "wn", 2), ("grouped", "b", 4),
            ("grouped", "z", 2), ("grouped", "dyw", 2), ("grouped", "counts", 2)]


@pytest.mark.parametrize("family,operand,nbytes", REJECTED)
def test_expert_ops_reject_misaligned_operand(family, operand, nbytes):
    """A contiguous operand whose base is `nbytes` off alignment: every predicate that takes it says no, and every op
    that needs it aligned raises on the host without a launch.  That is every op that reads it, except the grouped
    column sum, which reads its bf16 / fp32 input element by element but its counts as int32 words."""
    ops = _ops()
    t = _expert_operands(family)
    t[operand] = _int32_at_2_bytes(t[operand]) if operand == "counts" else _at_offset(t[operand], nbytes, NAN)
    readers = [c for c in (BATCHED_OPS if family == "batched" else GROUPED_OPS)
               if operand in c[3] or (operand in c[1] and operand in ("z", "counts"))]
    assert readers
    for op, names, pred, pred_names in readers:
        if operand in pred_names:
            accepted = bool(getattr(ops, pred)(*(t[n] for n in pred_names)))  # a plain bool: the assertion reprs no tensor
            assert not accepted, f"{pred} accepts {operand} at +{nbytes} B"
    for op, names, _, _ in readers:
        _assert_raises_without_launch(lambda: _call(ops, op, names, t), f"{op} with {operand} at +{nbytes} B")


@pytest.mark.parametrize("grouped", [False, True], ids=["expert_mlp", "grouped_expert_mlp"])
def test_node_takes_a_misaligned_upstream_gradient(grouped):
    """The forward runs on the kernels; the upstream gradient is contiguous but 2 bytes off alignment (a slice of a
    larger buffer).  The gradients equal those of an aligned copy of it, and the backward runs on the kernels."""
    from mpi4torch_b200.ops import expert_mlp, expert_mlp_supported, grouped_expert_mlp, grouped_expert_mlp_supported

    E, M, D, H, O = 3, 128, 128, 256, 128
    counts = _counts([5, 0, 200])
    x = _grouped(counts.tolist(), D, 1, 0.0) if grouped else _randn(E, M, D, seed=1)
    w1, b1 = _randn(E, H, D, seed=2) * 0.1, _randn(E, H, dtype=F32, seed=3)
    w2, b2 = _randn(E, O, H, seed=4) * 0.1, _randn(E, O, dtype=F32, seed=5)
    lead = (x, counts) if grouped else (x,)
    supported = grouped_expert_mlp_supported if grouped else expert_mlp_supported
    node = grouped_expert_mlp if grouped else expert_mlp
    assert supported(*lead, w1, b1, w2, b2)
    kernel = "gemm_nn_gelu_bwd_colsum_grouped" if grouped else "gemm_nn_gelu_bwd_colsum_batched"

    def grads(dy):
        ins = [t.detach().clone().requires_grad_() for t in (x, w1, b1, w2, b2)]
        y = node(ins[0], *lead[1:], *ins[1:])
        before = _launches().get(kernel, 0)
        y.backward(dy)
        assert _launches().get(kernel, 0) == before + 1, "the backward left the kernels"
        return [t.grad for t in ins]

    shape = (x.shape[0], O) if grouped else (E, M, O)
    dy = _randn(*shape, seed=6)
    misaligned = _at_offset(dy, 2, NAN)
    assert misaligned.is_contiguous() and misaligned.data_ptr() % 16 == 2
    want = grads(dy.clone())
    got = grads(misaligned)
    for name, g, w in zip(("x", "w1", "b1", "w2", "b2"), got, want):
        assert_same_bits(g, w, f"{'grouped_' if grouped else ''}expert_mlp d{name}")


# ---- 4. limits -----------------------------------------------------------------------------------------------------
LIMIT_COUNTS = (0, 1, 127, 128, 129, 300)


def test_grouped_ops_at_1024_groups():
    """E = 1024 fills the kernels' shared-memory group table: every grouped op equals the single-expert op on each
    group's rows, padding rows are zero, and empty groups get zero weight gradients and column sums."""
    ops = _ops()
    counts = [LIMIT_COUNTS[e % len(LIMIT_COUNTS)] for e in range(1024)]
    E, N, K = len(counts), 128, 128
    t = _expert_operands("grouped", E=E, N=N, K=K, counts=counts)
    cnt, gs = t["counts"], t["gs"]
    for op, names, pred, pred_names in GROUPED_OPS:
        if pred is not None:
            assert getattr(ops, pred)(*(t[n] for n in pred_names)), f"{pred} rejects 1024 groups"
    h, z = ops.grouped_linear_bias_gelu_forward(t["x"], t["w"], t["b"], cnt)
    y = ops.grouped_linear_bias_forward(t["x"], t["w"], t["b"], cnt)
    dz, part = ops.grouped_gemm_nn_gelu_backward(t["dy"], t["wn"], t["z"], cnt)
    c_nn = ops.grouped_gemm_nn(t["dy"], t["wn"], cnt)
    db = ops.grouped_column_sum(part, cnt)
    gw = ops.grouped_wgrad_bf16(t["dyw"], t["x"], cnt, gs)
    sums = ops.grouped_column_sum(t["dyw"], cnt)
    got, want = {}, {}

    def add(name, g, w):
        got.setdefault(name, []).append(g.flatten())
        want.setdefault(name, []).append(w.flatten())

    empty = []
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if c == 0:
            empty.append(e)
            continue
        h1, z1 = ops.linear_bias_gelu_forward(t["x"][s:s + c], t["w"][e], t["b"][e])
        add("h", h[s:s + c], h1), add("z", z[s:s + c], z1), add("y", y[s:s + c], z1)
        dz1, part1 = ops.gemm_nn_gelu_backward(t["dy"][s:s + c], t["wn"][e], t["z"][s:s + c])
        add("dz", dz[s:s + c], dz1), add("partials", part[s // 16:s // 16 + part1.shape[0]], part1)
        add("nn", c_nn[s:s + c], ops.gemm_bf16_nn(t["dy"][s:s + c], t["wn"][e]))
        add("column sum", db[e], ops.column_sum(part1))
        pad = -(-c // 64) * 64
        dy_e = torch.zeros(pad, N, device="cuda", dtype=BF16)
        x_e = torch.zeros(pad, K, device="cuda", dtype=BF16)
        dy_e[:c], x_e[:c] = t["dyw"][s:s + c], t["x"][s:s + c]
        add("wgrad", gw[e], ops.wgrad_bf16(dy_e, x_e, gs))
        add("row sum", sums[e], t["dyw"][s:s + c].double().sum(0))
        add("row sum bound", sums[e], 1e-5 * t["dyw"][s:s + c].double().abs().sum(0))
    bound = torch.cat(want.pop("row sum bound"))
    got.pop("row sum bound")
    for name in got:
        g, w = torch.cat(got[name]), torch.cat(want[name])
        if name == "row sum":
            err = (g.double() - w).abs()
            assert bool((err <= bound).all()), f"1024 groups: row sums off by up to {float((err - bound).max()):.3g}"
        else:
            assert_same_bits(g, w, f"1024 groups: {name}")
    for v, n in ((h, "h"), (z, "z"), (y, "y"), (dz, "dz"), (c_nn, "nn")):
        _assert_zero_padding(v, counts, f"1024 groups: {n}")
    idx = torch.tensor(empty, device="cuda")
    assert len(empty) == 171 and empty[-1] == 1020
    for v, n in ((gw, "wgrad"), (db, "column sum"), (sums, "row sum")):
        assert bool((v[idx] == 0).all()), f"1024 groups: an empty group has a non-zero {n}"


@pytest.mark.parametrize("case", ["E1025", "empty_counts"])
def test_grouped_ops_reject_1025_groups_and_empty_counts(case):
    """Past the group table, or with no group at all: every grouped predicate says no, every grouped op raises without
    a launch, and grouped_expert_mlp runs its composition."""
    from mpi4torch_b200.ops import grouped_expert_mlp, grouped_expert_mlp_supported

    ops = _ops()
    counts = [0] * 1020 + [5, 0, 130, 0, 2] if case == "E1025" else []
    E, R, N, K = len(counts), 512, 128, 128
    t = {"x": _randn(R, K, seed=1), "dy": _randn(R, K, seed=5), "z": _randn(R, N, seed=6), "dyw": _randn(R, N, seed=7),
         "part": _randn(R // 16, N, dtype=F32, seed=8), "w": _randn(E, N, K, seed=2), "b": _randn(E, N, dtype=F32, seed=3),
         "wn": _randn(E, K, N, seed=4), "counts": _counts(counts) if counts else torch.empty(0, dtype=torch.int32,
                                                                                          device="cuda"),
         "gs": torch.full((1,), 1.0, device="cuda")}
    w1, b1 = _randn(E, N, K, seed=9) * 0.1, _randn(E, N, dtype=F32, seed=10)
    w2, b2 = _randn(E, N, N, seed=11) * 0.1, _randn(E, N, dtype=F32, seed=12)
    # every predicate first: nothing below may launch a kernel with a table that does not fit
    for op, names, pred, pred_names in GROUPED_OPS:
        if pred is not None:
            assert not getattr(ops, pred)(*(t[n] for n in pred_names)), f"{pred} accepts {case}"
    assert not grouped_expert_mlp_supported(t["x"], t["counts"], w1, b1, w2, b2), f"the node accepts {case}"
    for op, names, _, _ in GROUPED_OPS:
        _assert_raises_without_launch(lambda: _call(ops, op, names, t), f"{op} with {case}")
    x = t["x"].clone().requires_grad_()
    before = _launch_count()
    y = grouped_expert_mlp(x, t["counts"], w1, b1, w2, b2)
    if y.requires_grad:
        y.float().sum().backward()
    torch.cuda.synchronize()
    assert _launch_count() == before, f"{case}: the composition launched a library kernel"
    ref = torch.zeros(R, N, device="cuda")
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        if c:
            hid = torch.nn.functional.gelu(x[s:s + c].detach().float() @ w1[e].float().t() + b1[e], approximate="tanh")
            ref[s:s + c] = hid @ w2[e].float().t() + b2[e]
    torch.testing.assert_close(y.float(), ref.to(BF16).float(), rtol=2e-2, atol=2e-2)


def test_batched_ops_at_1024_experts():
    """E = 1024 at M = 128: the first, the last and a few experts between equal the single-expert ops."""
    ops = _ops()
    E, M, N, K = 1024, 128, 128, 128
    t = _expert_operands("batched", E=E, M=M, N=N, K=K)
    gs = t["gs"]
    for op, names, pred, pred_names in BATCHED_OPS:
        if pred is not None:
            assert getattr(ops, pred)(*(t[n] for n in pred_names)), f"{pred} rejects 1024 experts"
    h, z = ops.batched_linear_bias_gelu_forward(t["x"], t["w"], t["b"])
    y = ops.batched_linear_bias_forward(t["x"], t["w"], t["b"])
    dz, part = ops.batched_gemm_nn_gelu_backward(t["dy"], t["wn"], t["z"], gs)
    c_nn = ops.batched_gemm_nn(t["dy"], t["wn"])
    gw = ops.batched_wgrad_bf16(t["dyw"], t["x"], gs)
    db = ops.batched_column_sum(part, gs)
    for e in (0, 1, 131, 132, 511, 512, 1000, 1022, 1023):
        h1, z1 = ops.linear_bias_gelu_forward(t["x"][e], t["w"][e], t["b"][e])
        dz1, part1 = ops.gemm_nn_gelu_backward(t["dy"][e], t["wn"][e], t["z"][e], gs)
        for got, ref, n in ((h[e], h1, "h"), (z[e], z1, "z"), (y[e], z1, "y"), (dz[e], dz1, "dz"),
                            (part[e], part1, "partials"), (c_nn[e], ops.gemm_bf16_nn(t["dy"][e], t["wn"][e]), "nn"),
                            (gw[e], ops.wgrad_bf16(t["dyw"][e], t["x"][e], gs), "wgrad"),
                            (db[e], ops.column_sum(part1, gs), "column sum")):
            assert_same_bits(got, ref, f"1024 experts: {n}[{e}]")


# Outputs of more than 2^31 elements.  Each case checks free memory first and skips (the GPU is shared), keeps its
# large tensors in `mem`, which frees them when the case ends, and checks the output in row chunks: against the
# float64 (exact) or fp32 reference, and bit for bit against the single-matrix op on the same rows.
def test_gemm_fp8_tn_output_beyond_2_31_elements(mem):
    M, N, K = 131072, 16392, 64
    assert M * N > 2 ** 31
    _require_free(M * N * 2)
    ops = _ops()
    gen = _gen(M, N, K)
    mem["a"], sa, mem["ad"] = quantized(exact_operand((M, K), gen, E4M3, 2.0 ** -3), E4M3)
    mem["b"], sb, mem["bd"] = quantized(exact_operand((N, K), gen, E4M3, 2.0 ** -4), E4M3)
    mem["c"] = ops.gemm_fp8_tn(mem["a"], mem["b"], sa, sb)
    for r0, r1 in _chunks(M):
        assert_same_bits(mem["c"][r0:r1], (mem["ad"][r0:r1] @ mem["bd"].t()).float().to(BF16),
                         f"gemm_fp8_tn rows {r0}:{r1}")


def test_batched_linear_bias_forward_output_beyond_2_31_elements(mem):
    E, M, N, K = 8, 16384, 16512, 128
    assert E * M * N > 2 ** 31 > (E - 1) * M * N  # the last expert's output straddles 2^31
    _require_free(E * M * N * 2)
    ops = _ops()
    mem["x"], mem["w"] = _randn(E, M, K, seed=1), _randn(E, N, K, seed=2) * K ** -0.5
    mem["b"] = _randn(E, N, dtype=F32, seed=3)
    mem["y"] = ops.batched_linear_bias_forward(mem["x"], mem["w"], mem["b"])
    for e in range(E):
        for r0, r1 in _chunks(M):
            what = f"batched_linear_bias_forward expert {e} rows {r0}:{r1}"
            xe, we, be = mem["x"][e, r0:r1], mem["w"][e], mem["b"][e]
            _assert_close_bf16(mem["y"][e, r0:r1], xe.float() @ we.float().t() + be, K=K, what=what)
            assert_same_bits(mem["y"][e, r0:r1], ops.linear_bias_gelu_forward(xe, we, be)[1], what)


def test_grouped_gemm_nn_output_beyond_2_31_elements(mem):
    counts = [40000, 50000, 41000, 300]
    E, N, K = len(counts), 16384, 128
    R, last = _rows(counts), _starts(counts)[-1]
    assert last * N > 2 ** 31  # the last group's rows start past 2^31 output elements
    _require_free(R * N * 2)
    ops = _ops()
    mem["a"], mem["b"] = _grouped(counts, K, 1), _randn(E, K, N, seed=2) * K ** -0.5
    cnt = _counts(counts)
    mem["c"] = ops.grouped_gemm_nn(mem["a"], mem["b"], cnt)
    for e, (s, c) in enumerate(zip(_starts(counts), counts)):
        for r0, r1 in _chunks(c):
            what = f"grouped_gemm_nn group {e} rows {s + r0}:{s + r1}"
            ae = mem["a"][s + r0:s + r1]
            _assert_close_bf16(mem["c"][s + r0:s + r1], ae.float() @ mem["b"][e].float(), K=K, what=what)
            assert_same_bits(mem["c"][s + r0:s + r1], ops.gemm_bf16_nn(ae, mem["b"][e]), what)
    _assert_zero_padding(mem["c"], counts, "grouped_gemm_nn beyond 2^31")


def test_batched_wgrad_bf16_output_beyond_2_31_elements(mem):
    E, Mb, N, K = 2, 64, 32768, 32896
    assert E * N * K > 2 ** 31
    _require_free(E * N * K * 2)
    ops = _ops()
    mem["dy"], mem["x"] = _randn(E, Mb, N, seed=1), _randn(E, Mb, K, seed=2)
    mem["gw"] = ops.batched_wgrad_bf16(mem["dy"], mem["x"])
    for e in range(E):
        for r0, r1 in _chunks(N, 4096):
            what = f"batched_wgrad_bf16 expert {e} rows {r0}:{r1}"
            dye = mem["dy"][e, :, r0:r1]
            _assert_close_bf16(mem["gw"][e, r0:r1], dye.float().t() @ mem["x"][e].float(), K=Mb, what=what)
            assert_same_bits(mem["gw"][e, r0:r1], ops.wgrad_bf16(dye, mem["x"][e]), what)
