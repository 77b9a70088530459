"""Float64 emulation of the unicast all-reduce kernels (csrc/kernels/allreduce.cu) and of the peer-store fused
wgrad -> reduce-scatter -> SGD kernel (csrc/kernels/wgrad_wgmma.cu), rounding exactly where the kernels round.

The unicast kernels reduce in a fixed rank order, so random inputs can be emulated bit for bit:
  * reduce in the accumulation type of Elem<DT> (reduce_ops.h): f32 for bf16 / f16 / f32, f64 for f64, u32 for
    u8 / bool, i32 for i8 / i16 / i32, i64 for i64, integers wrapping around; start from normalise_single;
  * scale: floats multiply by fl32(scale) (f64: by the double), integers truncate double(v) * scale toward zero;
  * one-shot: add the accumulate operand, then store once (RNE for bf16 / f16);
  * two-shot and pipelined: store the scaled reduction (phase B), then load it, add the accumulate operand and store
    again (phase C): a 16-bit float with an accumulate operand is rounded twice.
MIN / MAX follow Combine: a later NaN wins, and a tie keeps the earlier rank's value (max(-0, +0) keeps rank 0's).

Everything here runs on the CPU with numpy and torch; storage is kept as raw bits (bf16 / f16 as uint16)."""
import numpy as np
import torch

OPS = {"MAX": 0, "MIN": 1, "SUM": 2, "PROD": 3, "LAND": 4, "BAND": 5, "LOR": 6, "BOR": 7, "LXOR": 8, "BXOR": 9}
BITWISE = ("BAND", "BOR", "BXOR")
FLOAT_DTYPES = (torch.float32, torch.float64, torch.bfloat16, torch.float16)
INT_DTYPES = (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.bool)
ALL_DTYPES = INT_DTYPES + FLOAT_DTYPES

# storage (numpy view of the raw bits) and accumulation type of every dtype
_STORAGE = {torch.uint8: np.uint8, torch.int8: np.int8, torch.int16: np.int16, torch.int32: np.int32,
            torch.int64: np.int64, torch.bool: np.uint8, torch.float32: np.float32, torch.float64: np.float64,
            torch.bfloat16: np.uint16, torch.float16: np.uint16}
_ACC = {torch.uint8: np.uint32, torch.int8: np.int32, torch.int16: np.int32, torch.int32: np.int32,
        torch.int64: np.int64, torch.bool: np.uint32, torch.float32: np.float32, torch.float64: np.float64,
        torch.bfloat16: np.float32, torch.float16: np.float32}
_TORCH_BITS = {torch.bfloat16: torch.int16, torch.float16: torch.int16, torch.bool: torch.uint8}


def ops_for(dtype):
    """The ops check_op_dtype accepts for `dtype` (bitwise ops are rejected for floats)."""
    return [o for o in OPS if not (dtype.is_floating_point and o in BITWISE)]


def storage_type(dtype):
    """The numpy type of dtype's raw storage."""
    return _STORAGE[dtype]


def bits_of(t, dtype):
    """Numpy storage array of a tensor of `dtype`."""
    t = t.detach().cpu().contiguous()
    if dtype in _TORCH_BITS:
        t = t.view(_TORCH_BITS[dtype])
    return t.numpy().copy().view(_STORAGE[dtype])


def tensor_of(bits, dtype):
    """Inverse of bits_of."""
    t = torch.from_numpy(np.ascontiguousarray(bits))
    if dtype in (torch.bfloat16, torch.float16):
        return t.view(torch.int16).view(dtype)
    if dtype == torch.bool:
        return t.view(torch.bool)
    return t


def f32_to_bf16_bits(f):
    """float_to_bf16_bits of reduce_ops.h: RNE, NaN keeps its payload (quietened)."""
    u = np.asarray(f, dtype=np.float32).view(np.uint32).astype(np.uint64)
    nan = (u & 0x7FFFFFFF) > 0x7F800000
    rne = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    return np.where(nan, (u >> 16) | 0x40, rne).astype(np.uint16)


def bf16_bits_to_f32(b):
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def f32_to_f16_bits(f):
    """RNE to f16 (overflow to inf, subnormals kept); a NaN becomes sign | 0x7e00 (the host conversion).  The device
    conversion's NaN payload is not pinned: compare f16 NaNs by position only."""
    f = np.asarray(f, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        h = f.astype(np.float16).view(np.uint16)
    sign = (f.view(np.uint32) >> 16).astype(np.uint16) & 0x8000
    return np.where(np.isnan(f), sign | 0x7E00, h).astype(np.uint16)


def load(bits, dtype):
    """Elem<DT>::load: storage -> accumulation type."""
    if dtype == torch.bfloat16:
        return bf16_bits_to_f32(bits)
    if dtype == torch.float16:
        return np.asarray(bits, dtype=np.uint16).view(np.float16).astype(np.float32)
    if dtype == torch.bool:
        return (bits != 0).astype(np.uint32)
    return bits.astype(_ACC[dtype])


def store(acc, dtype):
    """Elem<DT>::store: accumulation type -> storage (one rounding)."""
    if dtype == torch.bfloat16:
        return f32_to_bf16_bits(acc)
    if dtype == torch.float16:
        return f32_to_f16_bits(acc)
    if dtype == torch.bool:
        return (acc != 0).astype(np.uint8)
    return acc.astype(_STORAGE[dtype])


def combine(a, b, op, is_float):
    """Combine<OP, A> of reduce_ops.h, elementwise over the accumulation type."""
    with np.errstate(over="ignore", invalid="ignore"):
        if op == "MAX":
            return np.where((b > a) | (np.isnan(b) if is_float else False), b, a)
        if op == "MIN":
            return np.where((b < a) | (np.isnan(b) if is_float else False), b, a)
        if op == "SUM":
            return a + b
        if op == "PROD":
            return a * b
        if op == "LAND":
            return ((a != 0) & (b != 0)).astype(a.dtype)
        if op == "LOR":
            return ((a != 0) | (b != 0)).astype(a.dtype)
        if op == "LXOR":
            return ((a != 0) != (b != 0)).astype(a.dtype)
        if op == "BAND":
            return a & b
        if op == "BOR":
            return a | b
        if op == "BXOR":
            return a ^ b
    raise ValueError(op)


def normalise_single(a, op):
    if op in ("LAND", "LOR", "LXOR"):
        return (a != 0).astype(a.dtype)
    return a


def scale_acc(acc, scale, dtype):
    """ScaleAcc: fl32(scale) for f32 accumulators, the double for f64, truncation toward zero for integers."""
    with np.errstate(over="ignore", invalid="ignore"):
        if _ACC[dtype] == np.float32:
            return acc * np.float32(scale)
        if _ACC[dtype] == np.float64:
            return acc * np.float64(scale)
        return np.trunc(acc.astype(np.float64) * np.float64(scale)).astype(_ACC[dtype])


def add_acc(acc, operand_bits, dtype):
    with np.errstate(over="ignore", invalid="ignore"):
        return acc + load(operand_bits, dtype)


def allreduce(xs, op, dtype, scale=None, acc=None, two_phase=False):
    """Bits every rank holds after the unicast all-reduce of xs (a list of storage arrays, rank order).

    scale: None or a float; acc: None or the accumulate operand's storage array.  two_phase: the two-shot /
    pipelined kernels (and the host backend's two-phase path), which store the scaled reduction before the
    accumulate operand is added."""
    is_float = dtype.is_floating_point
    a = normalise_single(load(xs[0], dtype), op)
    for x in xs[1:]:
        a = combine(a, load(x, dtype), op, is_float)
    if scale is not None:
        a = scale_acc(a, scale, dtype)
    if acc is None:
        return store(a, dtype)
    if two_phase:
        a = load(store(a, dtype), dtype)
    return store(add_acc(a, acc, dtype), dtype)


def nan_bits_pinned(dtype, op, scale, acc):
    """True where the kernels' NaN bit patterns are defined by selection alone: MIN / MAX without an arithmetic
    epilogue, for every float type whose conversions keep the payload (not f16: the device conversion to f16 does
    not).  Elsewhere a NaN's payload comes from the hardware's arithmetic and only its position is compared."""
    return op in ("MAX", "MIN") and scale is None and acc is None and dtype != torch.float16


def assert_bits(got, want, dtype, exact_nan=True, what=""):
    """got, want: storage arrays.  Bit equality; at the reference's NaNs the result must be NaN, with the same bits
    when exact_nan."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} vs {want.shape}"
    raw = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[got.itemsize]
    bad = got.view(raw) != want.view(raw)  # raw bits: the sign of zero and NaN payloads count
    if dtype.is_floating_point:
        gnan, wnan = np.isnan(load(got, dtype)), np.isnan(load(want, dtype))
        if not exact_nan:
            bad &= ~(wnan & gnan)
        bad |= gnan != wnan
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements differ, first at {i}: "
                             f"got {got.reshape(-1)[i]!r} want {want.reshape(-1)[i]!r} "
                             f"(bits {got.view(raw).reshape(-1)[i]:#x} vs {want.view(raw).reshape(-1)[i]:#x})")


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
_SUBNORMAL = {torch.float32: 2.0 ** -140, torch.float64: 2.0 ** -1060, torch.bfloat16: 2.0 ** -130,
              torch.float16: 2.0 ** -20}


def make_input(dtype, n, gen, rank=0):
    """Random values of dtype (gen: a numpy Generator) with the edges mixed in: for floats NaN (with a rank-specific
    payload), +-inf, +-0 and subnormals; for integers the wrap edges (min, max, -1, 0, 1)."""
    if dtype == torch.bool:
        return torch.from_numpy(gen.integers(0, 2, n).astype(bool))
    if dtype.is_floating_point:
        v = gen.standard_normal(n) * np.exp2(gen.integers(-4, 4, n))
        bits = bits_of(torch.from_numpy(v).to(dtype), dtype)
        raw = bits.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[bits.itemsize])
        # distinct quiet-NaN payloads per rank, so "a later NaN wins" is visible in the bits
        nan = {torch.float32: 0x7FC00000 | ((rank * 7 + 1) & 0x3FFFFF), torch.float64: 0x7FF8000000000000 | (rank * 7 + 1),
               torch.bfloat16: 0x7FC0 | ((rank * 7 + 1) & 0x3F), torch.float16: 0x7E00 | ((rank * 7 + 1) & 0x1FF)}[dtype]
        sub = _SUBNORMAL[dtype]
        specials = [bits_of(torch.tensor([c], dtype=dtype), dtype).view(raw.dtype)[0]
                    for c in (float("inf"), float("-inf"), 0.0, -0.0, sub, -3 * sub)]
        specials = [raw.dtype.type(nan)] + specials
    else:
        st = _STORAGE[dtype]
        info = np.iinfo(st)
        raw = gen.integers(info.min, info.max, n, dtype=st, endpoint=True)
        specials = [st(info.max), st(info.min), st(0), st(1)] + ([st(-1)] if info.min < 0 else [])
    pick = gen.integers(0, 40 if dtype.is_floating_point else 12, n)
    for k, c in enumerate(specials):
        raw[pick == k] = c
    return tensor_of(raw.view(_STORAGE[dtype]), dtype)


# ---------------------------------------------------------------------------------------------------------------
# fused wgrad -> reduce-scatter -> SGD, peer-store mode
# ---------------------------------------------------------------------------------------------------------------
def make_sched(num_tiles, num_ctas, ksplit):
    """make_sched of wgrad_wgmma.cu (mirrored in test_protocol_models.py): tiles [0, whole) run over the full batch,
    tiles [whole, num_tiles) of the last partial wave are split in `ksplit` batch slices."""
    whole = (num_tiles // num_ctas) * num_ctas if ksplit > 1 else num_tiles
    return whole, ksplit, whole + (num_tiles - whole) * ksplit


def fmaf(a, b, c):
    """Correctly rounded fp32 fmaf(a, b, c) of fp32 arrays: the exact product in fp64, the sum rounded to odd in
    fp64 (TwoSum gives the exact error), then one RNE to fp32."""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b  # 24 x 24 bits: exact
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    odd = (s.view(np.uint64) & 1) == 1
    fix = (err != 0) & ~odd
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def fused_wgrad_sgd(w, dys, xs, scale, gscale, ksplit, grid, prefetch):
    """Emulation of consecutive calls of the peer-store fused kernel.  w: bf16 [N, K]; dys[c][p] bf16 [Mb, N],
    xs[c][p] bf16 [Mb, K]; every per-half G must be exact in fp32 (integers below 2^24 here).  Returns the final
    weights (bf16) and the W_avg of the last call (bf16, or None).

    Per call: rank p's partial tile is bf16(fl32(gs * G_{p,h})), one per batch half h for the split tiles of the last
    wave; the owner sums the partials in fp32 in the order p0h0, p0h1, p1h0, ...; W' = bf16(fmaf(scale, sum, W));
    with prefetch W_avg = bf16(fl32(rank-order sum of W') * fl32(1 / P))."""
    N, K = w.shape
    P = len(dys[0])
    gs = np.float32(1.0 if gscale is None else gscale)
    n_tiles, k_tiles = N // 128, K // 128
    whole, split, _ = make_sched(n_tiles * k_tiles, grid, ksplit)
    tile_split = np.arange(n_tiles * k_tiles).reshape(n_tiles, k_tiles) >= whole
    split_mask = np.repeat(np.repeat(tile_split, 128, axis=0), 128, axis=1)
    W = bf16_bits_to_f32(bits_of(w, torch.bfloat16)).reshape(N, K)

    def partial(g):
        return bf16_bits_to_f32(f32_to_bf16_bits(gs * g.astype(np.float32)))

    wavg = None
    for dy_c, x_c in zip(dys, xs):
        a = np.zeros((N, K), dtype=np.float32)
        for dy, x in zip(dy_c, x_c):
            dy, x = dy.double().numpy(), x.double().numpy()
            Mb = dy.shape[0]
            halves = [dy[h * Mb // split:(h + 1) * Mb // split].T @ x[h * Mb // split:(h + 1) * Mb // split]
                      for h in range(split)]
            full = sum(halves)
            bound = Mb * np.abs(dy).max() * np.abs(x).max()
            assert bound < 2 ** 22, "G is not exact in fp32 for every summation order"
            a = a + np.where(split_mask, partial(halves[0]), partial(full))
            for h in range(1, split):
                a = a + np.where(split_mask, partial(halves[h]), np.float32(0))
        W = bf16_bits_to_f32(f32_to_bf16_bits(fmaf(np.float32(scale), a, W)))
        if prefetch:
            s = np.zeros((N, K), dtype=np.float32)
            for _ in range(P):
                s = s + W
            wavg = f32_to_bf16_bits(s * np.float32(1.0 / P))
    out = tensor_of(f32_to_bf16_bits(W), torch.bfloat16)
    return out, (tensor_of(wavg, torch.bfloat16) if prefetch else None)
