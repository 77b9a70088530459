"""The emulation of the unicast all-reduce and fused wgrad -> SGD kernels (virtual_ranks_emulation.py), checked on the
CPU: hand-made cases for each of its rounding rules, and every (dtype, op) pair bit for bit against the host backend,
whose reduction (host_kernels.h) uses the same element tables and the same one-/two-phase split."""
import numpy as np
import pytest
import torch

import virtual_ranks_emulation as emu
from conftest import run_spmd

BF16, F16 = torch.bfloat16, torch.float16


def _bits(values, dtype):
    return emu.bits_of(torch.tensor(values, dtype=dtype), dtype)


def _value(bits, dtype):
    return emu.tensor_of(bits, dtype).double().tolist()


def test_bf16_sum_with_accumulate_rounds_once_in_one_shot_and_twice_in_two_shot():
    # 1 + 2^-8 is a tie between two bf16 values: stored before the accumulate operand (two-shot) it rounds to even,
    # 1.0, and adding 2^-8 ties again; summed in fp32 with the operand first (one-shot) it is 1 + 2^-7 exactly
    xs = [_bits([1.0], BF16), _bits([2.0 ** -8], BF16)]
    acc = _bits([2.0 ** -8], BF16)
    assert _value(emu.allreduce(xs, "SUM", BF16, acc=acc), BF16) == [1.0 + 2.0 ** -7]
    assert _value(emu.allreduce(xs, "SUM", BF16, acc=acc, two_phase=True), BF16) == [1.0]
    # without an accumulate operand both store once
    assert _value(emu.allreduce(xs, "SUM", BF16, two_phase=True), BF16) == [1.0]
    # f16 has the same double rounding one binade lower; fp32 stores are exact, so f32 does not
    h = [_bits([1.0], F16), _bits([2.0 ** -11], F16)]
    assert _value(emu.allreduce(h, "SUM", F16, acc=_bits([2.0 ** -11], F16)), F16) == [1.0 + 2.0 ** -10]
    assert _value(emu.allreduce(h, "SUM", F16, acc=_bits([2.0 ** -11], F16), two_phase=True), F16) == [1.0]
    f = [_bits([1.0], torch.float32), _bits([2.0 ** -24], torch.float32)]
    one = emu.allreduce(f, "SUM", torch.float32, acc=_bits([2.0 ** -24], torch.float32))
    two = emu.allreduce(f, "SUM", torch.float32, acc=_bits([2.0 ** -24], torch.float32), two_phase=True)
    assert (one == two).all()


def test_scale_is_applied_in_the_accumulation_type():
    # fp32 accumulators multiply by fl32(0.1), fp64 by the double 0.1
    x = [_bits([3.0], torch.float32), _bits([0.0], torch.float32)]
    assert emu.allreduce(x, "SUM", torch.float32, scale=0.1)[0] == np.float32(3.0) * np.float32(0.1)
    d = [_bits([3.0], torch.float64), _bits([0.0], torch.float64)]
    assert emu.allreduce(d, "SUM", torch.float64, scale=0.1)[0] == 3.0 * 0.1
    # bf16 is scaled in fp32 before its single rounding
    b = [_bits([3.0], BF16), _bits([0.0], BF16)]
    want = emu.f32_to_bf16_bits(np.float32(3.0) * np.float32(0.1))
    assert emu.allreduce(b, "SUM", BF16, scale=0.1)[0] == want


def test_min_max_keep_the_earlier_rank_on_ties_and_the_later_nan():
    f32 = torch.float32
    neg, pos = _bits([-0.0], f32), _bits([0.0], f32)
    for op in ("MAX", "MIN"):
        assert np.signbit(emu.allreduce([neg, pos], op, f32).view(np.float32))[0]
        assert not np.signbit(emu.allreduce([pos, neg], op, f32).view(np.float32))[0]
    nan_a = np.array([0x7FC00001], dtype=np.uint32).view(np.float32)
    nan_b = np.array([0x7FC00002], dtype=np.uint32).view(np.float32)
    five = np.array([5.0], dtype=np.float32)
    for op in ("MAX", "MIN"):
        # a later NaN replaces an earlier one, a number never replaces a NaN, a NaN replaces any number
        assert emu.allreduce([nan_a, nan_b], op, f32).view(np.uint32)[0] == 0x7FC00002
        assert emu.allreduce([nan_a, five], op, f32).view(np.uint32)[0] == 0x7FC00001
        assert emu.allreduce([five, nan_b, five], op, f32).view(np.uint32)[0] == 0x7FC00002
    # bf16 keeps the payload through the fp32 accumulator and the store
    nb = np.array([0x7FC3], dtype=np.uint16)
    assert emu.allreduce([_bits([1.0], BF16), nb], "MAX", BF16)[0] == 0x7FC3
    # the logical ops read a NaN as true
    assert emu.allreduce([nan_a, five], "LAND", f32)[0] == 1.0


def test_integers_wrap_in_their_accumulation_type():
    i32, i8, u8, i64 = torch.int32, torch.int8, torch.uint8, torch.int64
    assert emu.allreduce([_bits([2 ** 31 - 1], i32), _bits([1], i32)], "SUM", i32)[0] == -2 ** 31
    assert emu.allreduce([_bits([65536], i32), _bits([65536], i32)], "PROD", i32)[0] == 0
    assert emu.allreduce([_bits([2 ** 63 - 1], i64), _bits([1], i64)], "SUM", i64)[0] == -2 ** 63
    # 8- and 16-bit integers accumulate in 32 bits and wrap in the store
    assert emu.allreduce([_bits([127], i8), _bits([1], i8)], "SUM", i8)[0] == -128
    assert emu.allreduce([_bits([255], u8), _bits([1], u8)], "SUM", u8)[0] == 0
    # ... so a scale sees the unwrapped 32-bit sum: trunc(256 * 0.75) = 192
    assert emu.allreduce([_bits([255], u8), _bits([1], u8)], "SUM", u8, scale=0.75)[0] == 192
    # bool sums count the true ranks; the store maps any non-zero count to true
    b = torch.bool
    assert emu.allreduce([_bits([True], b), _bits([True], b)], "SUM", b, scale=0.75)[0] == 1
    assert emu.allreduce([_bits([True], b), _bits([False], b)], "SUM", b, scale=0.75)[0] == 0


def test_integer_scale_truncates_toward_zero():
    i32 = torch.int32
    assert emu.allreduce([_bits([3], i32), _bits([4], i32)], "SUM", i32, scale=0.75)[0] == 5
    assert emu.allreduce([_bits([-3], i32), _bits([-4], i32)], "SUM", i32, scale=0.75)[0] == -5
    i64 = torch.int64
    # int64 goes through a double: 2^62 + 1 rounds to 2^62 before the scale
    assert emu.allreduce([_bits([2 ** 62 + 1], i64), _bits([0], i64)], "SUM", i64, scale=0.5)[0] == 2 ** 61


def test_fmaf_rounds_once():
    s = np.float32(1 + 2.0 ** -12)
    w = np.float32(-(1 + 2.0 ** -11))
    # s * s = 1 + 2^-11 + 2^-24: rounded on its own the product loses 2^-24 and the sum is 0
    assert np.float32(s * s) + w == 0
    assert emu.fmaf(s, s, w) == np.float32(2.0 ** -24)
    rng = np.random.default_rng(0)
    a, b, c = (rng.standard_normal(10000).astype(np.float32) for _ in range(3))
    exact = a.astype(np.float64) * b + c  # exact here: the three exponents are close
    assert (emu.fmaf(a, b, c) == exact.astype(np.float32)).mean() > 0.99


def test_fused_wgrad_emulation_stages_split_tiles_per_batch_half():
    """Tiles of the last partial wave are staged as two rounded halves, the others as one rounded full-batch tile;
    the owner adds the partials in rank order and applies one fmaf."""
    N, K, Mb, grid = 128, 384, 128, 2  # three tiles on two CTAs: tiles 0 and 1 are a whole wave, tile 2 is split
    g = torch.Generator().manual_seed(0)
    dys = [[torch.randint(-16, 17, (Mb, N), generator=g).to(BF16) for _ in range(2)]]
    xs = [[torch.randint(-16, 17, (Mb, K), generator=g).to(BF16) for _ in range(2)]]
    w = torch.randn(N, K, generator=g).to(BF16)
    scale, gs = -3.1e-4, 0.7
    got, _ = emu.fused_wgrad_sgd(w, dys, xs, scale, gs, 2, grid, prefetch=False)

    def rnd(v):
        return v.float().to(BF16).float()

    a = torch.zeros(N, K)
    for p in range(2):
        dy, x = dys[0][p].double(), xs[0][p].double()
        full = (dy.T @ x).float()
        halves = [(dy[h * 64:(h + 1) * 64].T @ x[h * 64:(h + 1) * 64]).float() for h in range(2)]
        a[:, :256] = a[:, :256] + rnd(full[:, :256] * gs)
        a[:, 256:] = a[:, 256:] + rnd(halves[0][:, 256:] * gs)
        a[:, 256:] = a[:, 256:] + rnd(halves[1][:, 256:] * gs)
    want = torch.from_numpy(emu.fmaf(np.float32(scale), a.numpy(), w.float().numpy())).to(BF16)
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    # the split is visible: staging the split tile as one full-batch partial gives other bits
    whole, _ = emu.fused_wgrad_sgd(w, dys, xs, scale, gs, 1, grid, prefetch=False)
    assert not torch.equal(whole[:, 256:].view(torch.int16), got[:, 256:].view(torch.int16))
    assert torch.equal(whole[:, :256].view(torch.int16), got[:, :256].view(torch.int16))


@pytest.mark.parametrize("nprocs", [2, 3])
def test_emulation_matches_the_host_backend(nprocs, tmp_path):
    res = run_spmd(nprocs, ["tests/spmd/vr_allreduce_steps.py", str(tmp_path)], device="cpu", timeout=600)
    assert res.returncode == 0, f"np={nprocs}\nSTDOUT:\n{res.stdout[-4000:]}\nSTDERR:\n{res.stderr[-8000:]}"
    ranks = [torch.load(tmp_path / f"rank{r}.pt", weights_only=False) for r in range(nprocs)]
    assert len(ranks[0]) > 0
    two_phase_seen = 0
    for recs in zip(*ranks):
        r0 = recs[0]
        dtype, op = r0["dtype"], r0["op"]
        scale = None if r0["variant"] == "none" else r0["scale"]
        acc = emu.bits_of(r0["acc"], dtype) if r0["variant"] == "scale+acc" else None
        want = emu.allreduce([emu.bits_of(x, dtype) for x in r0["xs"]], op, dtype, scale, acc, r0["two_phase"])
        two_phase_seen += r0["two_phase"]
        what = f"{dtype} {op} n={r0['n']} {r0['variant']}"
        for r, rec in enumerate(recs):
            # every rank drew the same inputs for every rank
            for a, b in zip(rec["xs"], r0["xs"]):
                emu.assert_bits(emu.bits_of(a, dtype), emu.bits_of(b, dtype), dtype, what="inputs")
            emu.assert_bits(emu.bits_of(rec["out"], dtype), want, dtype, emu.nan_bits_pinned(dtype, op, scale, acc),
                            what=f"rank {r}: {what}")
    assert two_phase_seen > 0
