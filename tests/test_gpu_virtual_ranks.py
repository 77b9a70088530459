"""The multi-rank kernels bit for bit on one GPU: P virtual ranks are P launches of the unchanged launchers in one
process (csrc/api/virtual_ranks.cpp), each rank with its own zeroed heap, counters and stream.  Covered:

  * the unicast all-reduce kernels (one-shot, two-shot, pipelined two-shot): every dtype x op at P = 2, 3, 5, 8 with
    NaN, +-inf, +-0, subnormals and integer wrap edges; scale, accumulate and in-place epilogues; ragged sizes,
    empty shard tails, several chunks with a ragged last one, operands 2, 4, 8 and 12 bytes off alignment, and calls of
    different sizes back to back (staging parity);
  * the peer-store fused wgrad -> reduce-scatter -> SGD kernel at P = 2, 3: fewer tiles than CTAs, one whole wave,
    whole waves plus a split last wave, with and without the device gradient scale and the W_avg prefetch, three
    consecutive calls on the same weights.

Every rank's result must equal the float64 emulation of virtual_ranks_emulation.py, which rounds where the kernels
round (checked against the host backend in test_virtual_ranks_emulator_cpu.py).  This checks the index arithmetic,
the flag protocol between ranks, the chunking and the epilogues; not the memory model across real NVLink peers."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import virtual_ranks_emulation as emu
from conftest import ROOT

pytestmark = pytest.mark.gpu

RANKS = (2, 3, 5, 8)
VARIANTS = ("none", "scale", "acc", "scale+acc", "inplace")
NO_CHUNKS = 1 << 40  # chunk_bytes above every message: one chunk, the plain two-shot kernel


def _C():
    import mpi4torch_b200 as m4t

    return m4t._C


def _es(dtype):
    return torch.empty(0, dtype=dtype).element_size()


def _scale(dtype):
    # not a power of two, so fl32(scale) and the double differ; positive, so unsigned accumulators stay in range
    return 0.3 if dtype.is_floating_point else 0.75


class _Operand:
    """One operand of a call on every rank: rank p's view of n elements starts `off` bytes past a 256-byte-aligned
    row of one device buffer whose other bytes hold `fill`.  One copy in, one copy out."""

    def __init__(self, values, dtype, off, fill):
        n, es = values[0].numel(), _es(dtype)
        self.dtype, self.off, self.nbytes = dtype, off, n * es
        self.stride = (off + n * es + 64 + 255) // 256 * 256
        host = np.full((len(values), self.stride), fill, dtype=np.uint8)
        for p, v in enumerate(values):
            host[p, off:off + n * es] = emu.bits_of(v, dtype).view(np.uint8)
        self.host = host
        self.raw = torch.from_numpy(host).cuda()
        self.views = [self.raw[p, off:off + n * es].view(dtype) for p in range(len(values))]

    def read(self):
        """(storage arrays of every rank, bytes outside the views unchanged)."""
        raw = self.raw.cpu().numpy()
        outside = np.ones(self.stride, dtype=bool)
        outside[self.off:self.off + self.nbytes] = False
        kept = (raw[:, outside] == self.host[:, outside]).all()
        return [raw[p, self.off:self.off + self.nbytes].view(emu.storage_type(self.dtype)) for p in range(raw.shape[0])], kept


def run_and_check(P, algo, dtype, op, calls, blocks=None, chunk_bytes=NO_CHUNKS, offsets=(0, 0, 0), seed=0):
    """calls: list of (n, variant).  All calls run back to back on the same virtual ranks; then every rank's output
    must equal the emulation, the inputs must be unchanged, and no byte around an operand may be written."""
    C = _C()
    blocks = C.vr_sm_count(P) if blocks is None else blocks
    g = np.random.default_rng(seed)
    ins, outs, accs, scales, checks = [], [], [], [], []
    for n, variant in calls:
        xs = [emu.make_input(dtype, n, g, rank=p) for p in range(P)]
        acc = emu.make_input(dtype, n, g, rank=P)
        scale = _scale(dtype) if "scale" in variant or variant == "inplace" else None
        x = _Operand(xs, dtype, offsets[0], 0x5A)
        if variant == "inplace":
            o = _Operand([acc] * P, dtype, offsets[1], 0xA5)
            a = o
        else:
            o = _Operand([torch.zeros(n, dtype=dtype)] * P, dtype, offsets[1], 0xA5)
            a = _Operand([acc] * P, dtype, offsets[2], 0x3C) if "acc" in variant else None
        ins.append(x.views)
        outs.append(o.views)
        accs.append(a.views if a is not None else [])
        scales.append(scale)
        acc_bits = emu.bits_of(acc, dtype) if a is not None else None
        want = emu.allreduce([emu.bits_of(v, dtype) for v in xs], op, dtype, scale, acc_bits, two_phase=algo == "twoshot")
        checks.append((n, variant, x, o, a if a is not o else None, want, emu.nan_bits_pinned(dtype, op, scale, acc_bits)))
    C.vr_allreduce(ins, outs, emu.OPS[op], algo, blocks, chunk_bytes, scales, accs)
    for n, variant, x, o, a, want, exact_nan in checks:
        what = f"P={P} {algo} {dtype} {op} n={n} {variant}"
        got, kept = o.read()
        assert kept, f"{what}: a store outside the output"
        for p in range(P):
            emu.assert_bits(got[p], want, dtype, exact_nan, what=f"{what} rank {p}")
        for operand in (x, a):
            if operand is not None:
                vals, kept = operand.read()
                assert kept and all((v.view(np.uint8) == operand.host[p, operand.off:operand.off + operand.nbytes]).all()
                                    for p, v in enumerate(vals)), f"{what}: an input was written"


def _table_calls(P, dtype):
    """Sizes at the vector, shard and rank edges: 1, 7, 8, 8P +- 1 elements, a vector count P + 2 (the last shards
    of a chunk are empty), and 65537; the epilogue variants rotate over the sizes, so every variant runs at every
    P at a different size."""
    epv = 16 // _es(dtype)
    sizes = [1, 7, 8, 8 * P - 1, 8 * P + 1, epv * (P + 1) + 1, 65537]
    return [(n, VARIANTS[(i + P) % len(VARIANTS)]) for i, n in enumerate(sizes)]


@pytest.mark.parametrize("P", RANKS)
@pytest.mark.parametrize("algo", ["oneshot", "twoshot"])
@pytest.mark.parametrize("dtype,op", [(d, o) for d in emu.ALL_DTYPES for o in emu.ops_for(d)],
                         ids=lambda v: str(v).replace("torch.", ""))
def test_allreduce_element_table_and_epilogue(P, algo, dtype, op):
    run_and_check(P, algo, dtype, op, _table_calls(P, dtype), seed=P * 1000 + emu.OPS[op])


@pytest.mark.parametrize("P", RANKS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float64, torch.int32, torch.uint8],
                         ids=str)
@pytest.mark.parametrize("op", ["SUM", "MAX"])
def test_pipelined_allreduce_chunks(P, dtype, op):
    """chunk_bytes below the message selects the role-split pipelined kernel.  Chunks of 24 vectors per shard (one
    CTA, five chunks) and of 1100 (three CTAs, two chunks); last chunks of 1 vector (one non-empty shard), P + 1
    vectors and a chunk less one."""
    epv = 16 // _es(dtype)
    for shard, blocks, k in ((24, 2, 5), (1100, None, 2)):
        cv = shard * P
        calls = [(epv * (k * cv + r) - 1, VARIANTS[i % len(VARIANTS)]) for i, r in enumerate((1, P + 1, cv - 1))]
        calls.append((epv * (k * cv + 1), "scale+acc"))
        run_and_check(P, "twoshot", dtype, op, calls, blocks=blocks, chunk_bytes=16 * cv, seed=shard + P)


def _misaligned(dtype):
    """(in, out, acc) byte offsets from 16-byte alignment that the dtype allows: 2, 4, 12 (8 for 8-byte types)."""
    offs = [o for o in (2, 4, 12) if o % _es(dtype) == 0] or [8]
    return [tuple(offs[(i + j) % len(offs)] for j in range(3)) for i in range(len(offs))] + [(0, offs[-1], 0)]


@pytest.mark.parametrize("P", [3, 5])
@pytest.mark.parametrize("kernel", ["oneshot", "twoshot", "pipelined"])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.bfloat16, torch.float16, torch.float32, torch.int32,
                                   torch.float64, torch.int64], ids=str)
def test_allreduce_on_misaligned_views(P, kernel, dtype):
    """Operands off 16-byte alignment take the scalar load_private / store_private path of every kernel."""
    algo = "oneshot" if kernel == "oneshot" else "twoshot"
    chunk = 16 * P * 300 if kernel == "pipelined" else NO_CHUNKS
    for offsets in _misaligned(dtype):
        calls = [(65537, "scale+acc"), (8 * P + 1, "acc"), (20001, "inplace")]
        run_and_check(P, algo, dtype, "SUM", calls, chunk_bytes=chunk, offsets=offsets, seed=sum(offsets) + P)


def test_plain_twoshot_chunk_loop_without_the_pipelined_kernel():
    """M4T_AR_PIPE=0 (read once per process) keeps the plain two-shot kernel for multi-chunk messages: its own chunk
    loop, with a ragged last chunk, in a fresh process."""
    code = (
        "import torch, mpi4torch_b200, test_gpu_virtual_ranks as t\n"
        "for P in (2, 3, 8):\n"
        "    for dt in (torch.bfloat16, torch.float32, torch.int64):\n"
        "        t.run_and_check(P, 'twoshot', dt, 'SUM', [(9001, 'scale+acc'), (40003, 'acc'), (777, 'none')],\n"
        "                        chunk_bytes=16 * P * 37, seed=P)\n"
        "print('plain two-shot chunks ok')\n")
    env = dict(os.environ, M4T_AR_PIPE="0")
    env["PYTHONPATH"] = os.pathsep.join([str(ROOT), str(ROOT / "tests"), env.get("PYTHONPATH", "")])
    res = subprocess.run([sys.executable, "-c", code], env=env, cwd=str(ROOT), capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0 and "plain two-shot chunks ok" in res.stdout, res.stdout[-3000:] + res.stderr[-6000:]


# ---------------------------------------------------------------------------------------------------------------
# fused wgrad -> reduce-scatter -> SGD, peer-store mode
# ---------------------------------------------------------------------------------------------------------------
CALLS = 3


def _wgrad_shape(kind, grid):
    """(N, K) of 128 x 128 tiles: fewer tiles than the grid, exactly one wave, or a whole wave plus 12 split tiles
    of the last wave."""
    if kind == "few":
        return 256, 256
    if kind == "one_wave":
        return 256, 128 * (grid // 2)
    return 256, 128 * (grid // 2 + 6)


@pytest.mark.parametrize("P", [2, 3])
@pytest.mark.parametrize("kind,ksplit", [("few", 2), ("one_wave", 2), ("split_wave", 2), ("split_wave", 1)])
@pytest.mark.parametrize("gscale,prefetch", [(None, True), (0.7, False)])
def test_fused_wgrad_sgd(P, kind, ksplit, gscale, prefetch):
    C = _C()
    grid = C.vr_sm_count(P)
    N, K = _wgrad_shape(kind, grid)
    Mb = 128 if ksplit == 2 else 192  # batch halves of one 64-row k-block; three k-blocks unsplit
    g = torch.Generator().manual_seed(P * 100 + N + K + Mb)
    # integers in [-16, 16]: every per-half G is exact in fp32 whatever the tensor cores' order, but most are not
    # exact in bf16, so the staging rounding, the rank-order sum and the fmaf all show in the bits
    dys = [[torch.randint(-16, 17, (Mb, N), generator=g).to(torch.bfloat16) for _ in range(P)] for _ in range(CALLS)]
    xs = [[torch.randint(-16, 17, (Mb, K), generator=g).to(torch.bfloat16) for _ in range(P)] for _ in range(CALLS)]
    w = torch.randn(N, K, generator=g).to(torch.bfloat16)
    scale = -6e-4  # a sum of P * Mb products of up to 256 moves W by about its own size
    gs_dev = torch.tensor([gscale], dtype=torch.float32, device="cuda") if gscale is not None else None
    res = C.vr_fused_wgrad_sgd([w.cuda() for _ in range(P)], [[t.cuda() for t in c] for c in dys],
                               [[t.cuda() for t in c] for c in xs], scale, gs_dev, ksplit, prefetch)
    assert res["grid"] == grid
    want_w, want_avg = emu.fused_wgrad_sgd(w, dys, xs, scale, gscale, ksplit, grid, prefetch)
    for p in range(P):
        emu.assert_bits(emu.bits_of(res["weights"][p], torch.bfloat16), emu.bits_of(want_w, torch.bfloat16),
                        torch.bfloat16, what=f"P={P} {kind} weights of rank {p}")
        if prefetch:
            emu.assert_bits(emu.bits_of(res["wavg"][p], torch.bfloat16), emu.bits_of(want_avg, torch.bfloat16),
                            torch.bfloat16, what=f"P={P} {kind} W_avg of rank {p}")
    assert res["wavg"] is None or prefetch
    # monotone counters: the owner's tile counter holds every call's signals, 8 per unit and rank; the device epoch
    # word counts the calls
    num_tiles = (N // 128) * (K // 128)
    whole, split, _ = emu.make_sched(num_tiles, grid, ksplit)
    parts = np.where(np.arange(num_tiles) < whole, 1, split)
    assert res["epochs"] == [CALLS] * P
    for p in range(P):
        owned = np.arange(num_tiles) % P == p
        want = np.where(owned, CALLS * 8 * P * parts, 0)
        assert (res["counters"][p].cpu().numpy() == want).all(), f"tile counters of rank {p}"
