"""The mixture-of-experts pieces that run without a GPU: ``expert_mlp``'s composition path against float64 autograd,
a model of the batched kernels' tile schedules, and the MoE example at two ranks."""
import re

import pytest
import torch
import torch.nn.functional as F

from conftest import run_spmd

from mpi4torch_b200.ops import expert_mlp, expert_mlp_supported


def _inputs(E, M, D, H, O, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    return [r(E, M, D).to(dtype), (r(E, H, D) / D ** 0.5).to(dtype), r(E, H).to(dtype), (r(E, O, H) / H ** 0.5).to(dtype),
            r(E, O).to(dtype)]


def _reference(ins, dy):
    """Per expert, in float64, with F.linear: an independent spelling of the same math."""
    x, w1, b1, w2, b2 = [t.detach().double().requires_grad_() for t in ins]
    y = torch.stack([F.linear(F.gelu(F.linear(x[e], w1[e], b1[e]), approximate="tanh"), w2[e], b2[e])
                     for e in range(x.shape[0])])
    y.backward(dy.double())
    return y.detach(), [t.grad for t in (x, w1, b1, w2, b2)]


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 2e-5), (torch.bfloat16, 2e-2)])
def test_composition_matches_float64(dtype, tol):
    E, M, D, H, O = 3, 10, 6, 12, 5
    ins = [t.requires_grad_() for t in _inputs(E, M, D, H, O, dtype)]
    assert not expert_mlp_supported(*ins)
    dy = torch.randn(E, M, O, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 3
    y = expert_mlp(*ins)
    assert y.dtype == dtype and tuple(y.shape) == (E, M, O)
    y.backward(dy.to(dtype))
    ref_y, ref_grads = _reference(ins, dy.to(dtype))
    for name, got, ref in zip(("y", "x", "w1", "b1", "w2", "b2"), [y] + [t.grad for t in ins], [ref_y] + ref_grads):
        assert got.dtype == dtype, name
        err = float((got.detach().double() - ref).abs().max())
        assert err <= tol * max(1.0, float(ref.abs().max())), f"{dtype} {name}: {err}"


@pytest.mark.parametrize("grouped", [False, True])
def test_composition_takes_a_misaligned_upstream_gradient(grouped):
    """An upstream gradient that is contiguous but sits one element into its buffer (a base the kernels could not
    read) gives the gradients of an aligned copy of it."""
    from mpi4torch_b200.ops import grouped_expert_mlp

    E, M, D, H, O = 3, 10, 6, 12, 5
    x, w1, b1, w2, b2 = _inputs(E, M, D, H, O, torch.float64)
    args = (x.reshape(E * M, D), torch.tensor([4, 0, 9], dtype=torch.int32)) if grouped else (x,)
    node = grouped_expert_mlp if grouped else expert_mlp
    grads = []
    for offset in (0, 1):
        ins = [t.clone().requires_grad_() for t in (args[0], w1, b1, w2, b2)]
        y = node(ins[0], *args[1:], *ins[1:])
        dy = torch.randn(y.shape, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
        buf = torch.full((y.numel() + 1,), float("nan"), dtype=torch.float64)
        view = buf[offset:offset + y.numel()].view(y.shape)
        view.copy_(dy)
        assert view.is_contiguous() and view.storage_offset() == offset
        y.backward(view)
        grads.append([t.grad for t in ins])
    for name, got, ref in zip(("x", "w1", "b1", "w2", "b2"), grads[1], grads[0]):
        torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12, msg=name)


def test_expert_mlp_rejects_mismatched_shapes():
    x, w1, b1, w2, b2 = _inputs(2, 4, 6, 8, 5, torch.float64)
    with pytest.raises(ValueError):
        expert_mlp(x, w1, b1, w2[:1], b2)
    with pytest.raises(ValueError):
        expert_mlp(x, w1, b1[:, :3], w2, b2)
    assert not expert_mlp_supported(x, w1, b1, w2[:1], b2)


# ------------------------------------------------------------------------------------------------------------------
# The tile schedules of the batched kernels (gemm_bf16_wgmma_kernel<.., BATCHED>, wgrad_bf16_wgmma_kernel<.., BATCHED>)
# ------------------------------------------------------------------------------------------------------------------
BM, BN, BK = 128, 256, 64


def gemm_tiles(E, M, N, grid):
    """Per CTA, the tiles it computes, as the kernel derives them: (expert, m_blk, n_blk, output rows, output columns,
    B rows)."""
    m_tiles, n_tiles = E * M // BM, -(-N // BN)
    out = []
    for cta in range(grid):
        for t in range(cta, m_tiles * n_tiles, grid):
            n_blk = t // m_tiles
            m_blk = t - n_blk * m_tiles
            expert = m_blk * BM // M
            rows = range(m_blk * BM, m_blk * BM + BM)
            cols = range(n_blk * BN, min(N, n_blk * BN + BN))  # the epilogue stores col < N only
            b_rows = range(expert * N + n_blk * BN, expert * N + min(N, n_blk * BN + BN))
            out.append((expert, m_blk, n_blk, rows, cols, b_rows))
    return out


def wgrad_tiles(E, Mb, N, K, grid):
    """(expert, n_blk, k_blk, output rows of the stacked [E N, K], output columns, contraction rows)."""
    n_tiles, k_tiles = N // BM, -(-K // BN)
    out = []
    for cta in range(grid):
        for t in range(cta, E * n_tiles * k_tiles, grid):
            n_blk = t // k_tiles
            k_blk = t - n_blk * k_tiles
            expert = n_blk // n_tiles
            rows = range(n_blk * BM, n_blk * BM + BM)
            cols = range(k_blk * BN, min(K, k_blk * BN + BN))
            contraction = [expert * Mb + kb * BK + i for kb in range(Mb // BK) for i in range(BK)]
            out.append((expert, n_blk, k_blk, rows, cols, contraction))
    return out


@pytest.mark.parametrize("E,M,N", [(1, 128, 128), (3, 384, 640), (8, 256, 1280), (8, 128, 1408), (5, 1024, 384)])
@pytest.mark.parametrize("sms", [7, 132])
def test_gemm_tile_schedule_covers_each_output_once_within_its_expert(E, M, N, sms):
    tiles = -(-E * M // BM) * -(-N // BN)
    seen = torch.zeros(E * M, N, dtype=torch.int32)
    for expert, m_blk, n_blk, rows, cols, b_rows in gemm_tiles(E, M, N, max(1, min(tiles, sms))):
        assert rows[0] // M == expert and rows[-1] // M == expert, "an M-tile crosses an expert boundary"
        assert b_rows[0] // N == expert and b_rows[-1] // N == expert, "stored columns read another expert's weights"
        seen[rows.start:rows.stop, cols.start:cols.stop] += 1
    assert bool((seen == 1).all()), "an output element is computed twice or never"


@pytest.mark.parametrize("E,Mb,N,K", [(1, 64, 128, 128), (3, 384, 256, 640), (8, 256, 384, 1408), (5, 128, 1024, 256)])
@pytest.mark.parametrize("sms", [7, 132])
def test_wgrad_tile_schedule_covers_each_output_once_within_its_expert(E, Mb, N, K, sms):
    tiles = E * (N // BM) * -(-K // BN)
    seen = torch.zeros(E * N, K, dtype=torch.int32)
    for expert, n_blk, k_blk, rows, cols, contraction in wgrad_tiles(E, Mb, N, K, max(1, min(tiles, sms))):
        assert rows[0] // N == expert and rows[-1] // N == expert, "an output tile crosses an expert boundary"
        assert contraction == list(range(expert * Mb, expert * Mb + Mb)), "the contraction leaves its expert's rows"
        seen[rows.start:rows.stop, cols.start:cols.stop] += 1
    assert bool((seen == 1).all()), "an output element is computed twice or never"


def test_moe_example_loss_decreases_cpu():
    res = run_spmd(2, ["examples/moe_layer.py", "--device", "cpu", "--steps", "20"], device="cpu", timeout=300)
    assert res.returncode == 0, res.stderr[-4000:]
    losses = [float(v) for v in re.findall(r"loss ([0-9.]+)", res.stdout)]
    assert len(losses) == 20 and losses[-1] < losses[0], losses
