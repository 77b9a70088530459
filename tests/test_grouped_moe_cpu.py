"""The dropless mixture-of-experts pieces that run without a GPU: the grouped layout helper against a plain model of
its rule, ``grouped_expert_mlp``'s composition path against float64 autograd, and the dropless layer at one rank under
a skewed router."""
import pytest
import torch
import torch.nn.functional as F

from mpi4torch_b200.ops import expert_group_starts, grouped_expert_mlp, grouped_expert_mlp_supported
from mpi4torch_b200.ops.expert_mlp import grouped_rows


def _model_starts(counts):
    out, s = [], 0
    for c in counts:
        out.append(s)
        s += 128 * ((max(c, 0) + 127) // 128)
    return out


@pytest.mark.parametrize("counts", [[0], [1], [127, 128, 129], [0, 1, 127, 128, 129, 300], [-5, 7, 0, 0, 256],
                                    [1000, 0, 3] * 5])
def test_group_starts_follow_the_layout_rule(counts):
    for dtype in (torch.int32, torch.int64):
        got = expert_group_starts(torch.tensor(counts, dtype=dtype))
        assert got.dtype == torch.int64 and got.tolist() == _model_starts(counts)
    # the groups fit in grouped_rows(pairs, E) rows, and no 128-row block holds two groups
    pairs = sum(max(c, 0) for c in counts)
    ends = [s + max(c, 0) for s, c in zip(_model_starts(counts), counts)]
    assert max(ends) <= grouped_rows(pairs, len(counts))
    assert all(s % 128 == 0 for s in _model_starts(counts))


def _inputs(counts, D, H, O, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)  # noqa: E731
    E = len(counts)
    R = grouped_rows(sum(max(c, 0) for c in counts), E)
    return [r(R, D).to(dtype), (r(E, H, D) / D ** 0.5).to(dtype), r(E, H).to(dtype),
            (r(E, O, H) / H ** 0.5).to(dtype), r(E, O).to(dtype)]


def _reference(counts, ins, dy):
    """Per group, in float64, with F.linear over the group's rows; zero elsewhere."""
    x, w1, b1, w2, b2 = [t.detach().double().requires_grad_() for t in ins]
    pieces, at = [], 0
    for e, (s, c) in enumerate(zip(_model_starts(counts), counts)):
        c = max(c, 0)
        pieces.append(torch.zeros(s - at, w2.shape[1], dtype=torch.float64))
        pieces.append(F.linear(F.gelu(F.linear(x[s:s + c], w1[e], b1[e]), approximate="tanh"), w2[e], b2[e]))
        at = s + c
    pieces.append(torch.zeros(x.shape[0] - at, w2.shape[1], dtype=torch.float64))
    y = torch.cat(pieces)
    y.backward(dy.double())
    return y.detach(), [t.grad for t in (x, w1, b1, w2, b2)]


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-12), (torch.float32, 2e-5), (torch.bfloat16, 2e-2)])
def test_grouped_composition_matches_float64(dtype, tol):
    counts = [5, 0, 130, 1]
    ins = [t.requires_grad_() for t in _inputs(counts, 6, 12, 5, dtype)]
    cnt = torch.tensor(counts, dtype=torch.int32)
    assert not grouped_expert_mlp_supported(ins[0], cnt, *ins[1:])
    dy = torch.randn(ins[0].shape[0], 5, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 3
    y = grouped_expert_mlp(ins[0], cnt, *ins[1:])
    assert y.dtype == dtype and tuple(y.shape) == (ins[0].shape[0], 5)
    y.backward(dy.to(dtype))
    ref_y, ref_grads = _reference(counts, ins, dy.to(dtype))
    for name, got, ref in zip(("y", "x", "w1", "b1", "w2", "b2"), [y] + [t.grad for t in ins], [ref_y] + ref_grads):
        assert got.dtype == dtype, name
        err = float((got.detach().double() - ref).abs().max())
        assert err <= tol * max(1.0, float(ref.abs().max())), f"{dtype} {name}: {err}"
    assert bool((ins[1].grad[1] == 0).all()), "the empty expert got a gradient"


def test_grouped_expert_mlp_rejects_mismatched_shapes():
    x, w1, b1, w2, b2 = _inputs([3, 4], 6, 8, 5, torch.float64)
    cnt = torch.tensor([3, 4], dtype=torch.int32)
    with pytest.raises(ValueError):
        grouped_expert_mlp(x, cnt[:1], w1, b1, w2, b2)
    with pytest.raises(ValueError):
        grouped_expert_mlp(x, cnt.float(), w1, b1, w2, b2)
    with pytest.raises(ValueError):
        grouped_expert_mlp(x[None], cnt, w1, b1, w2, b2)
    assert not grouped_expert_mlp_supported(x, cnt, w1, b1[:, :3], w2, b2)
