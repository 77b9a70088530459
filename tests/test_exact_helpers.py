"""The checking helpers of test_gpu_exact_arithmetic.py, on the CPU: the GELU and GELU-gradient bounds accept
torch's own fp32 tanh-GELU, and are tight enough to reject erf-GELU and a bf16 store that truncates.  The
bitwise helpers tell round-to-nearest-even from truncation and ties-away.  The MLP node emulation of
test_gpu_mlp_exact.py, with its rounding off, matches torch.autograd of the float64 composition."""
import pytest
import torch
import torch.nn.functional as F

from test_gpu_exact_arithmetic import (assert_same_bits, gelu_dz_violations, gelu_h_violations, quantum, rne_bf16,
                                       trunc_bf16)

Z = torch.arange(-8 * 256, 8 * 256 + 1, dtype=torch.float64) / 256  # every z on a 2^-8 grid in [-8, 8]


def _truncate(v32):
    return (v32.view(torch.int32) & -65536).view(torch.float32).to(torch.bfloat16)


def test_gelu_bound_accepts_fp32_tanh_gelu_and_rejects_erf_and_truncation():
    h32 = F.gelu(Z.float(), approximate="tanh")
    assert not bool(gelu_h_violations(h32.to(torch.bfloat16), Z).any())
    assert bool(gelu_h_violations(F.gelu(Z.float()).to(torch.bfloat16), Z).any()), "erf-GELU passed"
    assert bool(gelu_h_violations(_truncate(h32), Z).any()), "a truncated h passed"


def test_gelu_grad_bound_accepts_fp32_backward_and_rejects_erf_and_truncation():
    for a in (1.0, -37.0, 1000.0, 2.0 ** -9):
        upstream = torch.full_like(Z, a)
        z = Z.float().requires_grad_()
        F.gelu(z, approximate="tanh").backward(upstream.float())
        dz32 = z.grad
        assert not bool(gelu_dz_violations(dz32.to(torch.bfloat16), upstream, Z).any()), a
        z = Z.float().requires_grad_()
        F.gelu(z).backward(upstream.float())
        assert bool(gelu_dz_violations(z.grad.to(torch.bfloat16), upstream, Z).any()), f"erf-GELU gradient passed ({a})"
        assert bool(gelu_dz_violations(_truncate(dz32), upstream, Z).any()), f"a truncated dz passed ({a})"


def test_bitwise_helpers():
    v = torch.tensor([257.0, 258.0, 259.0, 261.0, -259.0, 1.0 + 2.0 ** -20, 0.0], dtype=torch.float64)
    # 257 and 259 are ties (bf16 has 8 significant bits): to even, 256 and 260; truncation gives 256 and 258
    assert rne_bf16(v).double().tolist() == [256.0, 258.0, 260.0, 260.0, -260.0, 1.0, 0.0]
    assert trunc_bf16(v).double().tolist() == [256.0, 258.0, 258.0, 260.0, -258.0, 1.0, 0.0]
    assert_same_bits(rne_bf16(v), rne_bf16(v), "self")
    for wrong in (trunc_bf16(v), (v + torch.sign(v) * 0.5).float().to(torch.bfloat16)):  # truncation, ties away
        try:
            assert_same_bits(wrong, rne_bf16(v), "wrong rounding")
        except AssertionError:
            continue
        raise AssertionError("a wrong rounding compared equal")
    nan = torch.tensor([float("nan"), 1.0])
    assert_same_bits(nan, nan.clone(), "NaN in place")
    try:
        assert_same_bits(torch.tensor([1.0, float("nan")]), nan, "NaN moved")
    except AssertionError:
        pass
    else:
        raise AssertionError("a moved NaN compared equal")
    assert quantum(torch.tensor([3.0 * 2 ** -5, 2.0 ** -3, 0.0, float("inf")])) == 2.0 ** -5
    assert quantum(torch.zeros(3)) == 1.0


# ------------------------------------------------------------------------------------------------------------------
# The float64 emulation of the MLP node in test_gpu_mlp_exact.py, with its rounding off, against torch.autograd
# ------------------------------------------------------------------------------------------------------------------
def _mlp_case(loss, seed):
    from test_gpu_exact_arithmetic import _gen
    from test_gpu_mlp_exact import mse_case, xent_case

    gen = _gen(64, 128, 256, seed, device="cpu")
    if loss == "mse":
        return mse_case(64, 128, 256, 128, gen)
    return xent_case(64, 128, 256, gen, ignore_index=3)


def _composition_grads(x, w1, b1, w2, b2, last, g, loss_fn):
    ins = [t.clone().requires_grad_() for t in (x, w1, b1, w2, b2)]
    y = F.linear(F.gelu(F.linear(ins[0], ins[1], ins[2]), approximate="tanh"), ins[3], ins[4])
    loss = loss_fn(y, last).reshape(1)
    grads = torch.autograd.grad(loss, ins, grad_outputs=torch.full((1,), g, dtype=torch.float64))
    return loss.detach(), grads


def _check_emulator(loss_kind, g, library):
    """The emulator without rounding equals autograd of F.linear -> F.gelu(tanh) -> F.linear -> loss in float64,
    either composed here or as the library's fallback (dp_mlp_mse / dp_mlp_cross_entropy on CPU tensors)."""
    from test_gpu_mlp_exact import emulate_node

    x, w1, b1, w2, b2, last = _mlp_case(loss_kind, 1 + int(g))
    ls = 2.0 ** -3
    if loss_kind == "mse":
        e = emulate_node(x, w1, b1, w2, b2, ls=ls, g=g, target=last, rnd=lambda v: v)
        fn = lambda y, t: (y - t).square().sum() * ls  # noqa: E731
    else:
        e = emulate_node(x, w1, b1, w2, b2, ls=ls, g=g, labels=last, ignore_index=3, rnd=lambda v: v)
        fn = lambda y, lab: F.cross_entropy(y, lab, reduction="sum", ignore_index=3) * ls  # noqa: E731
    if library:
        from mpi4torch_b200.ops import dp_mlp_cross_entropy, dp_mlp_mse

        if loss_kind == "mse":
            fn = lambda y, t: dp_mlp_mse(*y, t, loss_scale=ls)  # noqa: E731
        else:
            fn = lambda y, lab: dp_mlp_cross_entropy(*y, lab, loss_scale=ls, ignore_index=3)  # noqa: E731
        ins = [t.clone().requires_grad_() for t in (x, w1, b1, w2, b2)]
        loss = fn(ins, last).reshape(1)
        grads = torch.autograd.grad(loss, ins, grad_outputs=torch.full((1,), g, dtype=torch.float64))
        loss = loss.detach()
    else:
        loss, grads = _composition_grads(x, w1, b1, w2, b2, last, g, fn)
    want = [e[k] for k in ("gx", "G1", "gb1", "G2", "gb2")]
    assert any(bool((w != 0).any()) for w in want[:3]), "the case has no layer-1 gradient"
    if loss_kind == "mse":  # every value is exact in float64: equal, not close
        assert float(loss) == float(e["loss"])
        for name, got, w in zip(("x", "w1", "b1", "w2", "b2"), grads, want):
            assert torch.equal(got, w), f"grad {name}: {float((got - w).abs().max())}"
    else:  # softmax and log: float64 roundings in different places
        assert abs(float(loss) - float(e["loss"])) <= 1e-12 * abs(float(e["loss"]))
        for name, got, w in zip(("x", "w1", "b1", "w2", "b2"), grads, want):
            torch.testing.assert_close(got, w, rtol=1e-12, atol=1e-15, msg=f"grad {name}")


@pytest.mark.parametrize("library", [False, True], ids=["autograd", "library_fallback"])
@pytest.mark.parametrize("g", [1.0, 3.0])
@pytest.mark.parametrize("loss_kind", ["mse", "cross_entropy"])
def test_mlp_emulator_matches_autograd(loss_kind, g, library):
    _check_emulator(loss_kind, g, library)


def test_mlp_emulator_rounds_where_the_kernels_round():
    """With rounding on, the emulator differs from the unrounded one exactly through bf16 stores: a changed rounding
    function changes its gradients."""
    from test_gpu_mlp_exact import emulate_node

    x, w1, b1, w2, b2, t = _mlp_case("mse", 9)
    rne = emulate_node(x, w1, b1, w2, b2, ls=2.0 ** -3, g=3.0, target=t)
    trunc = emulate_node(x, w1, b1, w2, b2, ls=2.0 ** -3, g=3.0, target=t, rnd=trunc_bf16)
    assert all(bool(((rne[k] - rne[k].to(torch.bfloat16).double()) == 0).all()) for k in ("dy", "dz", "gx", "gw1", "gw2"))
    assert any(not torch.equal(rne[k], trunc[k]) for k in ("dy", "gw1", "gw2", "gx")), "truncation changed nothing"
