"""The checking helpers of test_gpu_exact_arithmetic.py, on the CPU: the GELU and GELU-gradient bounds accept
torch's own fp32 tanh-GELU, and are tight enough to reject erf-GELU and a bf16 store that truncates.  The
bitwise helpers tell round-to-nearest-even from truncation and ties-away."""
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
