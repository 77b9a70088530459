"""The fp8 recipe of ``dp_linear_mse(..., fp8=True)`` on the CPU (DESIGN §4.4).

* ``fp8_scale`` and ``quantize_fp8_reference`` against an independent numpy implementation of the scale rule and of
  round-to-nearest-even with saturation.
* The composition node's loss and gradients against a float64 emulation, with an upstream gradient g != 1, a frozen
  weight and ``x.grad``.
* The refusals: ``accumulator=``, ``train_step(micro_batches > 1)``, and ``InBackwardSGD`` off the kernel path.
"""
import math

import numpy as np
import pytest
import torch

import mpi4torch_b200 as m4t
from mpi4torch_b200.models import DPLinearModel
from mpi4torch_b200.ops import AccumulatedSGD, InBackwardSGD, dp_linear_mse
from mpi4torch_b200.ops.fp8 import E4M3, E5M2, FORMATS, fp8_scale, quantize_fp8_reference

# format -> (mantissa bits, smallest normal exponent, largest finite value)
NP_FMT = {E4M3: (3, -6, 448.0), E5M2: (2, -14, 57344.0)}


def np_scale(amax, fmt):
    """(s, 1/s) by search: the largest power of two with amax * s <= F, exponent clamped to [-126, 126]."""
    F = NP_FMT[fmt][2]
    if not math.isfinite(amax):
        return 1.0, math.nan
    if amax == 0.0:
        return 1.0, 1.0
    e = 0
    while amax * 2.0 ** e > F:
        e -= 1
    while amax * 2.0 ** (e + 1) <= F:
        e += 1
    e = max(-126, min(126, e))
    return 2.0 ** e, 2.0 ** -e


def np_round_fp8(v, fmt):
    """Round float64 values to the fp8 grid, nearest even, saturating at +-F (NaN stays NaN)."""
    mbits, emin, F = NP_FMT[fmt]
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(v)
    _, ex = np.frexp(np.where(np.isfinite(a) & (a > 0), a, 1.0))
    q = np.ldexp(1.0, np.maximum(ex - 1, emin) - mbits)  # the grid spacing of a's binade
    r = np.minimum(np.round(a / q) * q, F)  # np.round: half to even
    return np.where(np.isnan(v), np.nan, np.copysign(r, v))


def np_quantize(x, fmt):
    """(dequantized values, 1/s) of the recipe; the operand is taken in fp32."""
    xf = np.asarray(x, dtype=np.float32).astype(np.float64)
    s, inv = np_scale(float(np.max(np.abs(xf))), fmt)
    return np_round_fp8(xf * s, fmt) * inv, inv


def _amax_cases():
    out = [0.0, 448.0, 57344.0, 1.0]
    for k in list(range(-149, 128, 7)) + [-126, -127, -130, 0, 8, 9, 15, 16, 127]:
        p = 2.0 ** k
        out += [p, float(np.nextafter(np.float32(p), np.float32(np.inf))), 0.875 * p,
                float(np.nextafter(np.float32(0.875 * p), np.float32(np.inf)))]
    return [a for a in out if np.isfinite(np.float32(a)) and a == float(np.float32(a))]


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
def test_scale_rule(fmt):
    for a in _amax_cases():
        s, inv = fp8_scale(torch.tensor([a], dtype=torch.float32), fmt)
        ws, winv = np_scale(a, fmt)
        assert float(s) == ws and float(inv) == winv, (fmt, a, float(s), ws)


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf")])
def test_non_finite_gives_nan_scale(fmt, bad):
    x = torch.randn(8, 16)
    x[3, 5] = bad
    _, inv = quantize_fp8_reference(x, fmt)
    assert math.isnan(float(inv))


def _check_quantize(x, fmt):
    q, inv = quantize_fp8_reference(x, fmt)
    assert q.dtype == FORMATS[fmt][0]
    want, winv = np_quantize(x.numpy(), fmt)
    assert float(inv) == winv
    got = q.double().numpy() * float(inv)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
def test_quantize_random_magnitudes(fmt):
    g = torch.Generator().manual_seed(3)
    for scale in (1e-6, 1e-2, 1.0, 3.0, 1e3, 1e5):
        x = torch.randn(37, 53, generator=g) * scale
        x[0, 0] = scale * 2.0 ** torch.randint(-20, 4, (1,), generator=g).item()  # amax at a power of two, sometimes
        _check_quantize(x, fmt)


@pytest.mark.parametrize("fmt", [E4M3, E5M2])
def test_quantize_edges(fmt):
    mbits, emin, F = NP_FMT[fmt]
    sub = 2.0 ** (emin - mbits)  # smallest subnormal of the format
    top = 2.0 ** (math.floor(math.log2(F)) - mbits)  # grid spacing just below F
    vals = [F,  # amax: s = 1
            F - top / 4, F - top / 2, F - 3 * top / 4,  # round up to F, tie to even (F), round down
            -(F - top / 2),
            sub, 1.5 * sub, 2.5 * sub, 0.5 * sub, 0.25 * sub, 0.75 * sub, 3 * sub,  # subnormal results and ties
            2.0 ** emin, 2.0 ** emin * (1 - 2.0 ** -(mbits + 2)),  # smallest normal, just below it
            0.0, -0.0]
    _check_quantize(torch.tensor(vals, dtype=torch.float32).reshape(1, -1), fmt)
    # the same values under a non-unit scale: amax = F * 2^-10 gives s = 2^10
    _check_quantize(torch.tensor(vals, dtype=torch.float32).reshape(1, -1) * 2.0 ** -10, fmt)


def test_amax_zero():
    for fmt in (E4M3, E5M2):
        q, inv = quantize_fp8_reference(torch.zeros(4, 8), fmt)
        assert float(inv) == 1.0 and not bool(q.float().any())


# ---- the composition node -------------------------------------------------------------------------------------------
B, D, O = 24, 20, 12


def _case(seed):
    g = torch.Generator().manual_seed(seed)
    # fp32-representable float64 values: the recipe takes its operands in fp32
    x = torch.randn(B, D, generator=g).double()
    w = (torch.randn(O, D, generator=g) * D ** -0.5).double()
    t = torch.randn(B, O, generator=g).double()
    return x, w, t


def emulate(x, w, t, loss_scale, g):
    """float64 numpy: (loss, dL/dx, dL/dW) of g * loss under the recipe, at one rank."""
    x, w, t = x.numpy(), w.numpy(), t.numpy()
    xd, _ = np_quantize(x, E4M3)
    wd, _ = np_quantize(w, E4M3)
    d = xd @ wd.T - t
    loss = loss_scale * np.sum(d * d)
    dy = d * (2.0 * loss_scale)
    dyd, _ = np_quantize(dy, E5M2)
    return loss, g * (dy @ w), g * (dyd.T @ xd)


def _close(got, want, what, rel=1e-12):
    got = got.detach().double().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    err = float(np.max(np.abs(got - want)))
    assert err <= rel * float(np.max(np.abs(want))), f"{what}: off by {err}"


@pytest.mark.parametrize("g", [1.0, 3.0, 2.0 ** -5])
@pytest.mark.parametrize("frozen", [False, True])
def test_composition_against_emulation(g, frozen):
    x, w, t = _case(5)
    ls = 1.0 / B
    xr, wr = x.clone().requires_grad_(), w.clone().requires_grad_(not frozen)
    loss = dp_linear_mse(xr, wr, t, m4t.COMM_WORLD, loss_scale=ls, fp8=True)
    (loss * g).sum().backward()
    l_ref, gx_ref, gw_ref = emulate(x, w, t, ls, g)
    _close(loss, l_ref, "loss")
    _close(xr.grad, gx_ref, "x.grad")
    if frozen:
        assert wr.grad is None
    else:
        _close(wr.grad, gw_ref, "W.grad")


def test_fp8_differs_from_bf16_path():
    """The fp8 node really quantizes: its loss is not the unquantized one."""
    x, w, t = _case(6)
    l8 = dp_linear_mse(x, w, t, m4t.COMM_WORLD, loss_scale=1.0, fp8=True)
    l64 = dp_linear_mse(x, w, t, m4t.COMM_WORLD, loss_scale=1.0)
    assert float(l8) != float(l64)
    assert abs(float(l8) - float(l64)) <= 0.1 * float(l64)


def test_nan_input_gives_nan_loss():
    x, w, t = _case(7)
    x[2, 3] = float("inf")
    assert math.isnan(float(dp_linear_mse(x, w, t, m4t.COMM_WORLD, loss_scale=1.0, fp8=True)))


def test_model_trains_and_matches_emulation():
    comm = m4t.COMM_WORLD
    model = DPLinearModel(D, O, comm, device="cpu", dtype=torch.float64, lr=0.1, seed=2, fp8=True)
    x, _, t = _case(8)
    w0 = model.weight.detach().clone()
    losses = [float(model.train_step(x, t)) for _ in range(5)]
    assert losses[-1] < losses[0], losses
    # the first step against the emulation (in-backward SGD is off the kernel path: plain .grad + SGD)
    l_ref, _, gw_ref = emulate(x, w0, t, 1.0 / B, 1.0)
    assert abs(losses[0] - l_ref) <= 1e-12 * l_ref
    fresh = DPLinearModel(D, O, comm, device="cpu", dtype=torch.float64, lr=0.1, seed=2, fp8=True)
    fresh.train_step(x, t)
    _close(fresh.weight, w0.numpy() - 0.1 * gw_ref, "weight after one step")


def test_refusals():
    x, w, t = _case(9)
    comm = m4t.COMM_WORLD
    with pytest.raises(ValueError):
        dp_linear_mse(x, w, t, comm, loss_scale=1.0, fp8=True, accumulator=AccumulatedSGD(0.1))
    model = DPLinearModel(D, O, comm, device="cpu", dtype=torch.float64, fp8=True)
    with pytest.raises(ValueError):
        model.train_step(x.repeat(2, 1)[:2 * (B // 2)], t[:2 * (B // 2)], micro_batches=2)
    with pytest.raises(RuntimeError):
        dp_linear_mse(x, w.requires_grad_(), t, comm, loss_scale=1.0, fp8=True, optimizer=InBackwardSGD(0.1))
