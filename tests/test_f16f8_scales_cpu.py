"""CPU: the F16F8 format's oracle (oracle/quant.py) at fp16 scales s != 1 -- known answers for quantize / dequantize at
s = 2^-4 and 2^3, including an fp16 plane that saturates together with its residual -- and the calibration rule
activation_scales at and around its two thresholds (2^14: s leaves 1; 60000: the calibration's fp16 retry)."""
import numpy as np
import pytest
import torch

from oracle import quant


def e4m3(v):
    return float(torch.tensor(v, dtype=torch.float32).clamp(-448, 448).to(torch.float8_e4m3fn).float())


@pytest.mark.parametrize("s", [2.0 ** -4, 2.0 ** 3])
def test_quantize_known_answers_at_fp16_scale(s):
    t = 2.0 ** -2
    big = 65504.0 / s * 4.0                      # a s = 4 * 65504: the fp16 plane saturates, and so does the residual copy
    x = torch.tensor([[0.0, 1.0, -3.0, 0.1, 1000.0, big, -big, 2.0 ** -20] + [0.0] * 56], dtype=torch.float32)
    h, cross, (hd, v8, r8) = quant.quantize(x, s, t)
    want_h = [0.0, s, -3.0 * s, float(np.float16(np.float32(0.1) * np.float32(s))), float(np.float16(1000.0 * s)), 65504.0,
              -65504.0, float(np.float16(2.0 ** -20 * s))]
    np.testing.assert_array_equal(h[0, :8].double().numpy(), want_h)
    np.testing.assert_array_equal(hd[0, :8].numpy(), np.array(want_h) / s)
    # value copy: e4m3(a t), independent of s
    np.testing.assert_array_equal((v8[0, :8] * t).numpy(), [e4m3(float(v) * t) for v in x[0, :8]])
    # residual copy: e4m3((a s - h) 2^11 t / s); zero where a s is exact in fp16, +-448 where h saturated
    for i in range(8):
        r = np.float32(np.float32(x[0, i]) * np.float32(s)) - np.float32(want_h[i])
        assert r8[0, i].item() * 2048.0 * t == e4m3(float(r) * 2048.0 * t / s), i
    assert r8[0, 1].item() == r8[0, 2].item() == 0.0
    assert r8[0, 5].item() * 2048.0 * t == 448.0 and r8[0, 6].item() * 2048.0 * t == -448.0
    # dequantize: (h / s + residual, value copy); exact to e4m3 accuracy of the residual where nothing saturated
    full, copy = quant.dequantize(h, cross, s, t)
    np.testing.assert_array_equal(copy[0, :8].numpy(), v8[0, :8].numpy())
    np.testing.assert_array_equal(full[0, :8].numpy(), (hd + r8)[0, :8].numpy())
    ok = [0, 1, 2, 3, 4]
    rel = (full[0, ok] - x[0, ok].double()).abs() / x[0, ok].double().abs().clamp_min(1e-30)
    assert float(rel.max()) < 2.0 ** -14
    # saturated h and residual: the element is carried as 65504 / s + 448 / (2^11 t), far from a
    assert full[0, 5].item() == 65504.0 / s + 448.0 / (2048.0 * t)


def test_quantize_scales_the_fp16_plane_only():
    """h(2^k s) = 2^k h(s) and both e4m3 copies unchanged, wherever fp16 stays normal and unsaturated."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 5, 128, generator=g) * 40.0
    h0, c0, _ = quant.quantize(x, 1.0, 2.0 ** -3)
    for k in (-4, 3):
        h1, c1, _ = quant.quantize(x, 2.0 ** k, 2.0 ** -3)
        normal = (h0.float().abs() >= 2.0 ** -14) & (h1.float().abs() >= 2.0 ** -14) & (h1.float().abs() < 65504)
        assert torch.equal(h1.double()[normal], h0.double()[normal] * 2.0 ** k)
        assert torch.equal(c1, c0)


def test_activation_scales_around_two_to_the_fourteen():
    # t: 448 / 2^14 = 2^-5.19 -> 2^-6, two binades of headroom -> 2^-8
    assert quant.activation_scales(16384.0) == (1.0, 2.0 ** -8)
    assert quant.activation_scales(np.nextafter(16384.0, 0.0)) == (1.0, 2.0 ** -8)
    assert quant.activation_scales(np.nextafter(16384.0, np.inf)) == (0.5, 2.0 ** -8)
    assert quant.activation_scales(32768.0) == (0.5, 2.0 ** -9)
    # the calibration's fp16 retry range: amax >= 60000 gives s <= 1/4, so the plane keeps amax s < 2^14
    for amax in (59999.0, 60000.0, 65504.0, 1e6, 2.0 ** 60):
        s, t = quant.activation_scales(amax)
        assert 8192.0 < amax * s <= 16384.0 and 448.0 / 8 < amax * t <= 448.0 / 4
    assert quant.activation_scales(60000.0)[0] == 0.25
    # small maxima keep s = 1: the rule only ever shrinks the fp16 plane
    for amax in (2.0 ** -20, 1e-3, 1.0, 4.0):
        assert quant.activation_scales(amax)[0] == 1.0
