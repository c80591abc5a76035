"""The e4m3 GEMM allowance of tests/gemm_e4m3_ref.py on hand-built operands (no GPU): an fp32 emulation of the kernel's
k32 accumulation stays inside it, planted faults leave it, and the e4m3 rounding it assumes is torch.float8_e4m3fn's
with saturation at +-448, subnormals included."""
import math

import pytest
import torch

from gemm_e4m3_ref import E4M3_MAX, check_window, e4m3_window, quantize_rows, reference8, to_e4m3
from gemm_ref import check


def emulate(a8, w8, scale, bias=None, trunc_bits=14):
    """The kernel's arithmetic in fp32: per k32 step the exact products, each added to the accumulator with truncation to
    trunc_bits significant bits, then the scale and the bias."""
    a, w = a8.float(), w8.float()
    acc = torch.zeros(a.shape[0], w.shape[0])
    for j in range(0, a.shape[1], 32):
        for k in range(j, j + 32):
            acc = acc + a[:, k:k + 1] * w[:, k][None, :]
            m, e = torch.frexp(acc)
            acc = torch.ldexp(torch.trunc(m * 2.0 ** trunc_bits) / 2.0 ** trunc_bits, e)
    acc = acc * scale[None, :]
    return acc + bias[None, :] if bias is not None else acc


def operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g, dtype=torch.float64)
    y = (x - x.mean(1, keepdim=True)) / x.std(1, unbiased=False, keepdim=True)      # affine-free LayerNorm rows
    a8 = to_e4m3(y)
    w8, s = quantize_rows(torch.randn(N, K, generator=g) * torch.linspace(0.01, 3.0, N)[:, None])
    return a8, w8, s, torch.randn(N, generator=g)


@pytest.mark.parametrize("M,N,K", [(5, 64, 128), (33, 128, 256), (7, 64, 1024)])
def test_emulation_inside_and_faults_outside(M, N, K):
    a8, w8, s, bias = operands(M, N, K, M + N)
    val, err = reference8(a8, w8, s, M=M, N=N, K=K, bias=bias)
    ratio = check(emulate(a8, w8, s, bias), val, err, "emulation")
    assert ratio <= 0.5, ratio
    with pytest.raises(AssertionError):                      # a dropped k32 step
        bad = emulate(a8[:, :K - 32], w8[:, :K - 32], s, bias)
        check(bad, val, err, "dropped step")
    with pytest.raises(AssertionError):                      # a wrong column's scale
        check(emulate(a8, w8, s.roll(1), bias), val, err, "rolled scale")


def test_rows_at_sqrt_d_minus_1_and_per_channel_scales():
    """The extreme LayerNorm row (one value apart from all others) reaches sqrt(D - 1) and is representable."""
    for D in (128, 768, 1024):
        x = torch.zeros(1, D, dtype=torch.float64)
        x[0, 0] = 1.0
        y = (x - x.mean()) / x.std(unbiased=False)
        assert math.isclose(float(y.abs().max()), math.sqrt(D - 1), rel_tol=1e-12)
        assert float(y.abs().max()) < E4M3_MAX and torch.isfinite(to_e4m3(y).float()).all()
    w = torch.tensor([[1.0, -2.0, 0.5] + [0.0] * 125, [0.0] * 128, [1e-4] * 128])
    w8, s = quantize_rows(w)
    assert s.tolist() == pytest.approx([2.0 / 448, 1.0, 1e-4 / 448])
    assert float(w8[0].float().abs().max()) == 448.0 and float(w8[1].float().abs().max()) == 0.0


def test_rounding_saturation_and_subnormals():
    x = torch.tensor([500.0, -1e9, 448.0, 464.1, 2.0 ** -9, 2.0 ** -10, 3 * 2.0 ** -10, 2.0 ** -6 * 1.0625, 0.0, -0.0])
    got = to_e4m3(x).float()
    assert got.tolist()[:4] == [448.0, -448.0, 448.0, 448.0]
    assert got[4] == 2.0 ** -9 and got[5] == 0.0 and got[6] == 2.0 ** -8          # smallest subnormal, ties to even
    assert got[7] == 2.0 ** -6                                                     # 1.0625 x 2^-6: tie to even
    assert torch.isnan(to_e4m3(torch.tensor([float("nan")])).float()).all()
    lo, hi = e4m3_window(torch.tensor([[1.03]], dtype=torch.float64), torch.tensor([[0.05]], dtype=torch.float64))
    assert float(lo) == 1.0 and float(hi) == 1.125
    assert check_window(to_e4m3(torch.tensor([[1.06]])), torch.tensor([[1.03]], dtype=torch.float64),
                        torch.tensor([[0.05]], dtype=torch.float64)) == 0
    with pytest.raises(AssertionError):
        check_window(to_e4m3(torch.tensor([[1.25]])), torch.tensor([[1.03]], dtype=torch.float64),
                     torch.tensor([[0.05]], dtype=torch.float64))
