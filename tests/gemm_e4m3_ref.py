"""Float64 reference and element-wise allowance of the e4m3 GEMM (m3r_gemm_e4m3 / m3r_gemm_grouped_e4m3) and of the e4m3
LayerNorm outputs (m3r_normalize8, norm_out with norm_e4m3), on top of tests/gemm_ref.py.

Operands: A and W are float8_e4m3fn values, exact in float64; each product of two e4m3 values (4-bit significands) is
exact in fp32.  The kernel accumulates k32 steps (wgmma m64nNk32.f32.e4m3.e4m3).  Hopper's FP8 tensor-core adder keeps
fewer accumulator bits than its 16-bit path (about 14, as published for DeepSeek-V3's FP8 training), so the allowance
charges every one of the 33 additions of a k32 step a truncation of 2^-13 of the value being truncated:
    E_acc = 33 * 2^-13 * (sum_j |P_{j-1}| + sum_k |a_k w_k|)
The per-column scale is one fp32 product, E' = s E + U |v s|; bias, RoPE, GELU and residual follow gemm_ref.py.

e4m3 stores: round to nearest even, as torch.float8_e4m3fn rounds, saturating at +-448.  A value y computed within E in
fp32 is stored as one of the e4m3 values between round(y - E) and round(y + E) (rounding is monotone); e4m3_window()
gives that interval."""
import torch

from gemm_ref import U32, _add, gelu_apply, rope_apply

U_ACC8 = 2.0 ** -13
C_ACC8 = 33.0
E4M3_MAX = 448.0


def to_e4m3(x):
    """torch.float8_e4m3fn rounding with the kernel's saturation at +-448 (NaN stays NaN)."""
    return x.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def quantize_rows(w):
    """The model's weight quantisation (must3r_b200.model.common.quantize_e4m3_rows)."""
    from must3r_b200.model.common import quantize_e4m3_rows
    return quantize_e4m3_rows(w)


def acc_bound8(a, w):
    """Exact a w^T ([r, K] x [N, K] float64 of e4m3 values) and the allowance of the kernel's k32 accumulation."""
    K = a.shape[1]
    p = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float64, device=a.device)
    s = torch.zeros_like(p)
    for j in range(0, K, 32):
        s += p.abs()
        p += a[:, j:j + 32] @ w[:, j:j + 32].t()
    return p, C_ACC8 * U_ACC8 * (s + a.abs() @ w.abs().t())


def reference8(a8, w8, scale, *, M, N, K, groups=1, w_group_rows=0, bias=None, bias_group=0, act=0, residual=None,
               rope_tab=None, rope_cols=0, rope_period=1):
    """(value, allowance before the final store) of the e4m3 GEMM: a8 [groups * M, >= K], w8 [rows, >= K] e4m3,
    scale [rows] fp32 indexed by W row."""
    val = torch.empty(groups * M, N, dtype=torch.float64, device=a8.device)
    err = torch.empty_like(val)
    rows = torch.arange(M, device=a8.device)
    for g in range(groups):
        wr = slice(g * w_group_rows, g * w_group_rows + N)
        v, e = acc_bound8(a8[g * M:(g + 1) * M, :K].double(), w8[wr, :K].double())
        sc = scale[wr].double()
        v = v * sc
        e = e * sc.abs() + U32 * (v.abs() + e * sc.abs())
        if bias is not None:
            v, e = _add(v, e, bias[g * bias_group:g * bias_group + N].double())
        if rope_tab is not None and rope_cols > 0:
            v, e = rope_apply(v, e, rope_tab, rows, rope_cols, max(rope_period, 1))
        if act == 1:
            v, e = gelu_apply(v, e)
        if residual is not None:
            v, e = _add(v, e, residual[:M, :N].double())
        val[g * M:(g + 1) * M], err[g * M:(g + 1) * M] = v, e
    return val, err


def e4m3_window(val, err):
    """The e4m3 values a store of a value within err of val may produce: [lo, hi] as float64."""
    return to_e4m3(val - err).double(), to_e4m3(val + err).double()


def check_window(out8, val, err, what=""):
    """Every e4m3 output lies in its window; returns the number of elements not equal to the rounding of val."""
    o = out8.double()
    lo, hi = e4m3_window(val, err)
    bad = ~((o >= lo) & (o <= hi))
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        r, c = divmod(i, out8.shape[1])
        raise AssertionError(f"{what}: row {r} column {c}: got {float(o[r, c])}, window [{float(lo[r, c])}, "
                             f"{float(hi[r, c])}] around {float(val[r, c]):.7g} ({int(bad.sum())} elements outside)")
    return int((o != to_e4m3(val).double()).sum())
