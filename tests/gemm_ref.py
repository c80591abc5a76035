"""Float64 reference of m3r_gemm / m3r_gemm_grouped and of the LayerNorm kernels, the element-wise error allowance of
the kernels' arithmetic, and the operand generator that the CPU bound test and the GPU contract test share.

reference() takes the fields of m3r_gemm_args / m3r_gemm_group (A, W, the grouped strides, bias, RoPE table, row bias,
GELU, residual, split-K) on the same 16-bit inputs, computes every output element in float64 on the inputs' device
(chunked over rows), and carries along an fp32 error bound E of the value the epilogue holds before its final store.
layernorm() does the same for a LayerNorm of such values (the emitted norm_out, or m3r_layernorm & co.), out_bound()
adds the rounding of the stored type, check() compares an output with the allowance element by element and names the
first element over it.

Notation: U = 2^-24 (fp32 round-to-nearest unit roundoff; one ulp of a value x is at most 2U |x|), u = 2^-11 (fp16) or
2^-8 (bf16).

Accumulation (the tensor cores, m64nBNk16 wgmma in the kernel's K order; split-K: each half from zero):
  per k16 step 16 exact products (16-bit x 16-bit fits fp32) enter the fp32 accumulator with up to 17 truncations,
  each at most 2^-23 = 2U of the value being truncated, which is at most |P_{j-1}| + sum_{k in block j} |a_k w_k|
  (P_j = the exact prefix sum over the first j k16 blocks).  Truncation is biased towards zero, so the errors add:
      E_acc = 17 * 2U * (sum_j |P_{j-1}| + sum_k |a_k w_k|)                                                     (C_ACC)
  split-K: the same over each half with its own prefix sums, plus U (|P| + E_acc) for the round-to-nearest add of
  the two halves.
Epilogue, fp32 round-to-nearest, in the kernel's order (epilogue_apply), x the value entering an operation and E its
error bound; every rounding is at most U |result| and |result| <= |ref| + E:
  bias, row bias, residual add   E' = E + U (|x'| + E)
  RoPE (u' = u cos - w sin)      E' = |cos| E_u + |sin| E_w + U ((|u| + E_u)|cos| + (|w| + E_w)|sin|) + U (|u'| + ...)
                                 (two products and one add, or an fma; the fp32 table values are exact inputs, or
                                 with rope_tab_err the exact trig plus |u| e_cos + |w| e_sin, elementwise_ref.py)
  GELU 0.5 x (1 + erf(x/sqrt2))  E' = 1.13 E                              |gelu'| <= 1.129
                                    + 0.5 (|x| + E) U (4 |erf| + 2.26 |z| + |1 + erf|) + U |y|
                                 4 U |erf|: erff within 2 ulp; 2.26 U |z|: z = x * fl(1/sqrt2) is within 2U |z| of
                                 x / sqrt2 and erf' <= 1.1284; U |1 + erf|: the add; U |y|: the product (0.5 x is exact).
Output (out_bound): 2 u_o (|ref| + E) for the final store, u_o = u of the 16-bit type or U for fp32 (the factor 2, as
in attention_ref.py, keeps a correctly rounded result at half the allowance), plus for fp16 the subnormal floor
2 * 2^-25 (below 2^-14 rounding is absolute, half the 2^-24 spacing).

LayerNorm of computed values x^ (|x^ - x| <= E), m, v = float64 mean and variance of x, s = sqrt(v + eps),
d = x - m, y = d / s, A = max |x| + E over the row:
  input errors      dm_in = mean(E),  dv_in = mean(2 |d| E + E^2)
  fp32 mean         dm_fp = C_MEAN U A.  C_MEAN = 40: recursive summation errs by at most depth * U * sum |x|.  Emitted
                    (gemm.cu): each 32-column partial sums two chains of 16 (depth 16: 16 U A on the partial mean), the
                    row mean adds <= 24 partial means (depth 24) and divides (1).  Warp two-pass (elementwise.cu): float4
                    pairs (2), the lane's chain of <= 16 float4 (16), the 5-level shuffle tree (5), the division (1): 24.
  fp32 variance     dv_fp = C_VAR U (v + eps) + cancellation.  C_VAR = 69: emitted: x - mu rounded (2 on a square),
                    the fma chain of 16 (16), q0 + q1 (1), Chan's 2 np <= 48 sequential terms (48), the division and the
                    + eps (2); warp: 2 + 2 + 16 + 5 + 2 = 27 <= 69.  Cancellation (x - mu taken about a computed mean
                    dmu off adds 32 dmu^2 per partial): emitted mean_p(dmu^2 + 2 |d_p| D_p + D_p^2) with dmu = 16 U A,
                    d_p = the partial's float64 mean minus m and D_p = dmu + dm_fp + U |d_p| the error of the computed
                    d_p (Chan's 32 d_p^2 term); warp dm_fp^2.
  rstd              dr / r = (dv_in + dv_fp) / (2 (v + eps)) + 4 U             (rsqrtf within 2 ulp)
  y = (x^ - m^) r   E_y = (E + dm_in + dm_fp + U (|d| + E + dm)) / s + |y| dr / r + U |y|
  affine y g + b    E' = |g| E_y + U (|y g| + |y g + b|)
The output rounding of out_bound follows.

All of this is validated against a plain-torch emulation of the kernels' arithmetic in test_gemm_bound_cpu.py: the
faithful emulation stays within half the allowance and each planted fault exceeds it."""
import math
from dataclasses import dataclass
from typing import Optional

import torch

U32 = 2.0 ** -24
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
C_ACC = 17.0
C_MEAN, C_VAR = 40.0, 69.0
GELU_SLOPE = 1.13
BM = 128
STAGES = {256: 4, 192: 4, 160: 5, 128: 6, 64: 8, 32: 9}   # operand ring depth per tile width (GemmCfg)
CHUNK_ELEMS = 1 << 24                                      # float64 elements per [rows, N] temporary (128 MB)


# ------------------------------------------------------------------------------------------------ GEMM
@dataclass
class Ref:
    val: torch.Tensor          # [groups * M, N] float64: the exact epilogue result
    err: torch.Tensor          # [groups * M, N] float64: bound of the fp32 error before the final store
    M: int
    groups: int = 1


def acc_bound(a, w, ksplit=1):
    """Exact product P = a w^T ([r, K] x [N, K] float64) and E_acc of the kernel's fp32 accumulation."""
    K = a.shape[1]
    half = K // ksplit
    total = torch.zeros(a.shape[0], w.shape[0], dtype=torch.float64, device=a.device)
    s = torch.zeros_like(total)
    halves = []
    for h in range(ksplit):
        p = torch.zeros_like(total)
        for j in range(h * half, (h + 1) * half, 16):
            s += p.abs()
            p += a[:, j:j + 16] @ w[:, j:j + 16].t()
        halves.append(p)
        total += p
    e = C_ACC * 2 * U32 * (s + a.abs() @ w.abs().t())
    if ksplit == 2:
        e = e + U32 * (halves[0].abs() + halves[1].abs() + e)
    return total, e


def _add(v, e, t):
    v = v + t
    return v, e + U32 * (v.abs() + e)


def rope_apply(v, e, tab, rows, rope_cols, rope_period, tab_err=None):
    """RoPE of columns < rope_cols in 64-wide heads (32-column chunks: even = y half, odd = x half of the table) on the
    float64 value v and its bound e; tab [>= rope_period, 64] fp32, rows = the group-local row indices.  tab_err (same
    shape as tab): the table is the exact float64 trig and the kernel's fp32 table errs by at most tab_err per entry,
    which adds (|u| + E_u) e_cos + (|w| + E_w) e_sin before the fp32 terms (whose |cos|, |sin| grow by e_cos, e_sin).
    Without it the fp32 table values are exact inputs, as the docstring above states."""
    t = tab[rows % rope_period].double()
    te = tab_err[rows % rope_period].double() if tab_err is not None else None
    v, e = v.clone(), e.clone()
    for c0 in range(0, rope_cols, 32):
        h = (c0 // 32) % 2
        cs, sn = t[:, 32 * h:32 * h + 16], t[:, 32 * h + 16:32 * h + 32]
        uu, ww = v[:, c0:c0 + 16].clone(), v[:, c0 + 16:c0 + 32].clone()
        eu, ew = e[:, c0:c0 + 16].clone(), e[:, c0 + 16:c0 + 32].clone()
        ca, sa = cs.abs(), sn.abs()
        nu, nw = uu * cs - ww * sn, ww * cs + uu * sn
        if te is not None:
            ec, es = te[:, 32 * h:32 * h + 16], te[:, 32 * h + 16:32 * h + 32]
            tu = (uu.abs() + eu) * ec + (ww.abs() + ew) * es
            tw = (ww.abs() + ew) * ec + (uu.abs() + eu) * es
            ca, sa = ca + ec, sa + es
            base_u = tu + ca * eu + sa * ew + U32 * ((uu.abs() + eu) * ca + (ww.abs() + ew) * sa)
            base_w = tw + ca * ew + sa * eu + U32 * ((ww.abs() + ew) * ca + (uu.abs() + eu) * sa)
        else:
            base_u = ca * eu + sa * ew + U32 * ((uu.abs() + eu) * ca + (ww.abs() + ew) * sa)
            base_w = ca * ew + sa * eu + U32 * ((ww.abs() + ew) * ca + (uu.abs() + eu) * sa)
        v[:, c0:c0 + 16], v[:, c0 + 16:c0 + 32] = nu, nw
        e[:, c0:c0 + 16] = base_u + U32 * (nu.abs() + base_u)
        e[:, c0 + 16:c0 + 32] = base_w + U32 * (nw.abs() + base_w)
    return v, e


def gelu_apply(v, e):
    z = v * math.sqrt(0.5)
    erf = torch.erf(z)
    y = 0.5 * v * (1 + erf)
    e2 = GELU_SLOPE * e + 0.5 * (v.abs() + e) * U32 * (4 * erf.abs() + 2.26 * (z.abs() + e) + (1 + erf).abs())
    return y, e2 + U32 * (y.abs() + e2)


def reference(a, w, *, M, N, K, groups=1, w_group_rows=0, bias=None, bias_group=0, act=0, residual=None,
              rowbias=None, rb_period=1, rb_first=0, rope_tab=None, rope_cols=0, rope_period=1, ksplit=1,
              rope_tab_err=None) -> Ref:
    """a: [groups * M, >= K] 16-bit (group g = rows [g M, (g + 1) M)); w: [>= (groups - 1) w_group_rows + N, >= K];
    bias: 1-D fp32 (group g at g * bias_group); residual: [M, >= N] fp32; rope_tab: [>= rope_period, 64] fp32, or the
    exact float64 table with rope_tab_err the bound of the kernel table's error (rope_apply)."""
    dev = a.device
    f64 = dict(dtype=torch.float64, device=dev)
    val = torch.empty(groups * M, N, **f64)
    err = torch.empty(groups * M, N, **f64)
    step = max(1, CHUNK_ELEMS // N)
    rb_period = max(rb_period, 1)
    rope_period = max(rope_period, 1)
    for g in range(groups):
        wg = w[g * w_group_rows:g * w_group_rows + N, :K].double()
        bg = bias[g * bias_group:g * bias_group + N].double() if bias is not None else None
        for r0 in range(0, M, step):
            r1 = min(M, r0 + step)
            rows = torch.arange(r0, r1, device=dev)
            v, e = acc_bound(a[g * M + r0:g * M + r1, :K].double(), wg, ksplit)
            if bg is not None:
                v, e = _add(v, e, bg)
            if rope_tab is not None and rope_cols > 0:
                v, e = rope_apply(v, e, rope_tab, rows, rope_cols, rope_period, rope_tab_err)
            if rowbias is not None:
                on = ((rows % rb_period) >= rb_first)[:, None]
                v2, e2 = _add(v, e, rowbias[:N].double())
                v, e = torch.where(on, v2, v), torch.where(on, e2, e)
            if act == 1:
                v, e = gelu_apply(v, e)
            if residual is not None:
                v, e = _add(v, e, residual[r0:r1, :N].double())
            val[g * M + r0:g * M + r1], err[g * M + r0:g * M + r1] = v, e
    return Ref(val, err, M, groups)


# ------------------------------------------------------------------------------------------------ LayerNorm
def layernorm(x, e, eps, mode, gamma=None, beta=None):
    """Float64 LayerNorm of the rows of x ([R, D] float64, exact values) whose computed fp32 values err by at most e,
    and the bound of the kernel's fp32 result before its final store.  mode "emit": the GEMM epilogue's 32-column
    partials and Chan combination; "warp": the one-warp-per-row two-pass kernel."""
    R, D = x.shape
    out_v = torch.empty_like(x)
    out_e = torch.empty_like(x)
    step = max(1, CHUNK_ELEMS // D)
    for r0 in range(0, R, step):
        xv, ev = x[r0:r0 + step], e[r0:r0 + step]
        m = xv.mean(1, keepdim=True)
        d = xv - m
        v = (d * d).mean(1, keepdim=True)
        s = torch.sqrt(v + eps)
        y = d / s
        A = (xv.abs() + ev).amax(1, keepdim=True)
        dm_in = ev.mean(1, keepdim=True)
        dv_in = (2 * d.abs() * ev + ev * ev).mean(1, keepdim=True)
        dm_fp = C_MEAN * U32 * A
        if mode == "emit":
            dmu = 16 * U32 * A
            dp = xv.view(xv.shape[0], D // 32, 32).mean(2) - m                 # partial means minus the row mean
            Dp = dmu + dm_fp + U32 * dp.abs()
            canc = (dmu * dmu + 2 * dp.abs() * Dp + Dp * Dp).mean(1, keepdim=True)
        else:
            canc = dm_fp * dm_fp
        dv_fp = C_VAR * U32 * (v + eps) + canc
        dr = (dv_in + dv_fp) / (2 * (v + eps)) + 4 * U32
        dm = dm_in + dm_fp
        ey = (ev + dm + U32 * (d.abs() + ev + dm)) / s + y.abs() * dr + U32 * y.abs()
        if gamma is not None:
            g, b = gamma[:D].double(), beta[:D].double()
            yg = y * g
            o = yg + b
            ey = g.abs() * ey + U32 * (yg.abs() + o.abs())
            y = o
        out_v[r0:r0 + step], out_e[r0:r0 + step] = y, ey
    return out_v, out_e


# ------------------------------------------------------------------------------------------------ allowance
def out_bound(val, err, dtype):
    """Allowance of an output stored as `dtype` (fp32 or 16-bit) for a value val computed within err in fp32."""
    u = U16.get(dtype, U32)
    b = err + 2 * u * (val.abs() + err)
    if dtype == torch.float16:
        b = b + 2.0 ** -24
    return b


def check(out, val, bnd, what="", M=None, bn=None) -> float:
    """Fail on the first element of `out` ([G*M, N], logical rows) that is not finite or errs by more than its
    allowance, naming its group, row, column, tile (at tile width bn) and 32-column chunk; return the worst
    err / allowance."""
    err = (out.double() - val).abs()
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bnd)      # an exact result passes a zero allowance
    bad = ~(ratio <= 1)                                                   # also catches NaN
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        N = out.shape[1]
        row, col = divmod(i, N)
        M = M or out.shape[0]
        g, r = divmod(row, M)
        tile = f"tile (m {r // BM}, n {col // bn}) chunk {(col % bn) // 32}" if bn else f"chunk {col // 32}"
        raise AssertionError(
            f"{what}: group {g} row {r} column {col} [{tile}]: got {float(out[row, col]):.7g}, reference "
            f"{float(val[row, col]):.7g}, error {float(err[row, col]):.3g} > allowance {float(bnd[row, col]):.3g} "
            f"({int(bad.sum())} elements over)")
    return float(ratio.max())


# ------------------------------------------------------------------------------------------------ planted faults
def ulp(x):
    """One unit in the last place of 16-bit values x (normal range)."""
    bits = 11 if x.dtype == torch.float16 else 8
    e = torch.floor(torch.log2(x.float().abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - (bits - 1))


def off_by_4ulp(out, bnd):
    """One 16-bit element moved by 4 ulp: the one where that is largest against its allowance."""
    out = out.clone()
    i = int((4 * ulp(out).double() / bnd).flatten().argmax())
    r, c = divmod(i, out.shape[1])
    out[r, c] = (out[r, c].float() + 4 * ulp(out[r, c])).to(out.dtype)
    return out


# ------------------------------------------------------------------------------------------------ operands
NAN = float("nan")


@dataclass(frozen=True)
class Case:
    """One GEMM problem.  bn: the tile width forced through M3R_GEMM_BN (plain launches); emit: a LayerNorm-emitting
    launch (fp32 out + 16-bit norm_out); res: "" / "sep" (a separate residual) / "inplace" (residual = out);
    rb_first / rb_period: the row bias on rows (r % rb_period) >= rb_first; rope_cols / rope_period: RoPE;
    mean_offset / outlier: emitted rows with |mean| >> std and one channel 50x the others."""
    name: str
    M: int
    N: int
    K: int
    bn: Optional[int] = None
    out16: bool = True
    bias: bool = True
    gelu: bool = False
    res: str = ""
    rope_cols: int = 0
    rope_period: int = 0
    rb_first: int = -1
    rb_period: int = 200
    w_static: bool = False
    emit: bool = False
    mean_offset: float = 0.0
    outlier: bool = False
    groups: int = 1


def make_operands(c: Case, dtype, device, seed=0, pad_a_cols=True):
    """NaN-padded operands of case c: A [G*M, K] with NaN columns past K (lda = K + 64 unless pad_a_cols is False) and
    NaN rows after G*M; W rows [g*(N + 32) + 32, +N) of a larger NaN matrix; bias / rowbias with NaN after the used
    entries (group g's bias at g*(N + 32)); residual [M, N] inside an [M + 64, N + 64] NaN buffer; a RoPE table with
    NaN rows past rope_period.  Returns a dict of views (and the buffers that own them)."""
    g = torch.Generator().manual_seed(seed)
    M, N, K, G = c.M, c.N, c.K, c.groups
    rn = lambda *s: torch.randn(*s, generator=g)                             # noqa: E731
    lda = K + 64 if pad_a_cols else K
    abuf = torch.full((G * M + 64, lda), NAN)
    abuf[:G * M, :K] = rn(G * M, K)
    wg = N + 32
    wbuf = torch.full((G * wg + 32, K + (64 if pad_a_cols else 0)), NAN)
    for gg in range(G):
        wbuf[32 + gg * wg:32 + gg * wg + N, :K] = rn(N, K) * K ** -0.5
    abuf, wbuf = abuf.to(dtype).to(device), wbuf.to(dtype).to(device)
    d = dict(a=abuf[:G * M, :K], w=wbuf[32:, :K], w_group_rows=wg, keep=[abuf, wbuf])
    if c.bias:
        bbuf = torch.full((G * wg + 32,), NAN)
        for gg in range(G):
            bbuf[gg * wg:gg * wg + N] = rn(N)
        d["bias"], d["bias_group"] = bbuf.to(device), wg
    if c.rb_first >= 0:
        d["rowbias"] = torch.cat([rn(N), torch.full((32,), NAN)]).to(device)
    if c.rope_cols > 0:
        ang = rn(c.rope_period, 32) * 3.0
        tab = torch.cat([torch.cos(ang[:, :16]), torch.sin(ang[:, :16]), torch.cos(ang[:, 16:]), torch.sin(ang[:, 16:])], 1)
        d["rope_tab"] = torch.cat([tab, torch.full((16, 64), NAN)]).contiguous().to(device)
    if c.res:
        r = rn(M, N) * 3.0
        if c.mean_offset:
            r = r + c.mean_offset * (1 + rn(M, 1))
        if c.outlier:
            r[:, N // 3] *= 50.0
        rbuf = torch.full((M + 64, N + 64), NAN)
        rbuf[:M, :N] = r
        rbuf = rbuf.to(device)
        d["residual"] = rbuf[:M, :N]
        d["keep"].append(rbuf)
    return d


def ref_kwargs(c: Case, d, ksplit=1):
    """reference() keyword arguments of case c on operands d."""
    return dict(M=c.M, N=c.N, K=c.K, groups=c.groups, w_group_rows=d["w_group_rows"], bias=d.get("bias"),
                bias_group=d.get("bias_group", 0), act=int(c.gelu), residual=d.get("residual"),
                rowbias=d.get("rowbias"), rb_period=c.rb_period, rb_first=max(c.rb_first, 0),
                rope_tab=d.get("rope_tab"), rope_cols=c.rope_cols, rope_period=c.rope_period, ksplit=ksplit)


def emit_plan(M, N, K, sms):
    """(tile width, K split) the library picks for a LayerNorm-emitting launch (gemm.cu, m3r_gemm / launch_gemm)."""
    tiles_m = (M + BM - 1) // BM
    if tiles_m <= 16 and tiles_m * (N // 64) <= sms:
        tiles = tiles_m * (N // 64)
        ks = 2 if K >= 2048 and (K // 64) % 2 == 0 and 2 * tiles <= sms and tiles <= 80 else 1
        return 64, ks
    if tiles_m <= 16 and N % 128 == 0 and tiles_m * (N // 128) <= sms:
        return 128, 1
    return None, 1


# ------------------------------------------------------------------------------------------------ case matrix
def _forms():
    """Epilogue forms the plain matrix cycles through (Case fields)."""
    return [dict(), dict(gelu=True), dict(rope=True), dict(rb=True), dict(res="sep"), dict(res="inplace", out16=False),
            dict(bias=False), dict(gelu=True, rope=True, rb=True, res="sep")]


def _plain(name, M, N, K, bn, form, out16, w_static, rb_first):
    f = dict(form)
    rope = f.pop("rope", False)
    rb = f.pop("rb", False)
    out16 = f.pop("out16", out16)
    return Case(name, M, N, K, bn=bn, out16=out16, w_static=w_static, rope_cols=64 * max(1, N // 128) if rope else 0,
                rope_period=77 if rope else 0, rb_first=rb_first if rb else -1, **f)


def _plain_cases():
    cs, i = [], 0
    forms, Ms, rbf = _forms(), [1, 64, 127, 128, 129, 300], [127, 128, 129, 1]
    for bn in (32, 64, 128, 160, 192, 256):
        S = STAGES[bn]
        for K in (64, (S - 1) * 64, S * 64, (S + 1) * 64):
            for ws in (False, True):
                M = Ms[i % len(Ms)]
                cs.append(_plain(f"bn{bn}_k{K}_m{M}_{'ws' if ws else 'nows'}_{i % len(forms)}", M, 3 * bn, K, bn,
                                 forms[i % len(forms)], i % 3 != 0, ws, rbf[i % 4]))
                i += 1
    # long K
    cs += [_plain("bn64_k3072", 129, 192, 3072, 64, dict(gelu=True), True, True, 0),
           _plain("bn256_k4096", 300, 512, 4096, 256, dict(res="sep"), False, False, 0),
           _plain("bn160_k4096", 127, 320, 4096, 160, dict(rope=True), True, True, 0)]
    # several tiles per CTA: thread stores (BN 32, 64, 160, 192) and TMA stores (BN 128, 256)
    cs += [_plain("multi_bn160_rope", 805, 3840, 768, 160, dict(rope=True), True, True, 0),
           _plain("multi_bn192_gelu", 805, 3840, 256, 192, dict(gelu=True), True, False, 0),
           _plain("multi_bn32_rowbias", 805, 1024, 128, 32, dict(rb=True), False, False, 128),
           _plain("multi_bn64_res", 805, 1536, 384, 64, dict(res="sep"), False, True, 0),
           _plain("multi_tma_bn128_inplace", 1445, 1536, 512, 128, dict(res="inplace", out16=False), False, True, 0),
           _plain("multi_tma_bn128_gelu", 1445, 1536, 512, 128, dict(gelu=True), True, False, 0),
           _plain("multi_tma_bn256_all", 5157, 1024, 256, 256, dict(gelu=True, rope=True, rb=True, res="sep"), True, True,
                  129),
           _plain("multi_tma_bn256_f32_rowbias", 5157, 1024, 128, 256, dict(rb=True), False, False, 127)]
    return cs


PLAIN_CASES = _plain_cases()
EMIT_CASES = [
    Case("emit_bn64_sep", 263, 768, 768, res="sep"),
    Case("emit_bn64_k64_none", 129, 512, 64, res=""),
    Case("emit_embed_rowbias", 784, 768, 1024, res="", rb_first=196, rb_period=784),
    Case("emit_splitk_inplace", 263, 768, 3072, res="inplace"),
    Case("emit_splitk_sep", 196, 768, 3072, res="sep", w_static=True),
    Case("emit_bn128_inplace", 1500, 768, 768, res="inplace"),
    Case("emit_offset_outlier", 300, 768, 768, res="sep", mean_offset=300.0, outlier=True),
    Case("emit_splitk_offset", 196, 768, 3072, res="inplace", mean_offset=1000.0, outlier=True),
]
