"""m3r_gemm_e4m3, m3r_gemm_grouped_e4m3, m3r_normalize8 and the e4m3 norm_out of the LayerNorm-emitting GEMM, element by
element against the float64 allowances of tests/gemm_e4m3_ref.py and tests/gemm_ref.py.

Operands are e4m3 LayerNorm rows (the A operand the model feeds these GEMMs) and row-quantised weights; padding bytes of
A and W are 0x7f (an e4m3 NaN) and every output is a view into a sentinel-filled buffer that must stay untouched.  Cases
cover odd M, one wave and several tiles per CTA (TMA stores), every e4m3 tile width, RoPE, GELU, bias, residual, fp32
and bf16 outputs, the grouped memory append with its row remap, the split-K and multi-tile LayerNorm emitters with e4m3
norm_out, and the argument errors."""
import ctypes as C

import pytest
import torch

from gemm_e4m3_ref import check_window, reference8, to_e4m3
from gemm_ref import check, layernorm, out_bound, reference
from must3r_b200 import _lib

pytestmark = pytest.mark.gpu
SENTINEL, PAD, EPS = 7.0, 64, 1e-6
NAN8 = 0x7F


def sp():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ln_rows(M, K, g):
    x = torch.randn(M, K, generator=g, device="cuda", dtype=torch.float64) * 3 + 1
    x[0, :] = 0.0
    x[0, 0] = 1.0                                        # the extreme row: one value reaches sqrt(K - 1)
    return (x - x.mean(1, keepdim=True)) / x.std(1, unbiased=False, keepdim=True)


def padded8(t, extra_cols=32, extra_rows=8):
    """e4m3 copy of t inside a NaN-filled buffer: the view has leading dim cols + extra_cols (a multiple of 16)."""
    R, K = t.shape
    buf = torch.full((R + extra_rows, K + extra_cols), NAN8, dtype=torch.uint8, device="cuda")
    v = buf[:R, :K]
    v.copy_(to_e4m3(t).view(torch.uint8))
    return v.view(torch.float8_e4m3fn)


def out_buffer(rows, N, dtype):
    buf = torch.full((rows + PAD, N + 2 * PAD), SENTINEL, device="cuda", dtype=dtype)
    return buf, buf[:rows, PAD:PAD + N]


def untouched(buf, rows, N):
    m = torch.ones_like(buf, dtype=torch.bool)
    m[:rows, PAD:PAD + N] = False
    return bool((buf[m].float() == SENTINEL).all())


def operands(M, N, K, seed, w_rows=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a8 = padded8(ln_rows(M, K, g))
    w = torch.randn(w_rows or N, K, generator=g, device="cuda") * torch.linspace(0.02, 2.0, w_rows or N, device="cuda")[:, None]
    from must3r_b200.model.common import quantize_e4m3_rows
    wq, s = quantize_e4m3_rows(w)
    w8 = padded8(wq.float())
    bias = torch.randn(w_rows or N, generator=g, device="cuda")
    return a8, w8, s, bias, g


def args(a8, w8, M, N, K, out, bias=None, act=0, residual=None, rope=None):
    a = _lib.GemmArgs()
    a.A, a.lda, a.W, a.ldw = a8.data_ptr(), a8.stride(0), w8.data_ptr(), w8.stride(0)
    a.M, a.N, a.K, a.is_bf16 = M, N, K, 1
    a.bias = bias.data_ptr() if bias is not None else None
    a.act = act
    if residual is not None:
        a.residual, a.ldr = residual.data_ptr(), residual.stride(0)
    if rope is not None:
        a.rope_tab, a.rope_cols, a.rope_period = rope.data_ptr(), N, rope.shape[0]
    a.out, a.ldc, a.out_dtype = out.data_ptr(), out.stride(0), 0 if out.dtype == torch.float32 else 1
    a.w_static = 1
    return a


def e8(scale, a_e4m3=1, norm=0):
    x = _lib.GemmE4M3Args()
    x.a_e4m3, x.w_scale, x.norm_e4m3 = a_e4m3, scale.data_ptr() if scale is not None else None, norm
    return x


# (name, M, N, K, bias, gelu, residual, rope, out16)
CASES = [
    ("qkv_rope_odd", 77, 384, 128, True, False, False, True, True),
    ("fc1_gelu", 300, 512, 128, True, True, False, False, True),
    ("fp32_residual", 129, 192, 256, True, False, True, False, False),
    ("multiwave_tma", 4999, 1024, 1024, True, True, False, False, True),
    ("multiwave_fp32", 2048, 768, 768, False, False, True, False, False),
    ("k_deep", 33, 64, 4096, True, False, False, False, True),
]


@pytest.mark.parametrize("c", CASES, ids=[c[0] for c in CASES])
def test_plain_e4m3_against_float64(c):
    name, M, N, K, has_b, gelu, has_r, has_rope, out16 = c
    a8, w8, s, bias, g = operands(M, N, K, M + N + K)
    residual = torch.randn(M, N, generator=g, device="cuda") if has_r else None
    rope = None
    if has_rope:
        ang = torch.rand(M, 16, generator=g, device="cuda") * 6.28
        rope = torch.cat([ang.cos(), ang.sin(), (ang * 0.5).cos(), (ang * 0.5).sin()], 1).contiguous()
    odt = torch.bfloat16 if out16 else torch.float32
    buf, out = out_buffer(M, N, odt)
    a = args(a8, w8, M, N, K, out, bias if has_b else None, int(gelu), residual, rope)
    _lib.check(_lib.lib().m3r_gemm_e4m3(C.byref(a), C.byref(e8(s)), sp()), "gemm_e4m3")
    torch.cuda.synchronize()
    val, err = reference8(a8, w8, s, M=M, N=N, K=K, bias=bias if has_b else None, act=int(gelu), residual=residual,
                          rope_tab=rope, rope_cols=N if has_rope else 0, rope_period=M)
    worst = check(out, val, out_bound(val, err, odt), name, M)
    assert untouched(buf, M, N)
    print(f"\n[gemm-e4m3] {name}: worst err/bound {worst:.3f}")


def test_grouped_append_e4m3():
    """The memory append: 3 levels of [5D, D] stacked weights, rows [3D, 5D) of each, rows remapped into [B, cap, 2D]."""
    D, groups, B, rows_per = 128, 3, 2, 45
    M = B * rows_per
    a8 = padded8(ln_rows(groups * M, D, torch.Generator(device="cuda").manual_seed(3)))
    _, w8all, sall, ball, _ = operands(8, 5 * D, D, 5, w_rows=groups * 5 * D)
    W, S, Bi = w8all[3 * D:], sall[3 * D:], ball[3 * D:]
    cap = 64
    bufs = [out_buffer(B * cap, 2 * D, torch.bfloat16) for _ in range(groups)]
    a = args(a8, W, M, 2 * D, D, bufs[0][1], Bi)
    a.rows_per_batch, a.batch_stride_rows = rows_per, cap
    grp = _lib.GemmGroup()
    grp.groups, grp.w_group_rows, grp.bias_group, grp.max_ctas = groups, 5 * D, 5 * D, 40
    for l in range(groups):
        grp.out[l] = bufs[l][1].data_ptr()
    _lib.check(_lib.lib().m3r_gemm_grouped_e4m3(C.byref(a), C.byref(grp), C.byref(e8(S)), sp()), "gemm_grouped_e4m3")
    torch.cuda.synchronize()
    val, err = reference8(a8, W, S, M=M, N=2 * D, K=D, groups=groups, w_group_rows=5 * D, bias=Bi, bias_group=5 * D)
    for l in range(groups):
        buf, out = bufs[l]
        got = out.view(B, cap, 2 * D)[:, :rows_per].reshape(M, 2 * D)
        v, e = val[l * M:(l + 1) * M], err[l * M:(l + 1) * M]
        check(got, v, out_bound(v, e, torch.bfloat16), f"level {l}", M)
        assert bool((out.view(B, cap, 2 * D)[:, rows_per:].float() == SENTINEL).all())
        assert untouched(buf, B * cap, 2 * D)


@pytest.mark.parametrize("M,D", [(1, 128), (77, 768), (5000, 1024)])
def test_normalize8_is_the_e4m3_rounding_of_the_float64_layernorm(M, D):
    g = torch.Generator(device="cuda").manual_seed(M)
    x = (torch.randn(M, D, generator=g, device="cuda") * 4 + 2).float()
    x[0, :] = 0.0
    x[0, 0] = 50.0
    buf = torch.full((M + 4, D + 64), 0x55, dtype=torch.uint8, device="cuda")
    out = buf[:M, 16:16 + D]
    _lib.check(_lib.lib().m3r_normalize8(C.c_void_p(x.data_ptr()), D, None, 0, 0, 1, EPS, M, D, C.c_void_p(out.data_ptr()),
                                         buf.stride(0), sp()), "normalize8")
    torch.cuda.synchronize()
    v, e = layernorm(x.double(), torch.zeros_like(x, dtype=torch.float64), EPS, "warp")
    inexact = check_window(out.view(torch.float8_e4m3fn), v, e, "normalize8")
    assert inexact <= M * D * 1e-3, inexact                  # only values within the fp32 allowance of a rounding tie
    m = torch.ones_like(buf, dtype=torch.bool)
    m[:M, 16:16 + D] = False
    assert bool((buf[m] == 0x55).all())


@pytest.mark.parametrize("M,N,K", [(300, 768, 768), (128, 768, 3072), (1000, 128, 512)], ids=["tiles", "splitk", "multitile_m"])
def test_emitted_norm_out_e4m3(M, N, K):
    """A 16-bit (bf16) LayerNorm-emitting GEMM whose norm_out is e4m3: out (fp32) within the GEMM allowance, norm_out
    inside the e4m3 window of the float64 LayerNorm of the exact residual stream."""
    g = torch.Generator(device="cuda").manual_seed(K)
    a = torch.randn(M, K, generator=g, device="cuda").bfloat16()
    w = (torch.randn(N, K, generator=g, device="cuda") / K ** 0.5).bfloat16()
    bias = torch.randn(N, generator=g, device="cuda")
    res = torch.randn(M, N, generator=g, device="cuda")
    buf, out = out_buffer(M, N, torch.float32)
    nbuf = torch.full((M + 8, N + 64), 0x55, dtype=torch.uint8, device="cuda")
    nout = nbuf[:M, 32:32 + N]
    ga = args(a, w, M, N, K, out, bias, 0, res)
    ga.is_bf16 = 1
    ga.norm_out, ga.ldn, ga.norm_eps = nout.data_ptr(), nbuf.stride(0), EPS
    _lib.check(_lib.lib().m3r_gemm_e4m3(C.byref(ga), C.byref(e8(None, 0, 1)), sp()), "gemm norm_e4m3")
    torch.cuda.synchronize()
    ksplit = 2 if K >= 2048 else 1
    ref = reference(a, w, M=M, N=N, K=K, bias=bias, residual=res, ksplit=ksplit)
    check(out, ref.val, out_bound(ref.val, ref.err, torch.float32), "out", M)
    v, e = layernorm(ref.val, ref.err, EPS, "emit")
    check_window(nout.view(torch.float8_e4m3fn), v, e, "norm_out")
    assert untouched(buf, M, N)
    m = torch.ones_like(nbuf, dtype=torch.bool)
    m[:M, 32:32 + N] = False
    assert bool((nbuf[m] == 0x55).all())


def test_argument_errors():
    lib = _lib.lib()
    a8, w8, s, bias, _ = operands(64, 128, 128, 1)
    out = torch.empty(64, 128, device="cuda", dtype=torch.bfloat16)

    def err(a, x):
        assert lib.m3r_gemm_e4m3(C.byref(a), C.byref(x), sp()) != 0
        return lib.m3r_last_error().decode()

    assert "w_scale" in err(args(a8, w8, 64, 128, 128, out), e8(None))
    odd = torch.empty(130, device="cuda")[1:129]
    assert "8-byte" in err(args(a8, w8, 64, 128, 128, out), e8(odd))
    a = args(a8, w8, 64, 128, 128, out)
    a.is_bf16 = 0
    assert "is_bf16" in err(a, e8(s))
    a = args(a8, w8, 64, 128, 64, out)
    assert "K % 128" in err(a, e8(s))
    a = args(a8, w8, 64, 128, 128, out)
    a.lda = 136
    assert "lda" in err(a, e8(s))
    a = args(a8, w8, 64, 128, 128, out)
    a.norm_out, a.ldn = out.data_ptr(), 128
    assert "norm_out" in err(a, e8(s))
    assert "norm_e4m3 without norm_out" in err(args(a8, w8, 64, 128, 128, out), e8(s, 1, 1))
    grp = _lib.GemmGroup()
    grp.groups, grp.w_group_rows = 2, 3
    grp.out[0] = grp.out[1] = out.data_ptr()
    assert lib.m3r_gemm_grouped_e4m3(C.byref(args(a8, w8, 32, 128, 128, out)), C.byref(grp), C.byref(e8(s)), sp()) != 0
    assert "w_group_rows" in lib.m3r_last_error().decode()
