"""Base pointers the GEMM epilogue, the LayerNorm / cast kernels, im2col16, the attention state merge / fill and the peer
broadcast would access off their vector width are refused with a message that names the argument, before any CUDA call:
the library is called through ctypes with made-up device addresses that are misaligned by 2, 4 or 8 bytes, so no device
is touched (and none is needed).  So are a null broadcast destination, negative RoPE dimensions and an unpatchify
without channels."""
import ctypes as C

import pytest

from must3r_b200 import _lib

BASE = 1 << 32                  # a made-up, 256-byte aligned device address; only misaligned variants are passed


def lib():
    return _lib.lib()


def last_error():
    return lib().m3r_last_error().decode()


def gemm_args():
    a = _lib.GemmArgs()
    a.A, a.lda, a.W, a.ldw = BASE, 64, BASE + 0x100000, 64
    a.M, a.N, a.K = 128, 64, 64
    a.out, a.ldc, a.out_dtype = BASE + 0x200000, 64, 1
    return a


def expect_refused(rc, name):
    msg = last_error()
    assert rc != 0 and "aligned" in msg and name in msg, (rc, msg)


@pytest.mark.parametrize("field,off", [("bias", 4), ("rowbias", 4), ("rope_tab", 4), ("residual", 4),
                                       ("out", 8), ("norm_out", 8), ("peer_out", 8)])
def test_gemm_refuses_misaligned_pointers(field, off):
    a = gemm_args()
    if field == "rope_tab":
        a.rope_cols, a.rope_period = 64, 1
    if field == "residual":
        a.ldr = 64
    if field == "peer_out":
        a.n_peer_out = 1
        a.peer_out[0] = BASE + 0x300000 + off
    elif field == "out":
        a.out = BASE + 0x200000 + off
    else:
        setattr(a, field, BASE + 0x300000 + off)
    if field == "norm_out":
        a.out_dtype, a.ldn = 0, 64
    expect_refused(lib().m3r_gemm(C.byref(a), None), field)


@pytest.mark.parametrize("field,off", [("bias", 4), ("out", 8), ("peer_out", 8)])
def test_gemm_grouped_refuses_misaligned_pointers(field, off):
    a = gemm_args()
    grp = _lib.GemmGroup()
    grp.groups, grp.w_group_rows = 2, 64
    grp.out[0], grp.out[1] = BASE + 0x200000, BASE + 0x280000
    if field == "bias":
        a.bias, grp.bias_group = BASE + 0x300000 + off, 64
    elif field == "out":
        grp.out[1] = BASE + 0x280000 + off
    else:
        a.n_peer_out = 1
        grp.peer_out[0], grp.peer_out[8] = BASE + 0x400000, BASE + 0x480000 + off
    expect_refused(lib().m3r_gemm_grouped(C.byref(a), C.byref(grp), None), field)


def test_gemm_grouped_refuses_an_odd_bias_stride():
    a = gemm_args()
    grp = _lib.GemmGroup()
    grp.groups, grp.w_group_rows, grp.bias_group = 2, 64, 65
    grp.out[0], grp.out[1] = BASE + 0x200000, BASE + 0x280000
    a.bias = BASE + 0x300000
    expect_refused(lib().m3r_gemm_grouped(C.byref(a), C.byref(grp), None), "bias_group")


def ln_call(fn, **over):
    """Arguments of the LayerNorm family with aligned made-up pointers, `over` replacing some of them."""
    kw = dict(x=BASE, add=None, gamma=BASE + 0x10000, beta=BASE + 0x20000, out=BASE + 0x30000)
    kw.update(over)
    L = lib()
    if fn == "layernorm":
        return L.m3r_layernorm(kw["x"], 64, kw["add"], 64, kw["gamma"], kw["beta"], 1e-6, 4, 64, kw["out"], 64,
                               kw.get("out_dtype", 0), 0, None)
    if fn == "normalize16":
        return L.m3r_normalize16(kw["x"], 64, kw["add"], 64, 4, 1, 1e-6, 4, 64, kw["out"], 64, 0, None)
    if fn == "layernorm16":
        return L.m3r_layernorm16(kw["x"], 64, kw["gamma"], kw["beta"], 1e-6, 4, 64, kw["out"], 64, 0, None)
    if fn == "cast16":
        return L.m3r_cast16(kw["x"], 64, 4, 64, kw["out"], 64, 0, None)
    return L.m3r_add_cast16(kw["x"], 64, kw["add"] or BASE + 0x40000, 64, 4, 64, kw["out"], 64, 0, None)


@pytest.mark.parametrize("fn,field,off,extra", [
    ("layernorm", "x", 8, {}), ("layernorm", "add", 8, {}), ("layernorm", "gamma", 8, {}), ("layernorm", "beta", 4, {}),
    ("layernorm", "out", 8, {"out_dtype": 0}), ("layernorm", "out", 4, {"out_dtype": 1}),
    ("normalize16", "x", 4, {}), ("normalize16", "add", 8, {}), ("normalize16", "out", 4, {}),
    ("layernorm16", "x", 4, {}), ("layernorm16", "x", 2, {}), ("layernorm16", "gamma", 8, {}), ("layernorm16", "out", 4, {}),
    ("cast16", "x", 8, {}), ("cast16", "out", 4, {}),
    ("add_cast16", "x", 8, {}), ("add_cast16", "add", 4, {}), ("add_cast16", "out", 2, {}),
])
def test_layernorm_family_refuses_misaligned_pointers(fn, field, off, extra):
    base = dict(x=BASE, add=BASE + 0x40000, gamma=BASE + 0x10000, beta=BASE + 0x20000, out=BASE + 0x30000)
    rc = ln_call(fn, **{field: base[field] + off}, **extra)
    name = {"layernorm16": {"x": "x16", "out": "out16"}}.get(fn, {}).get(field, field)
    expect_refused(rc, name)


def ptrs(*addrs):
    return (C.c_void_p * len(addrs))(*addrs)


def elementwise_call(fn, field, off):
    """One vectorised elementwise entry point with aligned made-up pointers, `field` moved by `off` bytes."""
    L = lib()
    at = lambda f, a: a + off if f == field else a                          # noqa: E731
    if fn == "im2col16":
        return L.m3r_im2col16(at("img", BASE), 2, 32, 48, at("out", BASE + 0x100000), 0, None)
    if fn == "attn_merge":
        po = ptrs(BASE, BASE + 0x10000, at("parts_o[2]", BASE + 0x20000))
        pml = ptrs(BASE + 0x30000, at("parts_ml[1]", BASE + 0x40000), BASE + 0x50000)
        return L.m3r_attn_merge(po, pml, 3, 64, 2, at("out", BASE + 0x60000), 128, 0, None)
    if fn == "attn_state_fill":
        return L.m3r_attn_state_fill(at("export_o", BASE), at("export_ml", BASE + 0x10000), 64, 2, None)
    d = ptrs(BASE + 0x10000, BASE + 0x20000, at("dsts[2]", BASE + 0x30000))
    return L.m3r_peer_bcast(at("src", BASE), d, 3, 4096, None)


@pytest.mark.parametrize("fn,field,off", [
    ("im2col16", "img", 8), ("im2col16", "img", 4), ("im2col16", "out", 4), ("im2col16", "out", 2),
    ("attn_merge", "parts_o[2]", 8), ("attn_merge", "parts_ml[1]", 4), ("attn_merge", "out", 8),
    ("attn_state_fill", "export_o", 8), ("attn_state_fill", "export_ml", 4),
    ("peer_bcast", "src", 8), ("peer_bcast", "dsts[2]", 8), ("peer_bcast", "dsts[2]", 4),
])
def test_elementwise_refuses_misaligned_pointers(fn, field, off):
    expect_refused(elementwise_call(fn, field, off), field)


def expect_argument_error(rc, *words):
    msg = last_error()
    assert rc != 0 and all(w in msg for w in words), (rc, msg)


def test_peer_bcast_refuses_a_null_destination():
    d = ptrs(BASE + 0x10000, None, BASE + 0x30000)
    expect_argument_error(lib().m3r_peer_bcast(BASE, d, 3, 4096, None), "dsts[1]", "non-null")


@pytest.mark.parametrize("B,N,H,D", [(-1, -2, 3, 64), (2, -3, -1, 64), (-2, 5, -4, 12), (1, 1, 1, -4)])
def test_rope_2d_refuses_negative_dimensions(B, N, H, D):
    rc = lib().m3r_rope_2d(BASE, 1, B, N, H, D, 4096, 64, 64, BASE + 0x100000, 100.0, 1.0, None)
    expect_argument_error(rc, "rope_2d", "negative dimension")


@pytest.mark.parametrize("C_", [0, -1, -7])
def test_unpatchify_refuses_no_channels(C_):
    rc = lib().m3r_unpatchify(BASE, 2, 32, 48, C_, BASE + 0x100000, None)
    expect_argument_error(rc, "unpatchify", "C=")
