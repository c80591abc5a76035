"""The GEMM epilogue at every tile width and in every mode, with the output inside a larger buffer filled with a sentinel.

Each case checks that nothing outside the [M, N] result changed, the error of every row against fp32 torch math on the
same 16-bit inputs, and bitwise equality where two stores cover the same rows:
- plain launches at BN 32, 64, 128, 160, 192 and 256 (the 16-bit output of BN 32 and 160 ends in a half-width chunk),
  for each epilogue form, with M a multiple of the tile height and ragged;
- the batch row remap (rows_per_batch) with batch boundaries inside a 128-row tile, with two peer buffers on the same
  device that must receive exactly the rows of the output;
- the grouped GEMM with a ragged M, whose last m-tile of group g holds rows of group g + 1;
- the LayerNorm-emitting kernels at BN 64 with and without split-K and at BN 128, ragged M, both outputs."""
import os

import pytest
import torch
import torch.nn.functional as F

from must3r_b200 import ops

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
ROW_TOL = {torch.float16: 2.5e-3, torch.bfloat16: 2e-2, torch.float32: 1e-4}
SENTINEL = 7.0
PERIOD = 200                       # RoPE table rows and row-bias period
ROPE_COLS = 512
FORMS = ["bias_f32", "bias_16", "gelu", "rope", "rowbias", "residual_inplace", "ldc_slice"]


def rnd(*shape, dtype=torch.float32, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def padded(rows, cols, dtype, pad_rows=64, pad_cols=0):
    """A sentinel-filled buffer and the [rows, cols] view inside it (pad_cols columns on either side)."""
    buf = torch.full((rows + pad_rows, cols + 2 * pad_cols), SENTINEL, device="cuda", dtype=dtype)
    return buf, buf[:rows, pad_cols:pad_cols + cols]


def untouched(buf, view_mask):
    return bool((buf[~view_mask] == SENTINEL).all())


def inside(buf, r0, r1, c0, c1):
    m = torch.zeros_like(buf, dtype=torch.bool)
    m[r0:r1, c0:c1] = True
    return m


def assert_rows_close(out, ref, dtype):
    err = (out.float() - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-6)
    assert float(err.max()) < ROW_TOL[dtype], float(err.max())


def rope_ref(y, tab, rows):
    y = y.clone()
    t = tab[torch.arange(rows, device=y.device) % tab.shape[0]]
    for c0 in range(0, ROPE_COLS, 32):
        h = (c0 // 32) % 2
        cs, sn = t[:, 32 * h:32 * h + 16], t[:, 32 * h + 16:32 * h + 32]
        u, v = y[:, c0:c0 + 16].clone(), y[:, c0 + 16:c0 + 32].clone()
        y[:, c0:c0 + 16] = u * cs - v * sn
        y[:, c0 + 16:c0 + 32] = v * cs + u * sn
    return y


@pytest.fixture
def force_bn():
    def set_bn(bn):
        os.environ["M3R_GEMM_BN"] = str(bn)
    yield set_bn
    os.environ.pop("M3R_GEMM_BN", None)


@pytest.fixture(scope="module")
def plain_operands():
    N, K, M = 3840, 128, 512                                       # N: a multiple of every tile width
    ang = rnd(PERIOD, 32, seed=5) * 3.0
    rope = torch.cat([torch.cos(ang[:, :16]), torch.sin(ang[:, :16]), torch.cos(ang[:, 16:]), torch.sin(ang[:, 16:])], 1).contiguous()
    a = rnd(M, K, dtype=torch.bfloat16, seed=1)
    w = rnd(N, K, dtype=torch.bfloat16, seed=2, scale=K ** -0.5)
    return a, w, rnd(N, seed=3), {"rope": rope, "rowbias": rnd(N, seed=6), "res": rnd(M, N, seed=7)}


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("M", [512, 512 - 37])
@pytest.mark.parametrize("bn", [32, 64, 128, 160, 192, 256])
def test_plain_epilogue_every_tile_width(plain_operands, force_bn, bn, M, form):
    a, w, bias, extra = plain_operands
    a = a[:M]
    N = w.shape[0]
    force_bn(bn)
    out_dtype = torch.float32 if form in ("bias_f32", "rowbias", "residual_inplace") else a.dtype
    pad = 256 if form == "ldc_slice" else 0
    buf, out = padded(M, N, out_dtype, pad_cols=pad)
    kw = {}
    ref = a.float() @ w.float().t() + bias
    if form == "gelu":
        kw["act"] = "gelu"
        ref = F.gelu(ref)
    elif form == "rope":
        kw.update(rope_tab=extra["rope"], rope_cols=ROPE_COLS)
        ref = rope_ref(ref, extra["rope"], M)
    elif form == "rowbias":
        kw.update(rowbias=extra["rowbias"], rb_period=PERIOD, rb_first=1)
        ref = ref + ((torch.arange(M, device="cuda") % PERIOD) >= 1)[:, None].float() * extra["rowbias"]
    elif form == "residual_inplace":
        out.copy_(extra["res"][:M])
        kw["residual"] = out
        ref = ref + extra["res"][:M]
    ops.linear(a, w, bias, out=out, **kw)
    torch.cuda.synchronize()
    assert untouched(buf, inside(buf, 0, M, pad, pad + N)), "a store landed outside the output"
    assert_rows_close(out, ref, out_dtype)


@pytest.mark.parametrize("M", [900, 15000])                        # one wave / several tiles per CTA
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("dtype", DT)
def test_row_remap_with_peer_buffers(force_bn, dtype, bn, M):
    """rows_per_batch = 300 puts batch boundaries inside 128-row tiles; batch b goes to rows [400 b, 400 b + 300) of the
    output and of both peer buffers, which must all be bitwise equal, with the 100-row gaps untouched."""
    N, K, RPB, STRIDE = 1280, 256, 300, 400
    a, w = rnd(M, K, dtype=dtype, seed=1), rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3)
    force_bn(bn)
    batches = (M + RPB - 1) // RPB
    bufs = [padded(batches * STRIDE, N, dtype)[0] for _ in range(3)]
    outs = [b[:batches * STRIDE] for b in bufs]
    ops.linear(a, w, bias, act="gelu", out=outs[0], rows_per_batch=RPB, batch_stride_rows=STRIDE,
               peer_ptrs=[outs[1].data_ptr(), outs[2].data_ptr()])
    torch.cuda.synchronize()
    dest = torch.arange(M, device="cuda")
    dest = (dest // RPB) * STRIDE + dest % RPB
    written = torch.zeros(bufs[0].shape[0], dtype=torch.bool, device="cuda")
    written[dest] = True
    for b in bufs:
        assert bool((b[~written] == SENTINEL).all()), "a row landed outside its batch slot"
        assert torch.equal(b, bufs[0])
    assert_rows_close(bufs[0][dest], F.gelu(a.float() @ w.float().t() + bias), dtype)


@pytest.mark.parametrize("out_dtype", ["16", torch.float32])
@pytest.mark.parametrize("G,M,N,K", [(3, 300, 256, 128), (12, 1536 - 37, 1536, 128)])
@pytest.mark.parametrize("dtype", DT)
def test_grouped_ragged_groups_stay_apart(dtype, G, M, N, K, out_dtype):
    """Group g's last m-tile also multiplies the first rows of group g + 1: they must not reach group g's output (the
    sentinel rows after each output) nor its peer buffer."""
    od = dtype if out_dtype == "16" else torch.float32
    a = rnd(G, M, K, dtype=dtype, seed=1)
    w = rnd(G, N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    bias = rnd(G, N, seed=3)
    bufs = [padded(M, N, od)[0] for _ in range(G)]
    peer_bufs = [padded(M, N, od)[0] for _ in range(G)] if od != torch.float32 else None
    ops.linear_grouped(a, w, bias, [b[:M] for b in bufs],
                       peer_ptrs=[[p.data_ptr()] for p in peer_bufs] if peer_bufs else None)
    torch.cuda.synchronize()
    for g in range(G):
        assert untouched(bufs[g], inside(bufs[g], 0, M, 0, N)), g
        assert_rows_close(bufs[g][:M], a[g].float() @ w[g].float().t() + bias[g], od)
        if peer_bufs:
            assert torch.equal(peer_bufs[g], bufs[g]), g


@pytest.mark.parametrize("M,N,K,bn", [(300 - 37, 768, 3072, 64),       # split-K CTA pairs
                                      (300 - 37, 768, 768, 64),
                                      (1500, 768, 768, 128)])           # 12 m-tiles: 144 tiles at BN 64 exceed one wave
@pytest.mark.parametrize("dtype", DT)
def test_layernorm_emit_epilogue(force_bn, dtype, M, N, K, bn):
    a, w = rnd(M, K, dtype=dtype, seed=1), rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    bias, res = rnd(N, seed=3), rnd(M, N, seed=4, scale=3.0)
    pad = 64
    obuf, out = padded(M, N, torch.float32, pad_cols=pad)
    nbuf, nout = padded(M, N, dtype, pad_cols=pad)
    ops.linear(a, w, bias, residual=res, out=out, norm_out=nout, norm_eps=1e-6)
    torch.cuda.synchronize()
    x_ref = a.float() @ w.float().t() + bias + res
    assert untouched(obuf, inside(obuf, 0, M, pad, pad + N)) and untouched(nbuf, inside(nbuf, 0, M, pad, pad + N))
    assert_rows_close(out, x_ref, torch.float32)
    assert_rows_close(nout, F.layer_norm(x_ref, (N,), eps=1e-6), dtype)
    if K < 2048:
        # without split-K the fp32 output is the plain GEMM's at the same tile width, bit for bit
        force_bn(bn)
        plain = ops.linear(a, w, bias, residual=res, out_dtype=torch.float32)
        torch.cuda.synchronize()
        assert torch.equal(out, plain)
