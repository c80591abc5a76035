"""Operator-level parity of the sm_90a kernels (through the C ABI) against plain fp32 torch math on the
same 16-bit-rounded inputs.  Tolerances (rel-L2): fp32-out GEMM 2e-5 (accumulation order only); 16-bit
outputs add one rounding (fp16 2^-11, bf16 2^-8); attention adds the 16-bit rounding of P."""
import math
import os

import pytest
import torch

from must3r_b200 import ops
from must3r_b200.synthetic import rel_l2
from oracle import must3r_oracle as orc

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
OUT_TOL = {torch.float16: 6e-4, torch.bfloat16: 5e-3, torch.float32: 2e-5}


def rnd(*shape, dtype=torch.float32, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (300, 768, 128), (196, 2304, 768), (1000, 1024, 1024), (77, 256, 4096)])
def test_gemm_plain(dtype, bn, M, N, K):
    os.environ["M3R_GEMM_BN"] = str(bn)
    try:
        a, w = rnd(M, K, dtype=dtype, seed=1), rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
        bias = rnd(N, seed=3)
        ref = a.float() @ w.float().t() + bias
        out32 = ops.linear(a, w, bias, out_dtype=torch.float32)
        assert rel_l2(out32, ref) < OUT_TOL[torch.float32]
        out16 = ops.linear(a, w, bias)
        assert out16.dtype == dtype and rel_l2(out16, ref) < OUT_TOL[dtype]
    finally:
        os.environ.pop("M3R_GEMM_BN", None)


@pytest.mark.parametrize("M,N,K", [(768, 768, 768), (200, 256, 128), (5000, 1024, 1024), (768, 768, 3072)])
def test_gemm_static_weight_prefetch(M, N, K):
    """w_static=True: the weight halves of the first ring of stages are requested before the programmatic-dependency wait
    (K shorter / longer than the ring, more tiles than SMs); results must not change, also back to back on one stream."""
    dtype = torch.float16
    a, w = rnd(M, K, dtype=dtype, seed=1), rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
    bias = rnd(N, seed=3)
    ref = ops.linear(a, w, bias, out_dtype=torch.float32)
    for bn in (64, 128, 256):
        os.environ["M3R_GEMM_BN"] = str(bn)
        try:
            outs = [ops.linear(a, w, bias, out_dtype=torch.float32, w_static=True) for _ in range(3)]
        finally:
            os.environ.pop("M3R_GEMM_BN", None)
        for o in outs:
            assert torch.equal(o, ref) or rel_l2(o, ref) < 1e-6
    # a chain of dependent launches: each GEMM consumes the previous one's output as its activations
    x = a
    for _ in range(4):
        x = ops.linear(x, w[:K] if N >= K else w, None, w_static=True) if N == K else x
    if N == K:
        y = a
        for _ in range(4):
            y = ops.linear(y, w, None)
        assert torch.equal(x, y)


@pytest.mark.parametrize("dtype", DT)
def test_gemm_large_persistent(dtype):
    """More tiles than SMs: exercises the persistent loop and the smem ring wrap across tiles."""
    M, N, K = 5000, 4096, 1024
    a, w = rnd(M, K, dtype=dtype, seed=4), rnd(N, K, dtype=dtype, seed=5, scale=K ** -0.5)
    ref = a.float() @ w.float().t()
    out = ops.linear(a, w, None, out_dtype=torch.float32)
    assert rel_l2(out, ref) < OUT_TOL[torch.float32]
    # bit-level check of one far tile against a float64 dot product (fp32 accumulate: ~1e-6 abs here)
    sl = (slice(4900, 4916), slice(4000, 4016))
    ref64 = (a[sl[0]].double() @ w[sl[1]].double().t())
    assert (out[sl].double() - ref64).abs().max() < 1e-4


@pytest.mark.parametrize("dtype", DT)
def test_gemm_multi_destination_epilogue(dtype):
    """Fused GEMM -> all-gather building block: the 16-bit tile is stored to every pointer of peer_out with the same
    row mapping (here the 'peers' are other local buffers; over CUDA IPC they are the other GPUs' memory buffers)."""
    M, N, K = 768, 1536, 768
    a, w = rnd(M, K, dtype=dtype, seed=40), rnd(N, K, dtype=dtype, seed=41, scale=K ** -0.5)
    bias = rnd(N, seed=42)
    bufs = [torch.zeros(3 * M, N, device="cuda", dtype=dtype) for _ in range(3)]
    out = ops.linear(a, w, bias, peer_ptrs=[b[M:].data_ptr() for b in bufs])
    ref = a.float() @ w.float().t() + bias
    assert rel_l2(out, ref) < OUT_TOL[dtype]
    for b in bufs:
        assert torch.equal(b[M:2 * M], out) and float(b[:M].abs().max()) == 0 and float(b[2 * M:].abs().max()) == 0


@pytest.mark.parametrize("dtype", DT)
def test_gemm_epilogues(dtype):
    M, N, K = 392, 768, 768
    a, w = rnd(M, K, dtype=dtype, seed=6), rnd(N, K, dtype=dtype, seed=7, scale=K ** -0.5)
    bias, res, rb = rnd(N, seed=8), rnd(M, N, seed=9), rnd(N, seed=10)
    base = a.float() @ w.float().t() + bias
    # GELU (exact erf form)
    out = ops.linear(a, w, bias, act="gelu", out_dtype=torch.float32)
    assert rel_l2(out, torch.nn.functional.gelu(base)) < 2e-5
    # residual, in place on the fp32 stream
    x = res.clone()
    ops.linear(a, w, bias, residual=x, out=x)
    assert rel_l2(x, base + res) < 2e-5
    # image2_embed row bias: rows with (row % 196) >= 98
    out = ops.linear(a, w, bias, rowbias=rb, rb_period=196, rb_first=98, out_dtype=torch.float32)
    ref = base.clone()
    rows = (torch.arange(M, device="cuda") % 196) >= 98
    ref[rows] += rb
    assert rel_l2(out, ref) < 2e-5
    # append into a [B=2, cap=300, N] buffer at row offset 100 (196 rows per batch)
    buf = torch.zeros(2, 300, N, device="cuda", dtype=dtype)
    ops.linear(a, w, bias, out=buf.view(600, N)[100:], rows_per_batch=196, batch_stride_rows=300)
    assert rel_l2(buf[:, 100:296].reshape(M, N), base) < OUT_TOL[dtype]
    assert float(buf[:, :100].abs().max()) == 0 and float(buf[:, 296:].abs().max()) == 0


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("f0", [1.0, 224 / 512])
def test_gemm_rope_epilogue(dtype, f0):
    """Fused qkv projection + 2-D RoPE (attention.py:92-96 + curope) on a non-square 6x9 grid, 2 views."""
    H, D, gh, gw, V = 3, 192, 6, 9, 2
    N = gh * gw
    a, w = rnd(V * N, D, dtype=dtype, seed=11), rnd(3 * D, D, dtype=dtype, seed=12, scale=D ** -0.5)
    bias = rnd(3 * D, seed=13)
    ys, xs = torch.meshgrid(torch.arange(gh), torch.arange(gw), indexing="ij")
    pos = torch.stack([ys, xs], -1).reshape(1, N, 2).cuda()
    tab = ops.rope_table(pos[0].contiguous(), 100.0, f0)
    out = ops.linear(a, w, bias, rope_tab=tab, rope_cols=2 * D, out_dtype=torch.float32)
    qkv = (a.float() @ w.float().t() + bias).reshape(V, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    q = orc.rope2d(qkv[0], pos.expand(V, -1, -1), 100.0, f0)
    k = orc.rope2d(qkv[1], pos.expand(V, -1, -1), 100.0, f0)
    ref = torch.stack([q, k, qkv[2]], 0).permute(1, 3, 0, 2, 4).reshape(V * N, 3 * D)
    assert rel_l2(out, ref) < 3e-5


@pytest.mark.parametrize("out_dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("D", [768, 1024, 128])
def test_layernorm(out_dtype, D):
    M = 333
    x, add = rnd(M, D, seed=15, scale=3.0) + 0.5, rnd(M, D, seed=16)
    g, b = 1 + 0.1 * rnd(D, seed=17), 0.1 * rnd(D, seed=18)
    out = ops.layernorm(x, g, b, 1e-6, out_dtype=out_dtype)
    assert rel_l2(out, torch.nn.functional.layer_norm(x, (D,), g, b, 1e-6)) < OUT_TOL[out_dtype]
    out = ops.layernorm(x, g, b, 1e-5, add=add, out_dtype=out_dtype)
    assert rel_l2(out, torch.nn.functional.layer_norm(x + add, (D,), g, b, 1e-5)) < OUT_TOL[out_dtype]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("M,D", [(333, 768), (5000, 768), (100, 1024), (64, 128)])
def test_layernorm16_and_add_cast16(dtype, M, D):
    """16-bit-in LayerNorm and fp32 (x + add) -> 16-bit cast (memory_mode 'raw' / 'norm_y' building blocks), small and
    large launches (the small ones preload gamma / beta before the dependency wait)."""
    x, add = rnd(M, D, seed=15, scale=3.0) + 0.5, rnd(M, D, seed=16)
    g, b = 1 + 0.1 * rnd(D, seed=17), 0.1 * rnd(D, seed=18)
    x16 = x.to(dtype)
    out = ops.layernorm16(x16, g, b, 1e-6)
    assert out.dtype == dtype and rel_l2(out, torch.nn.functional.layer_norm(x16.float(), (D,), g, b, 1e-6)) < OUT_TOL[dtype]
    assert torch.equal(ops.cast16(x, dtype), x.to(dtype))
    assert torch.equal(ops.cast16(x, dtype, add=add), (x + add).to(dtype))
    out = ops.layernorm(x, g, b, 1e-6, out_dtype=dtype)
    assert rel_l2(out, torch.nn.functional.layer_norm(x, (D,), g, b, 1e-6)) < OUT_TOL[dtype]


def ref_attn(q, k, v, mask=None):
    s = (q.float() @ k.float().transpose(-1, -2)) * 0.125
    if mask is not None:
        s = s.masked_fill(~mask, float("-inf"))
    return torch.softmax(s, -1) @ v.float()


ATT_TOL = {torch.float16: 1.5e-3, torch.bfloat16: 8e-3}


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("B,H,N", [(1, 1, 128), (2, 2, 196), (1, 12, 768), (3, 16, 300)])
def test_self_attention(dtype, B, H, N):
    """Self-attention straight out of the fused [B*N, 3*H*64] qkv buffer (attention.py:94-97 layout)."""
    D = H * 64
    qkv = rnd(B * N, 3 * D, dtype=dtype, seed=19)
    out = ops.attention(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], B=B, H=H, Nq=N, Nk0=N)
    t = qkv.view(B, N, 3, H, 64).permute(2, 0, 3, 1, 4)
    ref = ref_attn(t[0], t[1], t[2]).permute(0, 2, 1, 3).reshape(B * N, D)
    assert rel_l2(out, ref) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("Nm,n,N", [(0, 2, 196), (392, 1, 196), (588, 3, 196), (1536, 2, 768), (100, 2, 50)])
def test_memory_cross_attention(dtype, Nm, n, N):
    """Memory cross-attention in update mode: keys = stored memory [B,cap,1536] (K|V, padding filled with
    NaN to prove rows beyond Nm are never consumed) + this step's new tokens, each view skipping its own
    segment (decoder.py:119-139, 304-317)."""
    B, H = 2, 12
    D = H * 64
    cap = Nm + 77
    mem = torch.full((B, cap, 2 * D), float("nan"), device="cuda", dtype=dtype)
    mem[:, :Nm] = rnd(B, Nm, 2 * D, dtype=dtype, seed=20)
    new = rnd(B, n * N, 2 * D, dtype=dtype, seed=21)
    q = rnd(B * n * N, D, dtype=dtype, seed=22)
    mem2 = mem.view(B * cap, 2 * D)
    new2 = new.view(B * n * N, 2 * D)
    use_skip = Nm > 0 or n > 1
    out = ops.attention(q, mem2[:, :D], mem2[:, D:], B=B * n, H=H, Nq=N, Nk0=Nm, kv_bstride0=cap,
                        k1=new2[:, :D], v1=new2[:, D:], Nk1=n * N, kv_bstride1=n * N, kv_group=n,
                        skip_lo=Nm, skip_step=N, skip_len=N if use_skip else 0)
    kv = torch.cat([mem[:, :Nm], new], 1)                                  # [B, Nk, 2D]
    Nk = kv.shape[1]
    k = kv[..., :D].view(B, 1, Nk, H, 64).expand(B, n, Nk, H, 64).reshape(B * n, Nk, H, 64).permute(0, 2, 1, 3)
    v = kv[..., D:].view(B, 1, Nk, H, 64).expand(B, n, Nk, H, 64).reshape(B * n, Nk, H, 64).permute(0, 2, 1, 3)
    mask = torch.ones(B * n, 1, 1, Nk, dtype=torch.bool, device="cuda")
    if use_skip:
        for j in range(B * n):
            mask[j, ..., Nm + (j % n) * N: Nm + (j % n + 1) * N] = False
    ref = ref_attn(q.view(B * n, N, H, 64).permute(0, 2, 1, 3), k, v, mask).permute(0, 2, 1, 3).reshape(B * n * N, D)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("cs", [1, 2])
@pytest.mark.parametrize("qt,splits", [(1, 1), (1, 3), (1, 16), (2, 1), (2, 2), (2, 7)])
def test_attention_kernel_variants(dtype, qt, splits, cs, monkeypatch):
    """Force each kernel configuration (1 or 2 query tiles per CTA, the 128-key score tile in 1 or 2 column slices per
    softmax pass, key-range splits + in-kernel merge) on a masked, two-segment, ragged problem and on a long-key problem
    with large score spread (exercises the lazy rescale)."""
    monkeypatch.setenv("M3R_ATTN_QT", str(qt))
    monkeypatch.setenv("M3R_ATTN_SPLITS", str(splits))
    monkeypatch.setenv("M3R_ATTN_CS", str(cs))
    B, H, n, N, Nm = 1, 3, 2, 300, 700
    D = H * 64
    mem = rnd(B, Nm, 2 * D, dtype=dtype, seed=30)
    new = rnd(B, n * N, 2 * D, dtype=dtype, seed=31)
    q = rnd(B * n * N, D, dtype=dtype, seed=32, scale=3.0)          # wide score range -> max refreshes
    out = ops.attention(q, mem.view(-1, 2 * D)[:, :D], mem.view(-1, 2 * D)[:, D:], B=B * n, H=H, Nq=N, Nk0=Nm,
                        k1=new.view(-1, 2 * D)[:, :D], v1=new.view(-1, 2 * D)[:, D:], Nk1=n * N, kv_group=n,
                        skip_lo=Nm, skip_step=N, skip_len=N)
    kv = torch.cat([mem, new], 1)
    Nk = kv.shape[1]
    k = kv[..., :D].view(B, 1, Nk, H, 64).expand(B, n, Nk, H, 64).reshape(B * n, Nk, H, 64).permute(0, 2, 1, 3)
    v = kv[..., D:].view(B, 1, Nk, H, 64).expand(B, n, Nk, H, 64).reshape(B * n, Nk, H, 64).permute(0, 2, 1, 3)
    mask = torch.ones(B * n, 1, 1, Nk, dtype=torch.bool, device="cuda")
    for j in range(B * n):
        mask[j, ..., Nm + (j % n) * N: Nm + (j % n + 1) * N] = False
    ref = ref_attn(q.view(B * n, N, H, 64).permute(0, 2, 1, 3), k, v, mask).permute(0, 2, 1, 3).reshape(B * n * N, D)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < ATT_TOL[dtype]
    # keys sorted so that the row max keeps growing tile after tile
    Nk2 = 2048
    kk = rnd(Nk2, 64, dtype=torch.float32, seed=33)
    kk = (kk * torch.linspace(0.2, 4.0, Nk2, device="cuda")[:, None]).to(dtype)
    vv = rnd(Nk2, 64, dtype=dtype, seed=34)
    qq = rnd(256, 64, dtype=dtype, seed=35, scale=2.0)
    out = ops.attention(qq, kk, vv, B=1, H=1, Nq=256, Nk0=Nk2)
    assert rel_l2(out, ref_attn(qq, kk, vv)) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
def test_render_cross_attention_long_memory(dtype):
    """Render mode: 4 views against a 20-view memory (Nmem = 15360), no mask, shared K/V (decoder.py:307-317)."""
    H, N, Nm, n = 12, 768, 15360, 4
    D = H * 64
    mem = rnd(Nm, 2 * D, dtype=dtype, seed=23)
    q = rnd(n * N, D, dtype=dtype, seed=24)
    out = ops.attention(q, mem[:, :D], mem[:, D:], B=n, H=H, Nq=N, Nk0=Nm, kv_group=n)
    k = mem[:, :D].view(1, Nm, H, 64).permute(0, 2, 1, 3)
    v = mem[:, D:].view(1, Nm, H, 64).permute(0, 2, 1, 3)
    ref = ref_attn(q.view(n, N, H, 64).permute(0, 2, 1, 3), k, v).permute(0, 2, 1, 3).reshape(n * N, D)
    assert rel_l2(out, ref) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
def test_patch_embed_path(dtype):
    V, H, W, Dm = 2, 48, 80, 128
    img = rnd(V, 3, H, W, seed=25).clamp(-1, 1)
    wconv = rnd(Dm, 3, 16, 16, seed=26, scale=768 ** -0.5)
    bias = rnd(Dm, seed=27)
    cols = ops.im2col16(img, dtype)
    out = ops.linear(cols, wconv.reshape(Dm, 768).to(dtype), bias, out_dtype=torch.float32)
    ref = torch.nn.functional.conv2d(img.to(dtype).float(), wconv.to(dtype).float(), bias, stride=16)
    ref = ref.flatten(2).transpose(1, 2).reshape(V * 15, Dm)
    assert rel_l2(out, ref) < 2e-5


def test_errors_are_loud():
    a = torch.zeros(4, 96, device="cuda", dtype=torch.float16)
    with pytest.raises(RuntimeError, match="multiple of 32 and K"):
        ops.linear(a, torch.zeros(64, 96, device="cuda", dtype=torch.float16))
    with pytest.raises(RuntimeError):
        ops.linear(a.cpu(), a.cpu())


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("B,H,Nq,Nk,shards", [(1, 12, 768, 7680, 4), (2, 3, 200, 1000, 3), (1, 12, 768, 76800, 8), (1, 2, 130, 300, 2)])
def test_attention_state_export_and_merge(dtype, B, H, Nq, Nk, shards):
    """Context-parallel building blocks on one GPU: the key range cut into `shards` pieces (uneven, one of them empty),
    every piece exported as an unnormalised attention state (with and without in-kernel key splits), the states merged
    (m3r_attn_merge) == attention over all keys."""
    D = H * 64
    q = rnd(B * Nq, D, dtype=dtype, seed=1)
    kv = rnd(B * Nk, 2 * D, dtype=dtype, seed=2)
    ref = ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk).float()
    cuts = sorted({0, Nk} | {int(Nk * f) for f in torch.linspace(0.13, 0.9, shards - 1).tolist()})
    states = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        kvs = kv.view(B, Nk, 2 * D)[:, lo:hi].contiguous().view(B * (hi - lo), 2 * D)
        states.append(ops.attention(q, kvs[:, :D], kvs[:, D:], B=B, H=H, Nq=Nq, Nk0=hi - lo, export=True))
    if len(states) < 8:
        states.insert(1, ops.attn_state_fill(B * Nq, H, q.device))         # a rank whose shard is empty
    got = ops.attn_merge(states, dtype).float()
    assert rel_l2(got, ref) < (6e-4 if dtype == torch.float16 else 5e-3)
    # a single state merges to plain attention
    one = ops.attn_merge([ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk, export=True)], dtype).float()
    assert rel_l2(one, ref) < (3e-4 if dtype == torch.float16 else 3e-3)


def test_peer_primitives_on_one_gpu():
    """m3r_peer_bcast / m3r_peer_signal / m3r_peer_wait with this GPU as its own only peer: data lands in every destination, the
    wait returns once the epoch is published (stream order), and a wait for an epoch that was already passed returns at once."""
    import ctypes as C
    from must3r_b200 import _lib
    lib = _lib.lib()
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    src = torch.randn(1 << 16, device="cuda")
    dsts = [torch.zeros_like(src) for _ in range(3)]
    arr = (C.c_void_p * 3)(*[d.data_ptr() for d in dsts])
    _lib.check(lib.m3r_peer_bcast(C.c_void_p(src.data_ptr()), arr, 3, src.numel() * 4, sp), "peer_bcast")
    flags = torch.zeros(8, dtype=torch.int32, device="cuda")
    slots = (C.c_void_p * 1)(flags.data_ptr() + 4 * 2)                     # "rank 2" publishes
    _lib.check(lib.m3r_peer_signal(slots, 1, 7, sp), "peer_signal")
    _lib.check(lib.m3r_peer_wait(C.c_void_p(flags.data_ptr()), 1 << 2, 7, sp), "peer_wait")
    _lib.check(lib.m3r_peer_wait(C.c_void_p(flags.data_ptr()), 1 << 2, 5, sp), "peer_wait")
    torch.cuda.synchronize()
    assert all(torch.equal(d, src) for d in dsts) and flags.tolist() == [0, 0, 7, 0, 0, 0, 0, 0]
