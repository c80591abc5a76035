"""m3r_gemm, m3r_gemm_grouped and the LayerNorm kernels element by element against the float64 allowance of
tests/gemm_ref.py, with guarded outputs and NaN-padded operands.

- Every output is a view into a sentinel-filled buffer: rows past M, columns on both sides, ldc > N (and ldn > N for
  norm_out); nothing outside it may change.
- A has NaN columns past K (lda > K) and NaN rows after M (after groups * M); W is a slice of a NaN matrix with NaN rows
  around and between the groups; bias, row bias and residual have NaN past their used entries; the RoPE table has NaN
  rows past rope_period.  A kernel that reads any of them produces a NaN, which fails the check.
- Plain launches at every tile width forced through M3R_GEMM_BN, one wave and several tiles per CTA on thread stores and
  on TMA stores, K on both sides of the operand ring depth, with and without w_static; the model's own call sites; the
  grouped GEMM with the memory append's row remap, peers and max_ctas; the LayerNorm-emitting kernels with and without
  split-K, back to back and across two streams; the LayerNorm family.
Every case prints its worst err / allowance."""
import ctypes as C

import pytest
import torch

from gemm_ref import (EMIT_CASES, PLAIN_CASES, U32, Case, check, emit_plan, layernorm, make_operands, out_bound,
                      ref_kwargs, reference)
from must3r_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
SENTINEL = 7.0
PAD = 64                                  # sentinel columns on either side of an output, and rows below it
EXTRA_LD = 32                             # ldc - N beyond the right-hand pad
EPS = 1e-6


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stream_ptr(s=None):
    return C.c_void_p((s or torch.cuda.current_stream()).cuda_stream)


def out_buffer(rows, N, dtype):
    buf = torch.full((rows + PAD, N + 2 * PAD + EXTRA_LD), SENTINEL, device="cuda", dtype=dtype)
    return buf, buf[:rows, PAD:PAD + N]


def untouched(buf, rows, N):
    m = torch.ones_like(buf, dtype=torch.bool)
    m[rows, PAD:PAD + N] = False
    return bool((buf[m] == SENTINEL).all())


def gemm_args(c: Case, d, dtype, out, norm_out=None):
    a = _lib.GemmArgs()
    a.A, a.lda = d["a"].data_ptr(), d["a"].stride(0)
    a.W, a.ldw = d["w"].data_ptr(), d["w"].stride(0)
    a.M, a.N, a.K = c.M, c.N, c.K
    a.is_bf16 = int(dtype == torch.bfloat16)
    a.bias = d["bias"].data_ptr() if c.bias else None
    a.act = int(c.gelu)
    if c.res == "sep":
        a.residual, a.ldr = d["residual"].data_ptr(), d["residual"].stride(0)
    elif c.res == "inplace":
        out.copy_(d["residual"])
        a.residual, a.ldr = out.data_ptr(), out.stride(0)
    if c.rb_first >= 0:
        a.rowbias, a.rb_period, a.rb_first = d["rowbias"].data_ptr(), c.rb_period, c.rb_first
    if c.rope_cols:
        a.rope_tab, a.rope_cols, a.rope_period = d["rope_tab"].data_ptr(), c.rope_cols, c.rope_period
    a.out, a.ldc = out.data_ptr(), out.stride(0)
    a.out_dtype = 0 if out.dtype == torch.float32 else 1
    a.w_static = int(c.w_static)
    if norm_out is not None:
        a.norm_out, a.ldn, a.norm_eps = norm_out.data_ptr(), norm_out.stride(0), EPS
    return a


def run(a, stream=None):
    _lib.check(_lib.lib().m3r_gemm(C.byref(a), stream_ptr(stream)), "gemm")


def report(group, c, dtype, worst):
    print(f"\n[gemm-contract] {group} {c.name} {str(dtype)[6:]}: worst err/bound {worst:.3f}")


def solve_plain(c: Case, dtype, monkeypatch, group):
    if c.bn is None:
        monkeypatch.delenv("M3R_GEMM_BN", raising=False)
    else:
        assert c.N % c.bn == 0, "the forced tile width must apply"
        monkeypatch.setenv("M3R_GEMM_BN", str(c.bn))
    d = make_operands(c, dtype, "cuda")
    od = dtype if c.out16 else torch.float32
    buf, out = out_buffer(c.M, c.N, od)
    run(gemm_args(c, d, dtype, out))
    torch.cuda.synchronize()
    assert untouched(buf, slice(0, c.M), c.N), f"{c.name}: a store landed outside the output"
    r = reference(d["a"], d["w"], **ref_kwargs(c, d))
    worst = check(out, r.val, out_bound(r.val, r.err, od), c.name, M=c.M, bn=c.bn)
    report(group, c, dtype, worst)


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c", PLAIN_CASES, ids=[c.name for c in PLAIN_CASES])
def test_plain_matrix(c, dtype, monkeypatch):
    solve_plain(c, dtype, monkeypatch, "plain")


# ------------------------------------------------------------------------------------------------ LayerNorm-emitting
def solve_emit(c: Case, dtype, stream=None, check_it=True):
    bn, ks = emit_plan(c.M, c.N, c.K, sms())
    assert bn is not None, c.name
    d = make_operands(c, dtype, "cuda")
    obuf, out = out_buffer(c.M, c.N, torch.float32)
    nbuf, nout = out_buffer(c.M, c.N, dtype)
    run(gemm_args(c, d, dtype, out, norm_out=nout), stream)
    if not check_it:
        return d, out, nout
    torch.cuda.synchronize()
    assert untouched(obuf, slice(0, c.M), c.N) and untouched(nbuf, slice(0, c.M), c.N), f"{c.name}: stray store"
    r = reference(d["a"], d["w"], **ref_kwargs(c, d, ks))
    w1 = check(out, r.val, out_bound(r.val, r.err, torch.float32), c.name, M=c.M, bn=bn)
    nv, ne = layernorm(r.val, r.err, EPS, "emit")
    w2 = check(nout, nv, out_bound(nv, ne, dtype), c.name + " norm_out", M=c.M, bn=bn)
    print(f"\n[gemm-contract] emit {c.name} (BN {bn}, split {ks}) {str(dtype)[6:]}: worst err/bound out {w1:.3f} "
          f"norm_out {w2:.3f}")
    return d, out, nout


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c", EMIT_CASES, ids=[c.name for c in EMIT_CASES])
def test_emit(c, dtype):
    torch.cuda.synchronize()
    solve_emit(c, dtype)


EMIT_SEQ = [Case("s_split", 196, 768, 3072, res="sep"), Case("s_plain", 196, 768, 768, res="inplace"),
            Case("s_split2", 263, 768, 2048, res="inplace"), Case("s_bn128", 1500, 768, 768, res="sep"),
            Case("s_split3", 130, 768, 3072, res=""), Case("s_plain2", 640, 768, 768, res="sep", rb_first=100)]


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("n_streams", [1, 2])
def test_emit_back_to_back(dtype, n_streams):
    """Split-K and unsplit emitting launches alternate without syncs on one stream (the counters and kflag must re-arm),
    or on two streams ordered by wait_stream; each result equals the same launch run alone, bit for bit."""
    alone = []
    for c in EMIT_SEQ:
        torch.cuda.synchronize()
        _, out, nout = solve_emit(c, dtype, check_it=False)
        torch.cuda.synchronize()
        alone.append((out.clone(), nout.clone()))
    streams = [torch.cuda.Stream() for _ in range(n_streams)]
    streams[0].wait_stream(torch.cuda.current_stream())
    got = []
    for i, c in enumerate(EMIT_SEQ):
        s = streams[(i * n_streams) // len(EMIT_SEQ)]                    # first half on stream 0, second on stream 1
        if s is not streams[0] and i == len(EMIT_SEQ) // 2:
            s.wait_stream(streams[0])
        with torch.cuda.stream(s):
            _, out, nout = solve_emit(c, dtype, stream=s, check_it=False)
            got.append((out, nout))
    torch.cuda.synchronize()
    for c, a, g in zip(EMIT_SEQ, alone, got):
        assert torch.equal(a[0], g[0]) and torch.equal(a[1], g[1]), c.name


def test_emit_argument_errors():
    c = Case("err", 130, 768, 768, res="")
    d = make_operands(c, torch.float16, "cuda")
    out = torch.empty(c.M, c.N, device="cuda")
    nout = torch.empty(c.M, c.N, device="cuda", dtype=torch.float16)
    a = gemm_args(c, d, torch.float16, out, norm_out=nout)
    a.rows_per_batch, a.batch_stride_rows = 64, 100
    with pytest.raises(RuntimeError, match="rows_per_batch"):
        run(a)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ model call sites
def _sites():
    cs = []
    for T in (196, 768):
        for V in (1, 4):
            M = T * V
            cs += [Case(f"enc_qkv_T{T}_V{V}", M, 3072, 1024, rope_cols=2048, rope_period=T),
                   Case(f"enc_proj_T{T}_V{V}", M, 1024, 1024, out16=False, res="inplace"),
                   Case(f"enc_fc1_T{T}_V{V}", M, 4096, 1024, gelu=True),
                   Case(f"enc_fc2_T{T}_V{V}", M, 1024, 4096, out16=False, res="inplace"),
                   Case(f"dec_qkvkv_T{T}_V{V}", M, 3840, 768, rope_cols=1536, rope_period=M, w_static=True),
                   Case(f"dec_kv_T{T}_V{V}", M, 1536, 768, w_static=True),
                   Case(f"dec_q_T{T}_V{V}", M, 768, 768, w_static=True),
                   Case(f"dec_head_T{T}_V{V}", M, 1792, 768, out16=False),
                   Case(f"dec_cproj_T{T}_V{V}", M, 768, 768, res="inplace", emit=True),
                   Case(f"dec_fc2_T{T}_V{V}", M, 768, 3072, res="inplace", emit=True),
                   Case(f"dec_embed_T{T}_V{V}", M, 768, 1024, res="", rb_first=T, rb_period=M, emit=True)]
    return cs


SITES = _sites()


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c", SITES, ids=[c.name for c in SITES])
def test_model_call_sites(c, dtype, monkeypatch):
    if not c.emit:
        solve_plain(c, dtype, monkeypatch, "site")
        return
    if emit_plan(c.M, c.N, c.K, sms())[0] is None:
        pytest.skip("more than one wave: the model normalises with m3r_normalize16 here")
    torch.cuda.synchronize()
    solve_emit(c, dtype)


# ------------------------------------------------------------------------------------------------ grouped
GROUPED = [  # (name, G, M, N, K, rows_per_batch, batch_stride_rows, peers, max_ctas, out16)
    ("g1", 1, 300, 256, 128, 0, 0, 0, 0, True),
    ("g3_f32", 3, 300, 256, 128, 0, 0, 0, 0, False),
    ("g12_multi_peer", 12, 1499, 1536, 128, 0, 0, 1, 0, True),
    ("g16_remap_peers_32ctas", 16, 196, 1536, 768, 100, 130, 2, 32, True),
    ("g12_append_few_ctas", 12, 392, 1536, 768, 196, 300, 1, 7, True),
    ("g3_remap_in_tile", 3, 129, 512, 256, 50, 64, 0, 5, True),
]


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", GROUPED, ids=[g[0] for g in GROUPED])
def test_grouped(case, dtype):
    name, G, M, N, K, rpb, stride, n_peers, max_ctas, out16 = case
    c = Case(name, M, N, K, groups=G)
    d = make_operands(c, dtype, "cuda", pad_a_cols=False)
    wg = d["w_group_rows"]
    a = d["a"].view(G, M, K)
    w = d["w"].as_strided((G, N, K), (wg * K, K, 1))
    bias = d["bias"].as_strided((G, N), (wg, 1))
    od = dtype if out16 else torch.float32
    rows = torch.arange(M, device="cuda")
    dest = (rows // rpb) * stride + rows % rpb if rpb > 0 else rows
    R = int(dest.max()) + 1
    bufs = [out_buffer(R, N, od) for _ in range(G)]
    peers = [[out_buffer(R, N, od) for _ in range(n_peers)] for _ in range(G)]
    ops.linear_grouped(a, w, bias, [o for _, o in bufs],
                       peer_ptrs=[[o.data_ptr() for _, o in pg] for pg in peers] if n_peers else None,
                       rows_per_batch=rpb, batch_stride_rows=stride, max_ctas=max_ctas)
    torch.cuda.synchronize()
    for g in range(G):
        assert untouched(bufs[g][0], dest, N), f"{name}: group {g}: a store landed outside its rows"
        for pb, _ in peers[g]:
            assert torch.equal(pb, bufs[g][0]), f"{name}: group {g}: a peer buffer differs from the output"
    got = torch.cat([o[dest] for _, o in bufs])
    r = reference(d["a"], d["w"], **ref_kwargs(c, d))
    worst = check(got, r.val, out_bound(r.val, r.err, od), name, M=M, bn=None)
    report("grouped", c, dtype, worst)


# ------------------------------------------------------------------------------------------------ LayerNorm family
LN_D = [100, 128, 768, 1024, 1280, 2048]
LN_M = [1, 4096, 4097]
LN_FNS = ["layernorm_f32", "layernorm_16", "normalize16", "layernorm16", "add_cast16"]
LN_CASES = [(f"{LN_FNS[(i + j) % len(LN_FNS)]}_D{D}_M{M}", LN_FNS[(i + j) % len(LN_FNS)], D, M)
            for i, D in enumerate(LN_D) for j, M in enumerate(LN_M)]


def ln_inputs(D, M, seed):
    """x [M, D] fp32 inside a NaN buffer (ldx = D + 12): unit-variance rows, every third row offset by 200, one outlier
    channel; add [7, D] (the period) inside a NaN buffer; gamma / beta."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, D, generator=g) * 2.0
    x[::3] += 200.0
    x[:, D // 2] *= 30.0
    xb = torch.full((M + 8, D + 12), float("nan"))
    xb[:M, :D] = x
    ab = torch.full((8, D + 4), float("nan"))
    ab[:7, :D] = torch.randn(7, D, generator=g)
    gamma = torch.cat([torch.randn(D, generator=g) * 0.5 + 1, torch.full((4,), float("nan"))])
    beta = torch.cat([torch.randn(D, generator=g) * 0.1, torch.full((4,), float("nan"))])
    xb, ab, gamma, beta = xb.cuda(), ab.cuda(), gamma.cuda(), beta.cuda()
    return xb, xb[:M, :D], ab, ab[:7, :D], gamma, beta


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", LN_CASES, ids=[c[0] for c in LN_CASES])
def test_layernorm_family(case, dtype):
    name, fn, D, M = case
    xb, x, ab, add, gamma, beta = ln_inputs(D, M, seed=D + M)
    L, P = _lib.lib(), lambda t: C.c_void_p(t.data_ptr())               # noqa: E731
    bf = int(dtype == torch.bfloat16)
    od = torch.float32 if fn == "layernorm_f32" else dtype
    buf, out = out_buffer(M, D, od)
    x64 = x.double()
    e = torch.zeros_like(x64)
    if fn in ("layernorm_f32", "layernorm_16"):
        rc = L.m3r_layernorm(P(x), x.stride(0), None, 0, P(gamma), P(beta), EPS, M, D, P(out), out.stride(0),
                             int(od != torch.float32), bf, stream_ptr())
        val, err = layernorm(x64, e, EPS, "warp", gamma, beta)
    elif fn == "normalize16":
        add_rows = M // 2 + 1                                              # rows at and past it get no add
        rc = L.m3r_normalize16(P(x), x.stride(0), P(add), add.stride(0), add_rows, 7, EPS, M, D, P(out), out.stride(0),
                               bf, stream_ptr())
        on = (torch.arange(M, device="cuda") < add_rows)[:, None]
        s = x64 + add.double()[torch.arange(M, device="cuda") % 7]
        x64 = torch.where(on, s, x64)
        e = torch.where(on, U32 * s.abs(), e)
        val, err = layernorm(x64, e, EPS, "warp")
    elif fn == "layernorm16":
        xb16 = torch.full((M + 8, D + 12), float("nan"), device="cuda", dtype=dtype)
        xb16[:M, :D] = x.to(dtype)
        x16 = xb16[:M, :D]
        rc = L.m3r_layernorm16(P(x16), x16.stride(0), P(gamma), P(beta), EPS, M, D, P(out), out.stride(0), bf,
                               stream_ptr())
        val, err = layernorm(x16.double(), e, EPS, "warp", gamma, beta)
    else:
        addf = torch.full((M + 8, D + 4), float("nan"), device="cuda")
        addf[:M, :D] = torch.randn(M, D, device="cuda")
        av = addf[:M, :D]
        rc = L.m3r_add_cast16(P(x), x.stride(0), P(av), av.stride(0), M, D, P(out), out.stride(0), bf, stream_ptr())
        val = x64 + av.double()
        err = U32 * val.abs()
    assert rc == 0, L.m3r_last_error().decode()
    torch.cuda.synchronize()
    assert untouched(buf, slice(0, M), D), f"{name}: a store landed outside the output"
    worst = check(out, val, out_bound(val, err, od), name)
    print(f"\n[gemm-contract] layernorm {name} {str(dtype)[6:]}: worst err/bound {worst:.3f}")
