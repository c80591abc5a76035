"""m3r_attention, its exported state and m3r_attn_merge element by element against the float64 allowance of
tests/attention_ref.py, with guarded outputs and hostile masked keys.

- Every output is a column slice of a wider sentinel-filled buffer with pad rows below; nothing outside it may change.
- Q, K and V are views into wider buffers whose extra columns and kv_bstride gap rows are NaN.
- Keys in a skip range would win every softmax (K along the mean query direction) and carry V of +-4096.
- Launch hygiene: back-to-back launches on one and on two streams, across a reallocation of the split scratch, are
  bitwise equal to the same launches run alone; the 16384-unit limit of the split counters; argument errors.
Every case prints its worst err / allowance."""
import ctypes as C

import pytest
import torch

from attention_ref import (C3_CASES, CASES, HD, Case, bound, check, lse_allowance, make_inputs, off_by_4ulp, ref_args,
                           reference, swap_tile_edge)
from must3r_b200 import _lib

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
SENTINEL = 7.0
PAD = 64                                 # sentinel columns either side of an output and rows below it
GUARD = 16                               # sentinel rows before and after an exported state


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def stream_ptr(s=None):
    return C.c_void_p((s or torch.cuda.current_stream()).cuda_stream)


def attn_args(kw, dtype, out=None, exp=None):
    a = _lib.AttnArgs()
    a.Q, a.ldq = kw["q"].data_ptr(), kw["q"].stride(0)
    a.K0, a.V0, a.ldk0 = kw["k0"].data_ptr(), kw["v0"].data_ptr(), kw["k0"].stride(0)
    a.kv_bstride0, a.Nk0 = kw["kv_bstride0"], kw["Nk0"]
    if kw["Nk1"] > 0:
        a.K1, a.V1, a.ldk1 = kw["k1"].data_ptr(), kw["v1"].data_ptr(), kw["k1"].stride(0)
        a.kv_bstride1, a.Nk1 = kw["kv_bstride1"], kw["Nk1"]
    if out is not None:
        a.O, a.ldo = out.data_ptr(), out.stride(0)
    if exp is not None:
        a.export_o, a.export_ml = exp[0].data_ptr(), exp[1].data_ptr()
        a.ldo = kw["H"] * HD
    a.B, a.H, a.Nq, a.kv_group = kw["B"], kw["H"], kw["Nq"], kw["kv_group"]
    a.skip_lo, a.skip_step, a.skip_len = kw["skip_lo"], kw["skip_step"], kw["skip_len"]
    a.is_bf16 = int(dtype == torch.bfloat16)
    a.scale = kw["scale"]
    return a


def run(a, stream=None):
    _lib.check(_lib.lib().m3r_attention(C.byref(a), stream_ptr(stream)), "attention")


def out_buffer(rows, H, dtype):
    """Sentinel-filled [rows + PAD, H*64 + 2 PAD] buffer and the [rows, H*64] output view inside it (ldo > H*64)."""
    buf = torch.full((rows + PAD, H * HD + 2 * PAD), SENTINEL, device="cuda", dtype=dtype)
    return buf, buf[:rows, PAD:PAD + H * HD]


def untouched_out(buf, rows, H):
    m = torch.ones_like(buf, dtype=torch.bool)
    m[:rows, PAD:PAD + H * HD] = False
    return bool((buf[m] == SENTINEL).all())


def export_buffers(rows, H):
    """Sentinel-guarded export_o [rows, H*64] and export_ml [rows, H, 2] (GUARD rows before and after)."""
    ob = torch.full((rows + 2 * GUARD, H * HD), SENTINEL, device="cuda")
    mb = torch.full((rows + 2 * GUARD, H, 2), SENTINEL, device="cuda")
    return (ob, mb), (ob[GUARD:GUARD + rows], mb[GUARD:GUARD + rows])


def untouched_export(bufs, rows):
    return all(bool((b[:GUARD] == SENTINEL).all()) and bool((b[GUARD + rows:] == SENTINEL).all()) for b in bufs)


def force_splits(monkeypatch, s):
    if s is None:
        monkeypatch.delenv("M3R_ATTN_SPLITS", raising=False)
    else:
        monkeypatch.setenv("M3R_ATTN_SPLITS", str(s))


def solve(c, dtype, monkeypatch, seed=0):
    """Run case c into a guarded output; check the guard, finiteness and every element.  Returns (out, ref, bound)."""
    kw, keep = make_inputs(c, dtype, "cuda", seed=seed)
    force_splits(monkeypatch, c.splits)
    rows = c.B * c.Nq
    buf, out = out_buffer(rows, c.H, dtype)
    run(attn_args(kw, dtype, out=out))
    torch.cuda.synchronize()
    assert untouched_out(buf, rows, c.H), f"{c.name}: a store landed outside the output"
    r = reference(kw["q"], kw["k0"], kw["v0"], **ref_args(kw))
    bnd = bound(r, dtype)
    assert bool(torch.isfinite(out).all()), c.name
    worst = check(out, r, bnd, c.name)
    print(f"\n[attn-contract] {c.name} {str(dtype)[6:]}: worst err/bound {worst:.3f}")
    return out, r, bnd, kw, keep


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_case_matrix(c, dtype, monkeypatch):
    solve(c, dtype, monkeypatch)


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c", C3_CASES, ids=[c.name for c in C3_CASES])
def test_c3_shapes(c, dtype, monkeypatch):
    out, r, bnd, _, _ = solve(c, dtype, monkeypatch)
    if c.name == "c3_render":
        # the allowance still sees one element 4 ulp off, and the rows on either side of a 64-row tile edge swapped
        for bad in (off_by_4ulp(out, r, bnd), swap_tile_edge(out)):
            with pytest.raises(AssertionError):
                check(bad, r, bnd, "mutated")


EXPORT_CASES = [c for c in CASES if c.name in ("nk1000_s1", "nk1000_s7", "skip_empty_splits32", "seg0_in_tile",
                                                "grow_split3", "update_qkv5", "qscale40", "nk1_sNone")]


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c", EXPORT_CASES, ids=[c.name for c in EXPORT_CASES])
def test_export_state(c, dtype, monkeypatch):
    """export_o / export_ml with and without key splits: o / l passes the allowance, m + log2(l) is the log-sum-exp."""
    kw, keep = make_inputs(c, dtype, "cuda")
    force_splits(monkeypatch, c.splits)
    rows = c.B * c.Nq
    bufs, (eo, eml) = export_buffers(rows, c.H)
    run(attn_args(kw, dtype, exp=(eo, eml)))
    torch.cuda.synchronize()
    assert untouched_export(bufs, rows), f"{c.name}: an exported store landed outside the state"
    r = reference(kw["q"], kw["k0"], kw["v0"], **ref_args(kw))
    m, l = eml[..., 0].double(), eml[..., 1].double()
    assert bool((l > 0).all()) and bool(torch.isfinite(m).all())
    o = eo.double().view(rows, c.H, HD) / l[..., None]
    worst = check(o.view(rows, c.H * HD), r, bound(r, dtype), c.name + " export")
    dl = (m + torch.log2(l) - r.lse2).abs()
    lse = float((dl / lse_allowance(r)).max())
    print(f"\n[attn-contract] export {c.name} {str(dtype)[6:]}: worst err/bound {worst:.3f}, lse {lse:.3f}")
    assert lse <= 1, (c.name, float(dl.max()))


def test_empty_state_fill():
    rows, H = 300, 3
    bufs, (eo, eml) = export_buffers(rows, H)
    _lib.check(_lib.lib().m3r_attn_state_fill(p(eo), p(eml), rows, H, stream_ptr()), "attn_state_fill")
    torch.cuda.synchronize()
    assert untouched_export(bufs, rows)
    assert bool((eo == 0).all()) and bool((eml[..., 0] == -float("inf")).all()) and bool((eml[..., 1] == 0).all())


def shard_problem(dtype, n_keys, offsets, seed):
    """Queries and the union of key shards whose score maxima are shifted apart: column 0 of every head is qc (per row:
    4, -4, 0, 0.5) in Q and off_k in shard k's K, so shard k's scores move by 0.125 qc off_k (off 190 at qc 4: 137 log2
    units; off 14: 10)."""
    B, H, Nq = 2, 2, 130
    D = H * HD
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B * Nq, H, HD, generator=g)
    q[..., 0] = torch.tensor([4.0, -4.0, 0.0, 0.5]).repeat(B * Nq // 4 + 1)[:B * Nq, None]
    ks, vs = [], []
    for n, off in zip(n_keys, offsets):
        k = torch.randn(B, n, H, HD, generator=g)
        k[..., 0] = off
        ks.append(k)
        vs.append(torch.randn(B, n, H, HD, generator=g))
    q = q.reshape(B * Nq, D).to(dtype).cuda()
    ks = [k.reshape(B, n, D).to(dtype).cuda() for k, n in zip(ks, n_keys)]
    vs = [v.reshape(B, n, D).to(dtype).cuda() for v, n in zip(vs, n_keys)]
    return B, H, Nq, q, ks, vs


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("layout", [
    ([300], [0.0], [None]),
    ([300, 0], [0.0, 0.0], [2, None]),
    ([200, 1, 257], [0.0, 14.0, -14.0], [3, None, 2]),
    ([129, 0, 300, 64, 500], [190.0, 0.0, -190.0, 14.0, 0.0], [None, None, 7, 1, 3]),
    ([100, 300, 0, 128, 255, 0, 1000, 77], [0.0, 14.0, 0.0, -14.0, 190.0, 0.0, -190.0, 0.0], [1, 2, None, 3, 32, None, 7, None]),
], ids=["1", "2_fill", "3", "5_fill", "8_fill"])
def test_merge_disjoint_shards(dtype, layout, monkeypatch):
    """1..8 states of disjoint key shards (n = 0: an attn_state_fill state) merged into a guarded column slice equal the
    float64 softmax over the union of the shards."""
    n_keys, offsets, splits = layout
    B, H, Nq, q, ks, vs = shard_problem(dtype, n_keys, offsets, seed=len(n_keys))
    rows = B * Nq
    states = []
    for k, v, sp in zip(ks, vs, splits):
        n = k.shape[1]
        e_o = torch.empty(rows, H * HD, device="cuda")
        e_ml = torch.empty(rows, H, 2, device="cuda")
        if n == 0:
            _lib.check(_lib.lib().m3r_attn_state_fill(p(e_o), p(e_ml), rows, H, stream_ptr()), "attn_state_fill")
        else:
            force_splits(monkeypatch, sp)
            kv = dict(q=q, k0=k.view(B * n, -1), v0=v.view(B * n, -1), B=B, H=H, Nq=Nq, Nk0=n, kv_bstride0=n, Nk1=0,
                      kv_group=1, skip_lo=0, skip_step=0, skip_len=0, scale=0.125)
            run(attn_args(kv, dtype, exp=(e_o, e_ml)))
        states.append((e_o, e_ml))
    buf, out = out_buffer(rows, H, dtype)
    po = (C.c_void_p * len(states))(*[o.data_ptr() for o, _ in states])
    pml = (C.c_void_p * len(states))(*[ml.data_ptr() for _, ml in states])
    _lib.check(_lib.lib().m3r_attn_merge(po, pml, len(states), rows, H, p(out), out.stride(0),
                                         int(dtype == torch.bfloat16), stream_ptr()), "attn_merge")
    torch.cuda.synchronize()
    assert untouched_out(buf, rows, H), "a merged store landed outside the output"
    ku = torch.cat(ks, 1)
    vu = torch.cat(vs, 1)
    nk = ku.shape[1]
    r = reference(q, ku.reshape(B * nk, -1), vu.reshape(B * nk, -1), B=B, H=H, Nq=Nq, Nk0=nk, kv_bstride0=nk)
    worst = check(out, r, bound(r, dtype), "merge")
    print(f"\n[attn-contract] merge {len(states)} states {str(dtype)[6:]}: worst err/bound {worst:.3f}")


# ------------------------------------------------------------------------------------------------ launch hygiene
SEQ = [  # (case, forced splits, export)
    (Case("h_a", B=2, H=2, Nq=100, Nk0=300, Nk1=200, skip=(250, 0, 100)), 3, False),
    (Case("h_b", B=3, H=1, Nq=65, Nk0=1000), 7, True),
    (Case("h_c", B=2, H=2, Nq=129, Nk0=257), 1, False),
    (Case("h_d", B=4, H=2, Nq=100, Nk0=600, kv_group=2, gap0=11), None, False),
    (Case("h_big", B=1, H=16, Nq=4096, Nk0=1024), 8, False),          # grows the split scratch mid-sequence
    (Case("h_e", B=2, H=2, Nq=100, Nk0=300, Nk1=200, skip=(250, 0, 100)), 2, True),
    (Case("h_f", B=2, H=2, Nq=193, Nk0=2000), 32, False),
    (Case("h_g", B=2, H=2, Nq=64, Nk0=128), None, True),
    (Case("h_h", B=3, H=1, Nq=65, Nk0=1000), 3, False),
    (Case("h_i", B=2, H=2, Nq=129, Nk0=257), 2, True),
]


def hygiene_launch(kw, c, dtype, export, stream, monkeypatch, splits):
    force_splits(monkeypatch, splits)
    rows = c.B * c.Nq
    if export:
        res = (torch.empty(rows, c.H * HD, device="cuda"), torch.empty(rows, c.H, 2, device="cuda"))
        run(attn_args(kw, dtype, exp=res), stream)
    else:
        res = (torch.empty(rows, c.H * HD, device="cuda", dtype=dtype),)
        run(attn_args(kw, dtype, out=res[0]), stream)
    return res


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("n_streams", [1, 2])
def test_back_to_back_launches_are_bitwise_stable(dtype, n_streams, monkeypatch):
    """About 10 launches without syncs on one fresh stream (or alternating over two), cycling shapes, split counts and
    export; the split scratch reallocates in the middle.  Each result equals the same launch run alone, bit for bit."""
    probs = [make_inputs(c, dtype, "cuda", seed=i) for i, (c, _, _) in enumerate(SEQ)]
    alone = []
    for (c, sp, ex), (kw, _) in zip(SEQ, probs):
        alone.append(hygiene_launch(kw, c, dtype, ex, None, monkeypatch, sp))
        torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(n_streams)]
    for s in streams:
        s.wait_stream(torch.cuda.current_stream())
    got = []
    for i, ((c, sp, ex), (kw, _)) in enumerate(zip(SEQ, probs)):
        s = streams[i % n_streams]
        with torch.cuda.stream(s):
            got.append(hygiene_launch(kw, c, dtype, ex, s, monkeypatch, sp))
    torch.cuda.synchronize()
    for (c, _, _), a, g in zip(SEQ, alone, got):
        for x, y in zip(a, g):
            assert torch.equal(x, y), c.name


# 16384 (batch, head, 64-row query tile) units is the size of the split counter table
LIMIT = Case("limit_16384", B=4, H=16, Nq=16374, Nk0=300)                  # 4 x 16 x 256
OVER = Case("limit_16385", B=5, H=29, Nq=7169, Nk0=300)                    # 5 x 29 x 113


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
def test_counter_table_limit(dtype, monkeypatch):
    from dataclasses import replace
    solve(replace(LIMIT, splits=2), dtype, monkeypatch)
    kw, keep = make_inputs(OVER, dtype, "cuda")
    out = torch.empty(OVER.B * OVER.Nq, OVER.H * HD, device="cuda", dtype=dtype)
    force_splits(monkeypatch, 2)
    with pytest.raises(RuntimeError, match="too many"):
        run(attn_args(kw, dtype, out=out))
    del kw, keep, out
    solve(OVER, dtype, monkeypatch)                                        # default: runs unsplit


def test_argument_errors(monkeypatch):
    dtype = torch.float16
    c = Case("err", B=4, H=2, Nq=64, Nk0=200, Nk1=100)
    kw, keep = make_inputs(c, dtype, "cuda")
    out = torch.empty(c.B * c.Nq, c.H * HD, device="cuda", dtype=dtype)
    monkeypatch.delenv("M3R_ATTN_SPLITS", raising=False)

    def expect(msg, a):
        with pytest.raises(RuntimeError, match=msg):
            run(a)

    expect("skip range covers every key", attn_args(dict(kw, skip_lo=0, skip_step=0, skip_len=300), dtype, out=out))
    expect("must be a multiple of kv_group", attn_args(dict(kw, kv_group=3), dtype, out=out))
    a = attn_args(kw, dtype, out=out)
    a.ldq += 4
    expect("multiples of 8", a)
    a = attn_args(kw, dtype, out=out)
    e = torch.empty(c.B * c.Nq, c.H * HD, device="cuda")
    a.export_o = e.data_ptr()
    expect("export_o and export_ml go together", a)
    torch.cuda.synchronize()
