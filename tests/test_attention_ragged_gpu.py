"""m3r_attention_ragged (per-batch segment-0 lengths) element by element against the float64 allowance of
tests/attention_ref.py, with the guarded, sentinel-filled outputs of test_attention_contract_gpu.py.

- Each K/V batch's reference is computed over its own keys only: segment 0 rows [0, len_b), then segment 1.
- Every segment-0 row at or past a batch's length is overwritten with NaN, +inf and -inf: no output bit may change.
- Equal lengths give bitwise the result of m3r_attention with the same plan.
Every case prints its worst err / allowance."""
import ctypes as C

import pytest
import torch

from attention_ref import Case, bound, check, make_inputs, reference
from must3r_b200 import _lib
from test_attention_contract_gpu import attn_args, force_splits, out_buffer, run, stream_ptr, untouched_out

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]

# (case, segment-0 length of every K/V batch); the skip range, if any, lies inside segment 1 (global index Nk0 + j)
RAGGED = [
    (Case("len1_127_128_129", B=4, H=2, Nq=100, Nk0=300, splits=1), [1, 127, 128, 129]),
    (Case("len_edges_split3", B=4, H=2, Nq=65, Nk0=300, splits=3), [129, 1, 128, 127]),
    (Case("len_many_splits", B=3, H=2, Nq=130, Nk0=2000, splits=7), [2000, 1500, 1001]),
    (Case("len_auto_splits", B=3, H=12, Nq=100, Nk0=3000), [3000, 700, 1]),
    (Case("one_far_short", B=2, H=2, Nq=129, Nk0=4096, splits=8), [4096, 5]),
    (Case("short_32_splits", B=2, H=2, Nq=64, Nk0=4096, splits=32), [3, 4096]),
    (Case("group2_seg1", B=4, H=2, Nq=100, Nk0=600, Nk1=200, kv_group=2, splits=3), [600, 130]),
    (Case("group2_seg1_skip", B=4, H=2, Nq=100, Nk0=600, Nk1=200, kv_group=2, skip=(600, 100, 100), splits=3),
     [1, 600]),
    (Case("group3_no_seg1", B=6, H=2, Nq=70, Nk0=500, kv_group=3, splits=2), [257, 500]),
    (Case("zero_len_seg1", B=2, H=2, Nq=100, Nk0=300, Nk1=150, splits=2), [0, 300]),
    (Case("update_qkv5", B=4, H=12, Nq=100, Nk0=900, Nk1=100, kv_group=1, skip=(900, 0, 100), gap0=33,
          layout="qkv5", splits=3), [900, 255, 256, 1]),
]


def lengths_tensor(lens):
    return torch.tensor(lens, dtype=torch.int32, device="cuda")


def run_ragged(a, nk0, stream=None):
    _lib.check(_lib.lib().m3r_attention_ragged(C.byref(a), C.c_void_p(nk0.data_ptr()), stream_ptr(stream)),
               "attention_ragged")


def ragged_reference(kw, lens):
    """The reference of each K/V batch over its own keys, stacked in query order."""
    G, Nq, Nk0 = kw["kv_group"], kw["Nq"], kw["Nk0"]
    parts = []
    for kvb, n in enumerate(lens):
        q = kw["q"][kvb * G * Nq:(kvb + 1) * G * Nq]
        r0 = kvb * kw["kv_bstride0"]
        k0, v0 = kw["k0"][r0:r0 + max(n, 1)], kw["v0"][r0:r0 + max(n, 1)]
        k1 = v1 = None
        if kw["Nk1"] > 0:
            r1 = kvb * kw["kv_bstride1"]
            k1, v1 = kw["k1"][r1:r1 + kw["Nk1"]], kw["v1"][r1:r1 + kw["Nk1"]]
        lo = kw["skip_lo"]
        if kw["skip_len"] > 0:
            assert lo >= Nk0, "the test's skip ranges lie in segment 1"
            lo = lo - Nk0 + n
        parts.append(reference(q, k0, v0, k1, v1, B=G, H=kw["H"], Nq=Nq, Nk0=n, kv_bstride0=0, Nk1=kw["Nk1"],
                               kv_bstride1=0, kv_group=G, skip_lo=lo, skip_step=kw["skip_step"],
                               skip_len=kw["skip_len"], scale=kw["scale"]))
    r = parts[0]
    for f in ("out", "pv2", "e_v", "v2", "lse2", "e_l", "n_add"):
        setattr(r, f, torch.cat([getattr(p, f) for p in parts]))
    r.B = kw["B"]
    return r


def poison_tails(kw, lens, mode):
    """Overwrite segment-0 rows [len_b, Nk0) of every K/V batch: 'nan' = NaN / +inf / -inf in turn, 'rand' = finite."""
    D = kw["H"] * 64
    g = torch.Generator(device="cuda").manual_seed(11)
    for kvb, n in enumerate(lens):
        r0 = kvb * kw["kv_bstride0"]
        rows = kw["Nk0"] - n
        if rows <= 0:
            continue
        for t in (kw["k0"], kw["v0"]):
            blk = t[r0 + n:r0 + kw["Nk0"], :D]
            if mode == "rand":
                blk.copy_(torch.randn(blk.shape, generator=g, device="cuda") * 50)
            else:
                vals = torch.tensor([float("nan"), float("inf"), float("-inf")], device="cuda", dtype=t.dtype)
                idx = torch.arange(blk.numel(), device="cuda") % 3
                blk.copy_(vals[idx].view(blk.shape))


def solve(c, lens, dtype, monkeypatch, poison="nan"):
    kw, keep = make_inputs(c, dtype, "cuda", seed=1)
    force_splits(monkeypatch, c.splits)
    poison_tails(kw, lens, poison)
    rows = c.B * c.Nq
    buf, out = out_buffer(rows, c.H, dtype)
    nk0 = lengths_tensor(lens)
    run_ragged(attn_args(kw, dtype, out=out), nk0)
    torch.cuda.synchronize()
    assert untouched_out(buf, rows, c.H), f"{c.name}: a store landed outside the output"
    return out.clone(), kw, keep


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("c,lens", RAGGED, ids=[c.name for c, _ in RAGGED])
def test_ragged_against_float64(c, lens, dtype, monkeypatch):
    out, kw, keep = solve(c, lens, dtype, monkeypatch, poison="nan")
    r = ragged_reference(kw, lens)
    bnd = bound(r, dtype)
    assert bool(torch.isfinite(out).all()), c.name
    worst = check(out, r, bnd, c.name)
    print(f"\n[attn-ragged] {c.name} {str(dtype)[6:]}: worst err/bound {worst:.3f}")
    # the rows past each length: NaN / inf and finite garbage give the same bits
    out2, _, _ = solve(c, lens, dtype, monkeypatch, poison="rand")
    assert torch.equal(out.view(torch.int16), out2.view(torch.int16)), f"{c.name}: rows past a length changed the output"


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("splits", [None, 1, 3, 7])
def test_equal_lengths_are_bitwise_m3r_attention(dtype, splits, monkeypatch):
    c = Case("equal", B=4, H=2, Nq=129, Nk0=1000, Nk1=200, kv_group=2, skip=(1000, 100, 100), splits=splits)
    kw, keep = make_inputs(c, dtype, "cuda", seed=2)
    force_splits(monkeypatch, splits)
    rows = c.B * c.Nq
    _, ref = out_buffer(rows, c.H, dtype)
    _, rag = out_buffer(rows, c.H, dtype)
    run(attn_args(kw, dtype, out=ref))
    run_ragged(attn_args(kw, dtype, out=rag), lengths_tensor([1000, 1000]))
    torch.cuda.synchronize()
    assert torch.equal(ref.view(torch.int16), rag.view(torch.int16))


def test_argument_errors():
    c = Case("args", B=2, H=2, Nq=64, Nk0=200)
    kw, keep = make_inputs(c, torch.float16, "cuda")
    _, out = out_buffer(c.B * c.Nq, c.H, torch.float16)
    lib = _lib.lib()
    nk0 = lengths_tensor([100, 200])
    a = attn_args(kw, torch.float16, out=out)
    assert lib.m3r_attention_ragged(C.byref(a), None, stream_ptr()) != 0
    assert b"nk0_b" in lib.m3r_last_error()
    assert lib.m3r_attention_ragged(C.byref(a), C.c_void_p(nk0.data_ptr() + 2), stream_ptr()) != 0
    assert b"aligned" in lib.m3r_last_error()
    ob = torch.empty(c.B * c.Nq, c.H * 64, device="cuda")
    mb = torch.empty(c.B * c.Nq, c.H, 2, device="cuda")
    e = attn_args(kw, torch.float16, exp=(ob, mb))
    assert lib.m3r_attention_ragged(C.byref(e), C.c_void_p(nk0.data_ptr()), stream_ptr()) != 0
    assert b"export" in lib.m3r_last_error()
    z = attn_args(kw, torch.float16, out=out)
    z.Nk0, z.K1, z.V1, z.ldk1, z.Nk1 = 0, z.K0, z.V0, z.ldk0, 100
    assert lib.m3r_attention_ragged(C.byref(z), C.c_void_p(nk0.data_ptr()), stream_ptr()) != 0
    assert b"Nk0" in lib.m3r_last_error()
    s = attn_args(kw, torch.float16, out=out)
    s.skip_lo, s.skip_len = 0, 200
    assert lib.m3r_attention_ragged(C.byref(s), C.c_void_p(nk0.data_ptr()), stream_ptr()) != 0
    assert b"skip range" in lib.m3r_last_error()
    torch.cuda.synchronize()
