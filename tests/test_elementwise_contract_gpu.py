"""The small kernels of csrc/elementwise.cu and the nearest-neighbour scan element by element against the float64
allowances of tests/elementwise_ref.py (or bitwise where the kernel only moves or rounds data), with guarded outputs and
NaN-padded inputs.

- Every output is a view into a sentinel-filled buffer and nothing outside it may change: rows after the im2col16,
  unpatchify and RoPE-table outputs; the q and v slices, padding columns and rows past N of the fused qkv buffer that
  rope_2d rotates in place; past P and past Q for postprocess and nn_min_dist; around both attn_state_fill exports and
  around every peer_bcast destination.
- Inputs are followed by NaN, so a read past the end shows up as a NaN: head-output rows past V*N, pointmap rows past P,
  database points past P, queries past Q, and a NaN image after the last one of im2col16.
- Call-site shapes: every model aspect ratio (224x224, 512x384 both ways, 512x288, 512x336) with V = 1 and V = 20
  (20 views at 512x384 is the C3 workload, where the grid-stride loops wrap several times); the real RoPE table built
  from the encoder's positions and from a two-group decoder call, fed to the GEMM's RoPE epilogue and checked against
  gemm_ref.reference with the exact table plus the table's error bound.
- Argument errors raised before any launch: rope_2d positions that are not int64 or not on the tokens' device, negative
  RoPE dimensions, an unpatchify without channels.
Every case prints its worst err / allowance."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from elementwise_ref import (GRIDS, NN_KINDS, NN_P, NN_Q, ROPE_CASES, TABLE_CASES, check, grid_pos, nn_points, nn_ref,
                             pm_inputs, postprocess_ref, rope_2d_ref, rope_inputs, rope_table_ref, zero_sign_ok)
from gemm_ref import Case, make_operands, out_bound, ref_kwargs, reference
from gemm_ref import check as gemm_check
from must3r_b200 import _lib, ops

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
SENTINEL = 7.0
NAN = float("nan")
SITES = [(gh * 16, gw * 16, V) for gh, gw in GRIDS for V in (1, 20)]


def P(t):
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ok(rc):
    assert rc == 0, _lib.lib().m3r_last_error().decode()


def report(group, name, worst):
    print(f"\n[elementwise-contract] {group} {name}: worst err/allowance {worst:.3f}")


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ------------------------------------------------------------------------------------------------ RoPE table
@pytest.mark.parametrize("case", TABLE_CASES, ids=[c[0] for c in TABLE_CASES])
def test_rope_table(case):
    name, pos, base, f0 = case
    T = pos.shape[0]
    pos = pos.cuda().contiguous()
    buf = torch.full((T + 8, 64), SENTINEL, device="cuda")
    ok(_lib.lib().m3r_rope_table(P(pos), T, base, f0, P(buf), stream_ptr()))
    torch.cuda.synchronize()
    assert bool((buf[T:] == SENTINEL).all()), f"{name}: a store landed past the table"
    val, _, bnd = rope_table_ref(pos, base, f0)
    report("table", name, check(buf[:T], val, bnd, f"table {name}", dims=("token", "column")))


# ------------------------------------------------------------------------------------------------ stand-alone RoPE
WRAP = [(f"{str(dt)[6:]}_wrap_B2_N768_H12_D64", dt, 2, 768, 12, 64, -1.0, "large") for dt in (torch.float16, torch.bfloat16)]


@pytest.mark.parametrize("case", ROPE_CASES + WRAP, ids=[c[0] for c in ROPE_CASES + WRAP])
def test_rope_2d(case):
    """In place on the k slice of a fused [B, N + 3, 3, H, D + 8] buffer, as the curope seam passes it."""
    name, dt, B, N, H, D, fwd, kind = case
    assert B * N * H * D // 2 > 132 * 16 * 256 or "wrap" not in name, "the grid-stride loop must wrap"
    tok, pos = rope_inputs(dt, B, N, H, D, kind, seed=D + 1)
    g = torch.Generator().manual_seed(D)
    buf = (torch.randn(B, N + 3, 3, H, D + 8, generator=g) * 3).to(dt).cuda()
    buf[:, :N, 1, :, :D] = tok.cuda()
    before = buf.clone()
    view = buf[:, :N, 1, :, :D]
    pos = pos.cuda()
    val, bnd = rope_2d_ref(view, pos, 100.0, fwd)
    ops.rope_2d(view, pos, 100.0, fwd)
    torch.cuda.synchronize()
    keep = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    keep[:, :N, 1, :, :D] = False
    assert same_bits(buf[keep], before[keep]), f"{name}: an element outside the rotated slice changed"
    report("rope", name, check(view, val, bnd, f"rope {name}", dims=("b", "n", "head", "column")))


def test_rope_2d_argument_errors():
    tok = torch.zeros(2, 5, 3, 64, device="cuda", dtype=torch.float16)
    pos = torch.zeros(2, 5, 2, device="cuda", dtype=torch.int64)
    before = tok.clone()
    with pytest.raises(RuntimeError, match="Long"):
        ops.rope_2d(tok, pos.int(), 100.0, 1.0)
    with pytest.raises(RuntimeError, match="same device"):
        ops.rope_2d(tok, pos.cpu(), 100.0, 1.0)
    with pytest.raises(RuntimeError, match="4 dimensions"):
        ops.rope_2d(tok[0], pos, 100.0, 1.0)
    L = _lib.lib()
    for B, N, H in ((-2, -5, 3), (2, -5, -3)):
        assert L.m3r_rope_2d(P(tok), 1, B, N, H, 64, 960, 192, 64, P(pos), 100.0, 1.0, stream_ptr()) != 0
        assert "negative dimension" in L.m3r_last_error().decode()
    torch.cuda.synchronize()
    assert torch.equal(tok, before)


# ------------------------------------------------------------------------------------------------ patch embedding
@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("site", SITES, ids=[f"{h}x{w}_V{v}" for h, w, v in SITES])
def test_im2col16(site, dtype):
    """Bitwise F.unfold(img, 16, stride=16).transpose(1, 2) rounded as tensor.to(dtype) rounds (NaN-ness for NaN)."""
    H, W, V = site
    g = torch.Generator().manual_seed(H + W + V)
    img = torch.full((V + 1, 3, H, W), NAN)
    img[:V] = torch.randn(V, 3, H, W, generator=g) * 2
    edge = torch.tensor([65504.0, 65519.99, 65520.0, -65520.0, -65519.99, 1e6, -1e6, 6e-8, 1e-9, -0.0, NAN,
                         math.inf, -math.inf, 3e38, 1.0000001, 2.0 ** -14])
    img[0, 1, 17, :len(edge)] = edge
    img[V - 1, 2, H - 1, W - len(edge):] = edge
    img = img.cuda()
    Np = V * (H // 16) * (W // 16)
    buf = torch.full((Np + 4, 768), SENTINEL, device="cuda", dtype=dtype)
    ok(_lib.lib().m3r_im2col16(P(img), V, H, W, P(buf), int(dtype == torch.bfloat16), stream_ptr()))
    torch.cuda.synchronize()
    assert bool((buf[Np:] == SENTINEL).all()), "a store landed past the patch matrix"
    ref = F.unfold(img[:V], 16, stride=16).transpose(1, 2).reshape(Np, 768).to(dtype)
    out = buf[:Np]
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(out), nan), "NaN-ness differs"
    diff = (out != ref) & ~nan
    assert not bool(diff.any()), f"first differing element (row, col) {diff.nonzero()[0].tolist()}"


# ------------------------------------------------------------------------------------------------ head
@pytest.mark.parametrize("site", SITES, ids=[f"{h}x{w}_V{v}" for h, w, v in SITES])
def test_unpatchify(site):
    """out[v, 16y + i, 16x + j, c] = proj[v N + y gw + x, 256 c + 16 i + j], bitwise, at C = 1, 4 and 7."""
    H, W, V = site
    gh, gw = H // 16, W // 16
    N = gh * gw
    g = torch.Generator(device="cuda").manual_seed(H + W + V)           # leaves the default generator alone
    for C_ in (1, 4, 7):
        proj = torch.full((V * N + 8, C_ * 256), NAN, device="cuda")
        proj[:V * N] = torch.randn(V * N, C_ * 256, device="cuda", generator=g)
        n_out = V * H * W * C_
        buf = torch.full((n_out + 64,), SENTINEL, device="cuda")
        ok(_lib.lib().m3r_unpatchify(P(proj), V, H, W, C_, P(buf), stream_ptr()))
        torch.cuda.synchronize()
        assert bool((buf[n_out:] == SENTINEL).all()), f"C={C_}: a store landed past the output"
        ref = proj[:V * N].view(V, gh, gw, C_, 16, 16).permute(0, 1, 4, 2, 5, 3).reshape(V, H, W, C_)
        assert torch.equal(buf[:n_out].view(V, H, W, C_), ref), f"C={C_}"


def test_unpatchify_refuses_no_channels():
    proj = torch.zeros(6, 256, device="cuda")
    out = torch.full((2 * 32 * 48,), SENTINEL, device="cuda")
    for C_ in (0, -7):
        assert _lib.lib().m3r_unpatchify(P(proj), 2, 32, 48, C_, P(out), stream_ptr()) != 0
        assert "C=" in _lib.lib().m3r_last_error().decode()
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())


# ------------------------------------------------------------------------------------------------ postprocess
@pytest.mark.parametrize("site", SITES, ids=[f"{h}x{w}_V{v}" for h, w, v in SITES])
def test_postprocess(site):
    H, W, V = site
    Pn = V * H * W
    pm = torch.full((Pn + 8, 7), NAN, device="cuda")
    pm[:Pn] = pm_inputs(Pn, seed=Pn, device="cuda")
    bufs = [torch.full((Pn + 8, 3), SENTINEL, device="cuda"), torch.full((Pn + 8, 3), SENTINEL, device="cuda"),
            torch.full((Pn + 8,), SENTINEL, device="cuda")]
    ok(_lib.lib().m3r_postprocess(P(pm), Pn, P(bufs[0]), P(bufs[1]), P(bufs[2]), stream_ptr()))
    torch.cuda.synchronize()
    assert all(bool((b[Pn:] == SENTINEL).all()) for b in bufs), "a store landed past P"
    ref = postprocess_ref(pm[:Pn])
    worst = 0.0
    for (k, (val, bnd)), b in zip(ref.items(), bufs):
        worst = max(worst, check(b[:Pn], val, bnd, f"postprocess {k} {H}x{W} V={V}", dims=("point", "channel")))
    for k, lo, b in (("pts3d", 0, bufs[0]), ("pts3d_local", 3, bufs[1])):
        assert zero_sign_ok(pm[:Pn], b[:Pn], lo), f"{k}: a zero vector did not give a zero of its sign"
    report("postprocess", f"{H}x{W}_V{V}", worst)


# ------------------------------------------------------------------------------------------------ nearest neighbour
NN_CASES = [(P_, Q_) for P_ in NN_P for Q_ in NN_Q]


@pytest.mark.parametrize("i", range(len(NN_CASES)), ids=[f"P{p}_Q{q}" for p, q in NN_CASES])
def test_nn_min_dist(i):
    Pn, Qn = NN_CASES[i]
    kind = NN_KINDS[i % 3]
    q, db = nn_points(kind, Pn, Qn, seed=100 + i)
    qb = torch.full((Qn + 4, 3), NAN, device="cuda")
    qb[:Qn] = q.cuda()
    dbb = torch.full((Pn + 4, 3), NAN, device="cuda")
    dbb[:Pn] = db.cuda()
    out = torch.full((Qn + 8,), SENTINEL, device="cuda")
    ok(_lib.lib().m3r_nn_min_dist(P(qb), Qn, P(dbb) if Pn else None, Pn, P(out), stream_ptr()))
    torch.cuda.synchronize()
    assert bool((out[Qn:] == SENTINEL).all()), "a store landed past Q"
    val, bnd = nn_ref(qb[:Qn], dbb[:Pn])
    report("scan", f"P{Pn}_Q{Qn}_{kind}", check(out[:Qn], val, bnd, f"nn P={Pn} Q={Qn} {kind}", dims=("query",)))


def test_nn_min_dist_exact_classes():
    """Empty database, a database of only NaN / inf points, a NaN query: +inf; an exact duplicate: 0."""
    q = torch.tensor([[0.0, 0.0, 0.0], [NAN, 0.0, 0.0], [1.0, 2.0, 3.0], [1e3, -1e3, 5.0]], device="cuda")
    bad = torch.tensor([[NAN, 0.0, 0.0], [0.0, math.inf, 0.0], [NAN, NAN, NAN], [-math.inf, 1.0, 1.0]] * 300,
                       device="cuda")
    mixed = torch.cat([bad, torch.tensor([[1.0, 2.0, 3.0]], device="cuda"), bad])
    L = _lib.lib()
    for db, want in ((None, [math.inf] * 4), (bad, [math.inf] * 4), (mixed, None)):
        out = torch.full((12,), SENTINEL, device="cuda")
        ok(L.m3r_nn_min_dist(P(q), 4, P(db) if db is not None else None, 0 if db is None else db.shape[0], P(out),
                             stream_ptr()))
        torch.cuda.synchronize()
        assert bool((out[4:] == SENTINEL).all())
        if want is not None:
            assert out[:4].tolist() == want
        else:
            assert float(out[2]) == 0.0 and math.isinf(float(out[1]))
            assert float(out[0]) == pytest.approx(math.sqrt(14.0), rel=1e-6)


# ------------------------------------------------------------------------------------------------ attention state fill
@pytest.mark.parametrize("rows,H", [(1, 1), (130, 12), (5000, 16)])
def test_attn_state_fill(rows, H):
    """o = 0 and (m, l) = (-inf, 0), nothing written outside either export (5000 x 16: the grid-stride loop wraps)."""
    n_o, n_ml, G = rows * H * 64, rows * H * 2, 64
    ob = torch.full((n_o + 2 * G,), SENTINEL, device="cuda")
    mb = torch.full((n_ml + 2 * G,), SENTINEL, device="cuda")
    ok(_lib.lib().m3r_attn_state_fill(P(ob[G:]), P(mb[G:]), rows, H, stream_ptr()))
    torch.cuda.synchronize()
    assert bool((ob[:G] == SENTINEL).all() and (ob[G + n_o:] == SENTINEL).all()), "export_o guard changed"
    assert bool((mb[:G] == SENTINEL).all() and (mb[G + n_ml:] == SENTINEL).all()), "export_ml guard changed"
    o, ml = ob[G:G + n_o], mb[G:G + n_ml].view(-1, 2)
    assert bool((o == 0).all()) and not bool(torch.signbit(o).any())
    assert bool((ml[:, 0] == -math.inf).all()) and bool((ml[:, 1] == 0).all())


# ------------------------------------------------------------------------------------------------ peer broadcast
TAIL = 3 * 4096 + 48                      # not a multiple of one block's 4096 bytes
BIG = 20 * (1 << 20) + 80                 # several passes of the grid-stride loop
BCAST = [(1, 16), (2, TAIL), (3, BIG), (4, 16), (5, TAIL), (6, BIG), (7, 16), (8, TAIL), (8, BIG)]


@pytest.mark.parametrize("n,nbytes", BCAST, ids=[f"n{n}_{b}B" for n, b in BCAST])
def test_peer_bcast(n, nbytes):
    G = 256
    g = torch.Generator(device="cuda").manual_seed(n)
    src_buf = torch.randint(0, 256, (nbytes + 2 * G,), dtype=torch.uint8, device="cuda", generator=g)
    dst = [torch.full((nbytes + 2 * G,), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(n)]
    arr = (C.c_void_p * n)(*[d.data_ptr() + G for d in dst])
    ok(_lib.lib().m3r_peer_bcast(C.c_void_p(src_buf.data_ptr() + G), arr, n, nbytes, stream_ptr()))
    torch.cuda.synchronize()
    for k, d in enumerate(dst):
        assert torch.equal(d[G:G + nbytes], src_buf[G:G + nbytes]), f"destination {k} differs from the source"
        assert bool((d[:G] == 0xA5).all() and (d[G + nbytes:] == 0xA5).all()), f"destination {k}: a guard changed"


# ------------------------------------------------------------------------------------------------ real table into the GEMM
def view_pos(gh, gw, views):
    return grid_pos(gh, gw).repeat(views, 1)


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("form", ["encoder", "decoder"])
def test_gemm_with_the_real_table(form, dtype):
    """ops.rope_table of the encoder's positions for one view, used with rope_period = N by a V = 2 qkv projection; or
    the decoder's per-group table rows of a two-group call (2 views of 18x32, 1 view of 21x32) written at each group's
    row offset, used with rope_period = M.  Checked against gemm_ref.reference with the exact float64 table and the
    table's error bound; the table itself against its allowance."""
    Dm, base = 256, 100.0
    if form == "encoder":
        f0 = 1.0
        pos = grid_pos(24, 32).cuda()
        tab = ops.rope_table(pos, base, f0)
        M = 2 * pos.shape[0]
    else:
        f0 = 224 / 512
        groups = [view_pos(18, 32, 2).cuda(), view_pos(21, 32, 1).cuda()]
        pos = torch.cat(groups).contiguous()
        M = pos.shape[0]
        buf = torch.full((M + 8, 64), SENTINEL, device="cuda")
        row0 = 0
        for g in groups:
            ok(_lib.lib().m3r_rope_table(P(g), g.shape[0], base, f0, C.c_void_p(buf[row0:].data_ptr()), stream_ptr()))
            row0 += g.shape[0]
        torch.cuda.synchronize()
        assert bool((buf[M:] == SENTINEL).all()), "a table store landed past the last group"
        tab = buf[:M]
    tval, terr, tbnd = rope_table_ref(pos, base, f0)
    worst_tab = check(tab, tval, tbnd, f"{form} table", dims=("token", "column"))
    c = Case(f"real_table_{form}", M, 3 * Dm, Dm, rope_cols=2 * Dm, rope_period=tab.shape[0])
    d = make_operands(c, dtype, "cuda")
    out = ops.linear(d["a"], d["w"][:c.N], d["bias"], rope_tab=tab, rope_cols=2 * Dm)
    torch.cuda.synchronize()
    r = reference(d["a"], d["w"], **{**ref_kwargs(c, d), "rope_tab": tval, "rope_tab_err": terr})
    worst = gemm_check(out, r.val, out_bound(r.val, r.err, dtype), c.name, M=M)
    report("real-table gemm", f"{form} {str(dtype)[6:]}", worst)
    report("real-table table", f"{form}", worst_tab)
