"""The epilogue of persistent plain GEMM launches (more tiles than SMs, so every CTA owns several tiles) drains its
staged chunks through TMA stores that complete while the next tile's MMAs run.

Each epilogue form is checked three ways, at BN 256 and 128, fp16 and bf16, with M a multiple of the tile height and M
ragged:
- against fp32 torch math on the same 16-bit inputs;
- bitwise against the first rows computed by a one-wave launch (few enough tiles for one per CTA), whose threads copy
  the staged chunks to global memory: both drains must store the same values;
- output memory outside the [M, N] result (rows past M, columns beside a column slice) must stay untouched, so a store
  that is dropped or lands in the wrong place fails."""
import os

import pytest
import torch
import torch.nn.functional as F

from must3r_b200 import ops
from must3r_b200.synthetic import rel_l2

pytestmark = pytest.mark.gpu
DT = [torch.float16, torch.bfloat16]
OUT_TOL = {torch.float16: 6e-4, torch.bfloat16: 5e-3, torch.float32: 2e-5}
N, K = 1024, 128
M_FULL = 15360
M_WAVE = 1024                      # 8 m-tiles: at most 64 tiles at BN 128, one per CTA
PERIOD = 768                       # tokens per view (RoPE table rows, row-bias period)
ROPE_COLS = 512
SENTINEL = 7.0
FORMS = ["bias_f32", "bias_16", "gelu", "rope", "rowbias", "residual_inplace", "ldc_slice"]


def rnd(*shape, dtype=torch.float32, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def rope_ref(y, tab, rows):
    """RoPE as the epilogue applies it: per 64-column head, each 32-column half rotates (u = cols 0..15, v = 16..31) with
    cos = tab[row % period, 32 h + i] and sin = tab[row % period, 32 h + 16 + i]."""
    y = y.clone()
    t = tab[torch.arange(rows, device=y.device) % tab.shape[0]]
    for c0 in range(0, ROPE_COLS, 32):
        h = (c0 // 32) % 2
        cs, sn = t[:, 32 * h:32 * h + 16], t[:, 32 * h + 16:32 * h + 32]
        u, v = y[:, c0:c0 + 16].clone(), y[:, c0 + 16:c0 + 32].clone()
        y[:, c0:c0 + 16] = u * cs - v * sn
        y[:, c0 + 16:c0 + 32] = v * cs + u * sn
    return y


def run(form, dtype, M, a, w, bias, extra):
    """One launch of `form` over the first M rows; returns (result [M, N], whole output buffer, untouched-region mask)."""
    a = a[:M]
    out_dtype = torch.float32 if form in ("bias_f32", "rowbias", "residual_inplace") else dtype
    # the output lives inside a larger buffer: 64 rows below it and, for ldc_slice, 256 columns on either side
    pad = 256 if form == "ldc_slice" else 0
    buf = torch.full((M + 64, N + 2 * pad), SENTINEL, device="cuda", dtype=out_dtype)
    out = buf[:M, pad:pad + N]
    kw = {}
    if form == "gelu":
        kw["act"] = "gelu"
    elif form == "rope":
        kw.update(rope_tab=extra["rope"], rope_cols=ROPE_COLS)
    elif form == "rowbias":
        kw.update(rowbias=extra["rowbias"], rb_period=PERIOD, rb_first=1)
    elif form == "residual_inplace":
        out.copy_(extra["res"][:M])
        kw["residual"] = out
    ops.linear(a, w, bias, out=out, **kw)
    outside = torch.ones_like(buf, dtype=torch.bool)
    outside[:M, pad:pad + N] = False
    return out, buf, outside


def reference(form, M, a, w, bias, extra):
    y = a[:M].float() @ w.float().t() + bias
    if form == "gelu":
        y = F.gelu(y)
    elif form == "rope":
        y = rope_ref(y, extra["rope"], M)
    elif form == "rowbias":
        on = (torch.arange(M, device="cuda") % PERIOD) >= 1
        y = y + on[:, None].float() * extra["rowbias"]
    elif form == "residual_inplace":
        y = y + extra["res"][:M]
    return y


@pytest.fixture(scope="module")
def operands():
    ops_by_dtype = {}
    for dtype in DT:
        a, w = rnd(M_FULL, K, dtype=dtype, seed=1), rnd(N, K, dtype=dtype, seed=2, scale=K ** -0.5)
        ang = rnd(PERIOD, 32, seed=5) * 3.0
        rope = torch.cat([torch.cos(ang[:, :16]), torch.sin(ang[:, :16]), torch.cos(ang[:, 16:]), torch.sin(ang[:, 16:])], 1).contiguous()
        extra = {"rope": rope, "rowbias": rnd(N, seed=6), "res": rnd(M_FULL, N, seed=7)}
        ops_by_dtype[dtype] = (a, w, rnd(N, seed=3), extra)
    return ops_by_dtype


@pytest.fixture
def force_bn():
    def set_bn(bn):
        os.environ["M3R_GEMM_BN"] = str(bn)
    yield set_bn
    os.environ.pop("M3R_GEMM_BN", None)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("M", [M_FULL, M_FULL - 37])
@pytest.mark.parametrize("bn", [256, 128])
@pytest.mark.parametrize("dtype", DT)
def test_persistent_epilogue(operands, force_bn, dtype, bn, M, form):
    a, w, bias, extra = operands[dtype]
    force_bn(bn)
    out, buf, outside = run(form, dtype, M, a, w, bias, extra)
    wave, _, _ = run(form, dtype, M_WAVE, a, w, bias, extra)
    torch.cuda.synchronize()
    assert bool((buf[outside] == SENTINEL).all()), "a store landed outside the output"
    assert torch.equal(out[:M_WAVE], wave), "persistent and one-wave epilogues differ"
    ref = reference(form, M, a, w, bias, extra)
    assert rel_l2(out, ref) < OUT_TOL[out.dtype]
    # every row, the ragged last tile's included, holds its own result
    row_err = (out.float() - ref).norm(dim=1) / ref.norm(dim=1)
    assert float(row_err.max()) < 4 * OUT_TOL[out.dtype]


@pytest.mark.parametrize("bn", [256, 128])
def test_persistent_epilogue_side_stream(operands, force_bn, bn):
    """Two launches on a side stream match the caller's stream bitwise (the stores of one launch are complete before
    the next kernel on the stream reads or overwrites its output)."""
    dtype = torch.bfloat16
    a, w, bias, extra = operands[dtype]
    force_bn(bn)
    base = ops.linear(a, w, bias, act="gelu")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        first = ops.linear(a, w, bias, act="gelu")
        second = ops.linear(a, w, bias, act="gelu")
        res = extra["res"].clone()
        ops.linear(a, w, bias, residual=res, out=res)
        ops.linear(a, w, bias, residual=res, out=res)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    assert torch.equal(first, base) and torch.equal(second, base)
    res_ref = extra["res"].clone()
    ops.linear(a, w, bias, residual=res_ref, out=res_ref)
    ops.linear(a, w, bias, residual=res_ref, out=res_ref)
    torch.cuda.synchronize()
    assert torch.equal(res, res_ref)
