"""The allowance of tests/gemm_ref.py is neither flaky nor blind: a plain-torch emulation of the GEMM kernel's arithmetic
stays within half of it on the case matrix of the GPU contract test (fewer rows, the same K, tile widths and epilogue
forms), and each planted fault exceeds it in at least one case where it applies, with a message naming the element.

The emulation follows csrc/gemm.cu: every k16 block of products summed exactly and added into an fp32 accumulator
rounding toward zero (each K half from zero under split-K, the halves then added in fp32), the epilogue in fp32 in the
kernel's order (bias, RoPE, row bias, GELU with erf, residual), the emitted LayerNorm from 32-column (mean, M2)
partials (two chains of 16, fma squares) combined with Chan's formula and rsqrt, and 16-bit outputs rounded to nearest."""
import pytest
import torch

from gemm_ref import (BM, EMIT_CASES, PLAIN_CASES, Case, check, emit_plan, layernorm, make_operands, off_by_4ulp,
                      out_bound, ref_kwargs, reference)

DT = [torch.float16, torch.bfloat16]
SMS = 132
EPS = 1e-6


def small(c: Case):
    """Case c with at most 130 rows (the same K, N, tile width and epilogue)."""
    from dataclasses import replace
    M = min(c.M, 130)
    return replace(c, M=M, rb_first=min(c.rb_first, M - 1) if c.rb_first > 0 else c.rb_first)


def rz_add(acc, blk):
    """fp32 acc + float64 blk rounded toward zero."""
    s = acc.double() + blk
    f = s.float()
    return torch.where(f.double().abs() > s.abs(), torch.nextafter(f, torch.zeros_like(f)), f)


def emulate_acc(a, w, ksplit, mut=None, bn=64):
    a64, w64 = a.double(), w.double()
    K = a.shape[1]
    half = K // ksplit
    parts = []
    for h in range(ksplit):
        acc = torch.zeros(a.shape[0], w.shape[0])
        for j in range(h * half, (h + 1) * half, 16):
            acc = rz_add(acc, a64[:, j:j + 16] @ w64[:, j:j + 16].t())
        parts.append(acc)
    if ksplit == 1:
        return parts[0]
    if mut == "splitk_half_dropped":
        parts[1][:BM, :bn] = 0                                             # tile (0, 0) loses its ks = 1 half
    return parts[0] + parts[1]


def emulate_gelu(x):
    z = x * torch.tensor(0.70710678118654752, dtype=torch.float32)
    return torch.tensor(0.5, dtype=torch.float32) * x * (1 + torch.erf(z))


def emulate(c: Case, d, dtype, ksplit, bn, mut=None):
    """(out, norm_out) of case c in the kernel's arithmetic; `mut` plants one fault (see MUTATIONS)."""
    M, N, K = c.M, c.N, c.K
    a, w = d["a"][:M, :K], d["w"][:N, :K]
    if mut == "bf16_operands":
        a, w = a.to(torch.bfloat16), w.to(torch.bfloat16)
    x = emulate_acc(a, w, ksplit, mut, bn)
    rows = torch.arange(M)
    col = torch.arange(N)
    if c.bias:
        b = d["bias"][:N].clone()
        if mut == "bias_q_off":                                            # column pair 2q of chunk 0 reads pair q + 1
            b[0:2] = d["bias"][2:4]
        if mut == "bias_chunk_missing":
            b[32:64] = 0
        x = x + b
    if c.rope_cols:
        t = d["rope_tab"][rows % c.rope_period]
        x = x.clone()
        for c0 in range(0, c.rope_cols, 32):
            h = (c0 // 32) % 2
            if mut == "rope_wrong_half" and c0 < 64:
                h ^= 1
            cs, sn = t[:, 32 * h:32 * h + 16], t[:, 32 * h + 16:32 * h + 32]
            uu, ww = x[:, c0:c0 + 16].clone(), x[:, c0 + 16:c0 + 32].clone()
            x[:, c0:c0 + 16] = uu * cs - ww * sn
            x[:, c0 + 16:c0 + 32] = ww * cs + uu * sn
    if c.rb_first >= 0:
        first = c.rb_first - 1 if mut == "rowbias_first_minus1" else c.rb_first
        on = ((rows % c.rb_period) >= first)[:, None]
        x = torch.where(on, x + d["rowbias"][:N], x)
    if c.gelu:
        g = emulate_gelu(x)
        if mut == "gelu_skip_half_chunk":                                   # the half-width last 16-bit chunk
            g = torch.where(((col % bn) >= 64 * (bn // 64))[None, :], x, g)
        x = g
    if c.res:
        r = d["residual"][:M, :N]
        if mut == "residual_row8":                                         # rows 16w + l/4 read row + 8
            src = torch.where((rows % 16 < 8) & (rows + 8 < M), rows + 8, rows)
            r = r[src]
        x = x + r
    norm = None
    if c.emit:
        norm = emulate_emit_ln(x, dtype, mut)
    out = x.to(dtype) if c.out16 and not c.emit else x
    if mut == "remap_off_by_one" and M > 64:
        out = out.clone()
        out[64] = out[63]                                                  # the row after a batch boundary at 64
    return out, norm


def emulate_emit_ln(x, dtype, mut=None):
    M, N = x.shape
    np_ = N // 32
    v = x.view(M, np_, 32)
    s0, s1 = torch.zeros(M, np_), torch.zeros(M, np_)
    for i in range(0, 32, 2):
        s0, s1 = s0 + v[..., i], s1 + v[..., i + 1]
    mu = (s0 + s1) * (1.0 / 32.0)
    q0, q1 = torch.zeros(M, np_), torch.zeros(M, np_)
    fma = lambda p, acc: (p.double() * p.double() + acc.double()).float()  # noqa: E731
    for i in range(0, 32, 2):
        q0, q1 = fma(v[..., i] - mu, q0), fma(v[..., i + 1] - mu, q1)
    m2p = q0 + q1
    n_mean = np_ - 1 if mut == "ln_mean_short" else np_
    msum = torch.zeros(M)
    for i in range(n_mean):
        msum = msum + mu[:, i]
    mean = msum / n_mean
    m2 = torch.zeros(M)
    for i in range(np_):
        dd = mu[:, i] - mean
        m2 = m2 + (m2p[:, i] if mut == "chan_dropped" else m2p[:, i] + 32.0 * dd * dd)
    rstd = torch.rsqrt(m2 / (32.0 * np_) + EPS)
    return ((x - mean[:, None]) * rstd[:, None]).to(dtype)


@pytest.fixture(scope="module")
def problems():
    cache = {}

    def get(c, dtype):
        key = (c, dtype)
        if key not in cache:
            d = make_operands(c, dtype, "cpu", seed=1)
            bn, ks = emit_plan(c.M, c.N, c.K, SMS) if c.emit else (c.bn, 1)
            cs = small(c)
            r = reference(d["a"], d["w"], **ref_kwargs(cs, d, ks))
            res = dict(d=d, c=cs, bn=bn, ks=ks, ref=r, bnd=out_bound(r.val, r.err, torch.float32 if (cs.emit or not cs.out16) else dtype))
            if c.emit:
                nv, ne = layernorm(r.val, r.err, EPS, "emit")
                res.update(nval=nv, nbnd=out_bound(nv, ne, dtype))
            cache[key] = res
        return cache[key]
    return get


EMIT = [Case(**{**c.__dict__, "emit": True}) for c in EMIT_CASES]
ALL = PLAIN_CASES + EMIT


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
def test_faithful_emulation_within_half_the_bound(problems, dtype):
    worst = {}
    for c in ALL:
        p = problems(c, dtype)
        out, norm = emulate(p["c"], p["d"], dtype, p["ks"], p["bn"])
        worst[c.name] = check(out, p["ref"].val, p["bnd"], c.name, M=p["c"].M, bn=p["bn"])
        if norm is not None:
            worst[c.name + " norm"] = check(norm, p["nval"], p["nbnd"], c.name + " norm", M=p["c"].M, bn=p["bn"])
    print({k: round(v, 3) for k, v in worst.items()})
    assert max(worst.values()) <= 0.5, max(worst.items(), key=lambda kv: kv[1])


def by(pred):
    return [c for c in ALL if pred(c)]


# planted fault -> the cases it applies to; each must be rejected in at least one of them.
MUTATIONS = {
    "bias_q_off": by(lambda c: c.bias and not c.emit and c.M >= 64)[:6],
    "bias_chunk_missing": by(lambda c: c.bias and c.N >= 64)[:6],
    "rope_wrong_half": by(lambda c: c.rope_cols > 0),
    "gelu_skip_half_chunk": by(lambda c: c.gelu and c.out16 and c.bn in (32, 160)),
    "residual_row8": by(lambda c: c.res != "" and c.M > 8)[:6],
    "remap_off_by_one": by(lambda c: c.M > 64 and not c.emit)[:4],
    "rowbias_first_minus1": by(lambda c: c.rb_first > 0),
    "ulp4": by(lambda c: c.out16 and not c.emit)[:6],
    "bf16_operands": by(lambda c: c.K >= 512)[:6],
    "ln_mean_short": EMIT,
    "chan_dropped": EMIT,
    "splitk_half_dropped": by(lambda c: c.emit and c.K >= 2048),
}
NORM_FAULTS = ("ln_mean_short", "chan_dropped")


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_each_fault_is_rejected(problems, dtype, mut):
    if mut == "bf16_operands" and dtype == torch.bfloat16:
        pytest.skip("the operands are already bf16")
    cases = MUTATIONS[mut]
    assert cases, mut
    for c in cases:
        p = problems(c, dtype)
        cs = p["c"]
        if mut == "ulp4":
            out, norm = emulate(cs, p["d"], dtype, p["ks"], p["bn"])
            out = off_by_4ulp(out, p["bnd"])
        else:
            out, norm = emulate(cs, p["d"], dtype, p["ks"], p["bn"], mut=mut)
        try:
            if mut in NORM_FAULTS:
                check(norm, p["nval"], p["nbnd"], f"{mut} {c.name} norm", M=cs.M, bn=p["bn"])
            else:
                check(out, p["ref"].val, p["bnd"], f"{mut} {c.name}", M=cs.M, bn=p["bn"])
        except AssertionError as e:
            msg = str(e)
            assert " row " in msg and " column " in msg and "tile" in msg, msg
            print(msg)
            return
    pytest.fail(f"{mut} passed the allowance in every case it applies to")
