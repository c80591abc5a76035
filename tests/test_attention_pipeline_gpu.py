"""The pipelined attention kernel at its tile, segment, skip-range and split boundaries, against an fp32 softmax reference,
with several key-split counts forced (M3R_ATTN_SPLITS)."""
import pytest
import torch

from must3r_b200 import ops

pytestmark = pytest.mark.gpu

DT = [torch.float16, torch.bfloat16]
ATT_TOL = {torch.float16: 1.5e-3, torch.bfloat16: 8e-3}
SPLITS = [1, 3, 7]


def rnd(*shape, dtype=torch.float32, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dtype)


def rel_l2(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def reference(q, k0, v0, k1, v1, B, H, Nq, Nk0, Nk1, kv_group, skip_lo, skip_step, skip_len):
    """fp32 softmax(Q K^T / 8) V over the keys [segment 0 | segment 1] of each batch's key/value batch, without the
    skip range of each batch."""
    D = H * 64
    Bkv = B // kv_group
    k = torch.cat([k0.float().view(Bkv, Nk0, D), k1.float().view(Bkv, Nk1, D)], 1) if Nk1 else k0.float().view(Bkv, Nk0, D)
    v = torch.cat([v0.float().view(Bkv, Nk0, D), v1.float().view(Bkv, Nk1, D)], 1) if Nk1 else v0.float().view(Bkv, Nk0, D)
    Nk = Nk0 + Nk1
    k = k.view(Bkv, Nk, H, 64).transpose(1, 2)
    v = v.view(Bkv, Nk, H, 64).transpose(1, 2)
    qh = q.float().view(B, Nq, H, 64).transpose(1, 2)
    out = torch.empty(B, H, Nq, 64, device="cuda")
    for j in range(B):                              # one batch at a time: the score matrix of the C3 shapes is ~0.5 GB each
        s = (qh[j] @ k[j // kv_group].transpose(-1, -2)) * 0.125
        if skip_len:
            lo = skip_lo + (j % kv_group) * skip_step
            s[..., lo:lo + skip_len] = float("-inf")
        out[j] = torch.softmax(s, -1) @ v[j // kv_group]
    return out.transpose(1, 2).reshape(B * Nq, D)


def run(dtype, B, H, Nq, Nk0, Nk1=0, kv_group=1, skip_lo=0, skip_step=0, skip_len=0, qscale=1.0, kscale=None, export=False):
    D = H * 64
    Bkv = B // kv_group
    q = rnd(B * Nq, D, dtype=dtype, seed=1, scale=qscale)
    k0 = rnd(Bkv * Nk0, D, seed=2)
    if kscale is not None:
        k0 = k0 * kscale.repeat(Bkv)[:, None]
    k0, v0 = k0.to(dtype), rnd(Bkv * Nk0, D, dtype=dtype, seed=3)
    k1 = rnd(Bkv * Nk1, D, dtype=dtype, seed=4) if Nk1 else None
    v1 = rnd(Bkv * Nk1, D, dtype=dtype, seed=5) if Nk1 else None
    kw = dict(B=B, H=H, Nq=Nq, Nk0=Nk0, k1=k1, v1=v1, Nk1=Nk1, kv_group=kv_group, skip_lo=skip_lo, skip_step=skip_step,
              skip_len=skip_len)
    ref = reference(q, k0, v0, k1, v1, B, H, Nq, Nk0, Nk1, kv_group, skip_lo, skip_step, skip_len)
    if export:
        o, ml = ops.attention(q, k0, v0, export=True, **kw)
        out = o.view(B * Nq, H, 64) / ml[..., 1:2]
        return out.reshape(B * Nq, D), ref
    return ops.attention(q, k0, v0, **kw), ref


CASES = {
    # name: (B, H, Nq, Nk0, Nk1, kv_group, skip_lo, skip_step, skip_len)
    "nq196": (2, 2, 196, 640, 0, 1, 0, 0, 0),
    "nq300": (1, 3, 300, 500, 0, 1, 0, 0, 0),
    "nq768": (1, 2, 768, 768, 0, 1, 0, 0, 0),
    "nq1": (3, 2, 1, 300, 0, 1, 0, 0, 0),
    "nq_cta_plus_one": (1, 2, 129, 256, 0, 1, 0, 0, 0),
    "nk_one_tile": (2, 2, 200, 128, 0, 1, 0, 0, 0),
    "nk_tile_plus_one": (2, 2, 200, 129, 0, 1, 0, 0, 0),
    "seg0_ends_inside_tile": (1, 2, 150, 200, 300, 1, 0, 0, 0),
    "skip_inside_tiles": (2, 2, 150, 300, 400, 2, 250, 200, 200),
    "one_key_left": (1, 2, 130, 129, 0, 1, 0, 0, 128),
}


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("splits", SPLITS)
@pytest.mark.parametrize("case", list(CASES))
def test_boundaries(dtype, splits, case, monkeypatch):
    monkeypatch.setenv("M3R_ATTN_SPLITS", str(splits))
    B, H, Nq, Nk0, Nk1, grp, lo, step, ln = CASES[case]
    out, ref = run(dtype, B, H, Nq, Nk0, Nk1, grp, lo, step, ln)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("splits", SPLITS)
def test_growing_max_and_large_scores(dtype, splits, monkeypatch):
    """Keys ordered so that the row max grows on every tile (lazy rescale), then scores near the fp16 overflow range."""
    monkeypatch.setenv("M3R_ATTN_SPLITS", str(splits))
    Nk = 1024
    out, ref = run(dtype, 1, 2, 200, Nk, qscale=2.0, kscale=torch.linspace(0.2, 4.0, Nk, device="cuda"))
    assert rel_l2(out, ref) < ATT_TOL[dtype]
    out, ref = run(dtype, 1, 2, 200, 384, qscale=40.0)
    assert torch.isfinite(out.float()).all()
    assert rel_l2(out, ref) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
@pytest.mark.parametrize("splits", [1, 3])
def test_export(dtype, splits, monkeypatch):
    monkeypatch.setenv("M3R_ATTN_SPLITS", str(splits))
    out, ref = run(dtype, 2, 2, 200, 700, 150, 2, 600, 100, 100, export=True)
    assert rel_l2(out, ref) < ATT_TOL[dtype]


@pytest.mark.parametrize("dtype", DT)
def test_c3_shapes(dtype):
    """The benchmarked shapes with the default configuration: render cross-attention (20 views sharing a 20-view memory)
    and the one-view update against a 19-view memory with its own tokens skipped."""
    out, ref = run(dtype, 20, 12, 768, 15360, kv_group=20)
    assert rel_l2(out, ref) < ATT_TOL[dtype]
    out, ref = run(dtype, 1, 12, 768, 18 * 768, 768, 1, 18 * 768, 0, 768)
    assert rel_l2(out, ref) < ATT_TOL[dtype]
