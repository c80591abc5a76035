import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import ops

def rnd(*shape, dtype=torch.float32, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()

def ref_attn(q, k, v, mask=None):
    s = (q.float() @ k.float().transpose(-1, -2)) * 0.125
    if mask is not None: s = s.masked_fill(~mask, float("-inf"))
    return torch.softmax(s, -1) @ v.float()

def case(dtype, Nm, n, N, B=2, H=12, env=None, tag=""):
    os.environ.pop("M3R_ATTN_SPLITS", None)
    if env: os.environ.update(env)
    D = H * 64
    cap = Nm + 77
    mem = torch.full((B, cap, 2 * D), float("nan"), device="cuda", dtype=dtype)
    mem[:, :Nm] = rnd(B, Nm, 2 * D, dtype=dtype, seed=20)
    new = rnd(B, n * N, 2 * D, dtype=dtype, seed=21)
    q = rnd(B * n * N, D, dtype=dtype, seed=22)
    mem2, new2 = mem.view(B * cap, 2 * D), new.view(B * n * N, 2 * D)
    out = ops.attention(q, mem2[:, :D], mem2[:, D:], B=B * n, H=H, Nq=N, Nk0=Nm, kv_bstride0=cap,
                        k1=new2[:, :D], v1=new2[:, D:], Nk1=n * N, kv_bstride1=n * N, kv_group=n, skip_lo=Nm, skip_step=N, skip_len=N)
    kv = torch.cat([mem[:, :Nm], new], 1); Nk = kv.shape[1]
    k = kv[..., :D].view(B, 1, Nk, H, 64).expand(B, n, Nk, H, 64).reshape(B * n, Nk, H, 64).permute(0, 2, 1, 3)
    v = kv[..., D:].view(B, 1, Nk, H, 64).expand(B, n, Nk, H, 64).reshape(B * n, Nk, H, 64).permute(0, 2, 1, 3)
    mask = torch.ones(B * n, 1, 1, Nk, dtype=torch.bool, device="cuda")
    for j in range(B * n): mask[j, ..., Nm + (j % n) * N: Nm + (j % n + 1) * N] = False
    ref = ref_attn(q.view(B * n, N, H, 64).permute(0, 2, 1, 3), k, v, mask)            # [Bn,H,N,64]
    o = out.float().view(B * n, N, H, 64).permute(0, 2, 1, 3)
    err = ((o - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-6))                    # [Bn,H,N]
    tot = float((o - ref).norm() / ref.norm())
    bad = (err > 0.02)
    print(f"{tag:30s} {str(dtype):15s} env={env} rel={tot:.3e} bad rows={int(bad.sum())}/{bad.numel()} nan={int(torch.isnan(o).sum())}")
    if bad.any():
        idx = bad.nonzero()
        bs = sorted(set(idx[:, 0].tolist())); hs = sorted(set(idx[:, 1].tolist()))
        rows = idx[:, 2]
        print("   bad batches", bs, "heads", hs[:12], "rows min/max", int(rows.min()), int(rows.max()), "row//128 set", sorted(set((rows // 128).tolist())))

for dt in (torch.float16, torch.bfloat16):
    for rep in range(2):
        case(dt, 1536, 2, 768, tag=f"default rep{rep}")
    for env in ({"M3R_ATTN_SPLITS": "1"}, {"M3R_ATTN_SPLITS": "2"}, {"M3R_ATTN_SPLITS": "3"}):
        case(dt, 1536, 2, 768, env=env, tag="forced")
    case(dt, 1536, 2, 768, B=1, tag="B=1")
    case(dt, 1536, 1, 768, tag="n=1")
    case(dt, 3072, 2, 768, tag="Nm=3072")
