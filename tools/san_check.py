"""Small problems through every kernel family, for compute-sanitizer (memcheck / racecheck / synccheck)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import ops, synthetic as syn
from must3r_b200.model import Dust3rEncoder, MUSt3R, set_precision
set_precision(torch.float16)
dt = torch.float16
a = torch.randn(300, 256, device="cuda").to(dt); w = torch.randn(512, 256, device="cuda").to(dt)
ops.linear(a, w, torch.randn(512, device="cuda"), act="gelu")
os.environ["M3R_GEMM_BN"] = "256"; ops.linear(a, w, None, out_dtype=torch.float32); os.environ.pop("M3R_GEMM_BN")
q = torch.randn(2 * 300, 3 * 128, device="cuda").to(dt)
ops.attention(q[:, :128], q[:, 128:256], q[:, 256:], B=2, H=2, Nq=300, Nk0=300)
os.environ["M3R_ATTN_SPLITS"] = "2"
ops.attention(q[:, :128], q[:, 128:256], q[:, 256:], B=2, H=2, Nq=300, Nk0=300)
os.environ.pop("M3R_ATTN_SPLITS")
enc = Dust3rEncoder(img_size=(64, 64), embed_dim=128, depth=1, num_heads=2).cuda()
dec = MUSt3R(img_size=(64, 64), enc_embed_dim=128, embed_dim=128, depth=2, num_heads=2, feedback_type="single_mlp", memory_mode="kv", landscape_only=False).cuda()
imgs, ts = syn.synthetic_views(3, 32, 48)
x, pos = enc(imgs.cuda(), ts.cuda())
mem, _ = dec(x[None, :2], pos[None, :2], ts[None, :2], None)
mem, _ = dec(x[None, 2:], pos[None, 2:], ts[None, 2:], mem)
dec(x[None], pos[None], ts[None], mem, render=True)
torch.cuda.synchronize()
print("sanitizer workload done")
