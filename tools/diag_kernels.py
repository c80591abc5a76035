"""Bring-up diagnostics for the wgmma kernels: structured inputs that localise descriptor / layout mistakes.
Prints one line per probe; never asserts.  Run on the GPU box: python tools/diag_kernels.py"""
import os
import sys
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import ops  # noqa: E402


def err(a, b):
    a, b = a.float(), b.float()
    return f"max|d|={float((a - b).abs().max()):.3e} rel={float((a - b).norm() / b.norm().clamp_min(1e-30)):.3e}"


def gemm_probes(dtype):
    dev = "cuda"
    for bn in (64, 128, 256):
        os.environ["M3R_GEMM_BN"] = str(bn)
        M, N, K = 128, 256, 64
        eye = torch.eye(M, K, device=dev, dtype=dtype)              # A = [I;0] -> out[:64] = W^T[:64]
        w = torch.randn(N, K, device=dev).to(dtype)
        out = ops.linear(eye, w, None, out_dtype=torch.float32)
        print(f"gemm[{dtype},BN={bn}] A=eye 1 k-block :", err(out[:K], w.float().t()), "| rows>=64 zero:", float(out[K:].abs().max()))
        a = torch.randn(M, K, device=dev).to(dtype)
        out = ops.linear(a, w, None, out_dtype=torch.float32)
        print(f"gemm[{dtype},BN={bn}] random 128x256x64 :", err(out, a.float() @ w.float().t()))
        M, N, K = 256, 512, 512
        a = torch.randn(M, K, device=dev).to(dtype); w = torch.randn(N, K, device=dev).to(dtype)
        out = ops.linear(a, w, None, out_dtype=torch.float32)
        print(f"gemm[{dtype},BN={bn}] random 256x512x512:", err(out, a.float() @ w.float().t()))
    os.environ.pop("M3R_GEMM_BN", None)


def attn_ref(q, k, v):
    s = (q.float() @ k.float().t()) * 0.125
    return torch.softmax(s, -1) @ v.float()


def attn_probes(dtype):
    dev = "cuda"
    N = 128
    q = torch.randn(N, 64, device=dev).to(dtype)
    k = torch.randn(N, 64, device=dev).to(dtype)
    v = torch.randn(N, 64, device=dev).to(dtype)
    z = torch.zeros_like(k)
    dcol = torch.arange(64, device=dev).float().expand(N, 64).contiguous().to(dtype) / 64
    krow = (torch.arange(N, device=dev).float()[:, None].expand(N, 64) / N).contiguous().to(dtype)

    def run(q_, k_, v_, n=N):
        return ops.attention(q_, k_, v_, B=1, H=1, Nq=n, Nk0=n)
    print(f"attn[{dtype}] K=0, V=const-per-col (expect V row):", err(run(q, z, dcol), dcol))
    print(f"attn[{dtype}] K=0, V=random (expect col means)  :", err(run(q, z, v), v.float().mean(0, keepdim=True).expand(N, 64)))
    print(f"attn[{dtype}] QK random, V=const-per-col        :", err(run(q, k, dcol), dcol))
    print(f"attn[{dtype}] QK random, V=key index            :", err(run(q, k, krow), attn_ref(q, k, krow)))
    print(f"attn[{dtype}] full random, 1 tile               :", err(run(q, k, v), attn_ref(q, k, v)))
    N2 = 384
    q2 = torch.randn(N2, 64, device=dev).to(dtype); k2 = torch.randn(N2, 64, device=dev).to(dtype); v2 = torch.randn(N2, 64, device=dev).to(dtype)
    print(f"attn[{dtype}] full random, 3x3 tiles            :", err(run(q2, k2, v2, N2), attn_ref(q2, k2, v2)))
    N3 = 200
    q3, k3, v3 = q2[:N3].contiguous(), k2[:N3].contiguous(), v2[:N3].contiguous()
    print(f"attn[{dtype}] full random, ragged N=200         :", err(run(q3, k3, v3, N3), attn_ref(q3, k3, v3)))


if __name__ == "__main__":
    torch.manual_seed(0)
    which = sys.argv[1:] or ["gemm", "attn"]
    for dt in (torch.float16, torch.bfloat16):
        for w in which:
            try:
                (gemm_probes if w == "gemm" else attn_probes)(dt)
                torch.cuda.synchronize()
            except Exception as e:  # noqa: BLE001
                print(f"{w}[{dt}] FAILED: {type(e).__name__}: {e}")
                sys.exit(2)
