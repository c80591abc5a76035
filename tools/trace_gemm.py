"""Timeline of the 1-CTA GEMM kernel from inside (m3r_debug_trace; needs a build made with M3R_TRACE=1).

    python tools/trace_gemm.py [M N K] [bn]
"""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import ops, _lib  # noqa: E402

M, N, K = (int(v) for v in sys.argv[1:4]) if len(sys.argv) > 3 else (768, 768, 768)
if len(sys.argv) > 4: os.environ["M3R_GEMM_BN"] = sys.argv[4]
dt = torch.bfloat16
a = torch.randn(M, K, device="cuda").to(dt); w = torch.randn(N, K, device="cuda").to(dt)
bias = torch.randn(N, device="cuda"); res = torch.randn(M, N, device="cuda")
out = torch.empty(M, N, device="cuda", dtype=torch.float32)
fn = lambda: ops.linear(a, w, bias, residual=res, out=out, w_static=True)  # noqa: E731  (the proj / fc2 form: bias + fp32 residual, fp32 out)
fn(); fn()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
lib = _lib.lib()
names = ["entry->setup done", "griddep wait", "producer: all TMA issued", "MMA: first stage landed", "MMA: last commit issued",
         "epilogue: accumulator ready", "epilogue: stores done", "exit"]
for cold in (True, False):
    buf = torch.zeros(16 * 1024, dtype=torch.int64, device="cuda")
    if cold:
        flush.zero_()
    torch.cuda.synchronize()
    lib.m3r_debug_trace(buf.data_ptr())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record(); torch.cuda.synchronize()
    lib.m3r_debug_trace(None)
    t = buf.view(-1, 16).cpu()
    t = t[t[:, 0] != 0]
    t0 = int(t[:, 0].min())
    print(f"--- M={M} N={N} K={K} {'cold' if cold else 'warm'} L2: {t.shape[0]} CTAs, span entry->last exit {(int(t[:, 9].max()) - t0) / 1e3:.2f} us")
    cols = [1, 2, 3, 4, 5, 6, 7, 9]
    for nm, c in zip(names, cols):
        d = (t[:, c] - t[:, 0]).double() / 1e3
        print(f"    {nm:30s} (since CTA entry) min/med/max {d.min():6.2f}/{d.median():6.2f}/{d.max():6.2f} us")
