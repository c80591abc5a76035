"""Timeline of the attention kernel from inside (m3r_debug_trace): where a launch's microseconds go.

    python tools/trace_attn.py [Nk=7680] [B=1] [splits]
"""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import ops, _lib  # noqa: E402

Nk = int(sys.argv[1]) if len(sys.argv) > 1 else 7680
B = int(sys.argv[2]) if len(sys.argv) > 2 else 1
if len(sys.argv) > 3: os.environ["M3R_ATTN_SPLITS"] = sys.argv[3]
H, Nq, D = 12, 768, 768
dt = torch.bfloat16
q = torch.randn(B * Nq, D, device="cuda").to(dt)
kv = torch.randn(B * Nk, 2 * D, device="cuda").to(dt)
fn = lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk)  # noqa: E731
fn(); fn()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
lib = _lib.lib()
for cold in (True, False):
    buf = torch.zeros(128 * 4096, dtype=torch.int64, device="cuda")
    if cold:
        flush.zero_()
    torch.cuda.synchronize()
    lib.m3r_debug_trace(buf.data_ptr())
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    lib.m3r_debug_trace(None)
    t = buf.view(-1, 128).cpu()
    t = t[t[:, 0] != 0]
    t0 = int(t[:, 0].min())
    rel = lambda v: (int(v) - t0) / 1e3  # noqa: E731
    print(f"--- Nk={Nk} B={B} {'cold' if cold else 'warm'} L2: event time {a.elapsed_time(b)*1e3:.1f} us, {t.shape[0]} CTAs, "
          f"span entry->last exit {rel(t[:, 6].max()):.1f} us")
    ent = (t[:, 0] - t0).double() / 1e3
    print(f"    CTA entry   min/med/max {ent.min():.1f}/{ent.median():.1f}/{ent.max():.1f} us")
    for nm, c0, c1 in [("prologue (entry->softmax start)", 0, 1), ("main loop", 1, 4), ("O read+store partial", 4, 5), ("merge / wait", 5, 6),
                       ("whole CTA", 0, 6)]:
        d = (t[:, c1] - t[:, c0]).double() / 1e3
        print(f"    {nm:34s} min/med/max {d.min():7.2f}/{d.median():7.2f}/{d.max():7.2f} us")
    sms = {}
    for r in t:
        sms.setdefault(int(r[2]), []).append(r)
    print(f"    SMs used {len(sms)}, CTAs per SM: " + str(sorted({len(v) for v in sms.values()})))
    # per-tile detail of the CTA with the median whole-CTA time
    order = sorted(range(t.shape[0]), key=lambda i: int(t[i, 6] - t[i, 0]))
    for tag, idx in (("median CTA", order[len(order) // 2]), ("slowest CTA", order[-1])):
        r = t[idx]
        n = min(int(r[3]), 12)
        print(f"    {tag}: sm {int(r[2])} tiles {int(r[3])}; per tile [s_full wait | S ld | o_done wait+max | exp+P st] us:")
        prev = int(r[1])
        for j in range(n):
            s = [int(v) for v in r[8 + 4 * j: 12 + 4 * j]]
            if j == 0:
                s[2] = s[1]
            mm = [int(v) for v in r[64 + 4 * j: 68 + 4 * j]]          # MMA thread: k_full ok, s_free ok (QK j+1 issued), p_full ok, PV j issued
            base = s[0]                                                # everything relative to this tile's s_full wait end
            mrel = " ".join(f"{(v - base) / 1e3:6.2f}" if v else "   n/a" for v in mm)
            print(f"      j={j:2d}: {(s[0]-prev)/1e3:6.2f} | {(s[1]-s[0])/1e3:5.2f} | {(s[2]-s[1])/1e3:5.2f} | {(s[3]-s[2])/1e3:5.2f}"
                  f"   || MMA thread rel. to S(j) ready: k_full(j+1) {mrel.split()[0]}  s_free(j)/QK(j+1) {mrel.split()[1]}  p_full(j) {mrel.split()[2]}  PV(j) issued {mrel.split()[3]}")
            prev = s[3]
