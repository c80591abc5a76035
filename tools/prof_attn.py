"""Stand-alone timing of the attention / GEMM kernels at the shapes of the C3 job (CUDA events, L2 flushed between
iterations by a 256 MB write).  `python tools/prof_attn.py [attn|gemm] [--once] [--compare] [--fp16]`; --once runs each shape
twice for ncu; --compare also times each attention shape at the key-split count of the earlier rule (old_splits); --fp16
uses fp16 operands instead of bf16."""
import os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import ops  # noqa: E402

once = "--once" in sys.argv
compare = "--compare" in sys.argv
warm = "--warm" in sys.argv      # do not flush L2 between iterations (operands stay L2-resident like inside a step)
which = [a for a in sys.argv[1:] if not a.startswith("--")] or ["attn", "gemm"]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, iters=10):
    fn(); fn()
    if once:
        torch.cuda.synchronize(); return 0.0
    ts = []
    for _ in range(iters):
        if not warm:
            flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def old_splits(B, H, Nq, Nk, sms):
    """Key splits of the earlier rule (CTAs of 128 or 256 query rows, split counts tuned for 148 SMs), for one key
    segment of Nk keys: what --compare forces through M3R_ATTN_SPLITS."""
    key_tiles = -(-Nk // 128)
    ctas2, ctas1 = -(-Nq // 256) * H * B, -(-Nq // 128) * H * B
    qt = 2 if (Nq > 128 and 2 * ctas2 >= sms) else 1
    long_keys = qt == 1 and Nq > 128 and key_tiles >= 384 and ctas2 < sms
    qt = 2 if long_keys else qt
    splits = 1
    if qt == 1 and ctas1 < 2 * sms:
        splits = min((2 * sms + ctas1 // 2) // ctas1, key_tiles // 4)
    elif qt == 2 and long_keys:
        splits = (sms + ctas2 // 2) // ctas2
    elif qt == 2 and key_tiles >= 64:
        eff = lambda sp: ctas2 * sp / (-(-ctas2 * sp // sms) * sms)  # noqa: E731
        best = eff(1)
        for sp in range(2, 5):
            if key_tiles // sp >= 16 and eff(sp) > best + 0.04:
                best, splits = eff(sp), sp
    splits = max(1, min(splits, key_tiles, 32))
    if B * H * -(-Nq // 128) > 16384:
        splits = 1
    chunk = -(-key_tiles // splits)
    return -(-key_tiles // chunk)


dt = torch.float16 if "--fp16" in sys.argv else torch.bfloat16
if "attn" in which:
    for name, (B, H, Nq, Nk, grp) in {
        "render CA 20 views x M=20": (20, 12, 768, 15360, 20),
        "render CA 4 views x M=20": (4, 12, 768, 15360, 4),
        "update CA 1 view x M=10": (1, 12, 768, 7680, 1),
        "update CA 1 view x M=19": (1, 12, 768, 14592, 1),
        "decoder SA 1 view": (1, 12, 768, 768, 1),
        "encoder SA 20 views": (20, 16, 768, 768, 1),
        "C2 decoder SA 10 views 224": (10, 12, 196, 196, 1),
        "C2 render CA 10 views 224": (10, 12, 196, 1960, 10),
        "C4 render CA 100 views x M=100": (100, 12, 768, 76800, 100),
        "C4 update CA 1 view x M=99": (1, 12, 768, 76032, 1),
        "C5 update CA 1 view x M=360": (1, 12, 768, 276480, 1),
    }.items():
        D = H * 64
        q = torch.randn(B * Nq, D, device="cuda").to(dt)
        nb = B // grp if grp > 1 else B
        kv = torch.randn(nb * Nk, 2 * D, device="cuda").to(dt)
        fn = lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk, kv_group=grp if grp > 1 else 1)  # noqa: E731
        ms = timeit(fn)
        fl = 4.0 * B * H * Nq * Nk * 64
        if compare:
            sp_old = old_splits(B, H, Nq, Nk, torch.cuda.get_device_properties(0).multi_processor_count)
            ms_old = float("inf")
            for _ in range(2):                  # alternate, best of two each: the first timing of a shape runs slow
                os.environ["M3R_ATTN_SPLITS"] = str(sp_old)
                ms_old = min(ms_old, timeit(fn))
                os.environ.pop("M3R_ATTN_SPLITS")
                ms = min(ms, timeit(fn))
            print(f"attn {name:28s} {ms*1e3:9.1f} us  {fl/ms/1e9 if ms else 0:8.1f} TFLOP/s | earlier split rule (s={sp_old}) {ms_old*1e3:9.1f} us", flush=True)
            continue
        print(f"attn {name:28s} {ms*1e3:9.1f} us  {fl/ms/1e9 if ms else 0:8.1f} TFLOP/s", flush=True)
if "upd" in which:           # the one-view update cross-attention alone (ncu target)
    B, H, Nq, Nk = 1, 12, 768, 7680
    D = H * 64
    q = torch.randn(B * Nq, D, device="cuda").to(dt)
    kv = torch.randn(B * Nk, 2 * D, device="cuda").to(dt)
    ms = timeit(lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk))
    print(f"attn update CA 1 view x M=10 {ms*1e3:9.1f} us  {4.0*B*H*Nq*Nk*64/ms/1e9 if ms else 0:8.1f} TFLOP/s", flush=True)
if "g64" in which:           # the one-view 768x768x768 GEMM (proj / q / cproj form) alone (ncu target)
    M = N = K = 768
    a = torch.randn(M, K, device="cuda").to(dt); w = torch.randn(N, K, device="cuda").to(dt)
    bias = torch.randn(N, device="cuda"); res = torch.randn(M, N, device="cuda"); out = torch.empty(M, N, device="cuda")
    ms = timeit(lambda: ops.linear(a, w, bias, residual=res, out=out, w_static=True))
    print(f"gemm one-view proj 768x768x768 (+bias +fp32 residual) {ms*1e3:9.1f} us  {2.0*M*N*K/ms/1e9 if ms else 0:8.1f} TFLOP/s", flush=True)
if "gemm" in which:
    for name, (M, N, K) in {
        "enc qkv 20v": (15360, 3072, 1024), "enc proj 20v": (15360, 1024, 1024), "enc fc1 20v": (15360, 4096, 1024),
        "enc fc2 20v": (15360, 1024, 4096), "dec qkv 20v": (15360, 2304, 768), "dec fc1 20v": (15360, 3072, 768),
        "dec fc2 20v": (15360, 768, 3072), "dec head 20v": (15360, 1792, 768),
        "dec qkv 1v": (768, 2304, 768), "dec proj 1v": (768, 768, 768), "dec kv 1v": (768, 1536, 768),
        "dec fc1 1v": (768, 3072, 768), "dec fc2 1v": (768, 768, 3072),
    }.items():
        a = torch.randn(M, K, device="cuda").to(dt); w = torch.randn(N, K, device="cuda").to(dt)
        out = torch.empty(M, N, device="cuda", dtype=dt)
        ms = timeit(lambda: ops.linear(a, w, None, out=out, w_static=True))
        print(f"gemm {name:14s} M={M:6d} N={N:5d} K={K:5d} {ms*1e3:9.1f} us  {2.0*M*N*K/ms/1e9 if ms else 0:8.1f} TFLOP/s", flush=True)

if "sweep" in which:
    shapes = {"update CA 1v M=10": (1, 12, 768, 7680), "update CA 1v M=19": (1, 12, 768, 14592), "update CA 1v M=3": (1, 12, 768, 2304),
              "decoder SA 1v": (1, 12, 768, 768), "SA 224 1v": (1, 12, 196, 196), "CA 224 1v M=9": (1, 12, 196, 1764)}
    for name, (B, H, Nq, Nk) in shapes.items():
        D = H * 64
        q = torch.randn(B * Nq, D, device="cuda").to(dt)
        kv = torch.randn(B * Nk, 2 * D, device="cuda").to(dt)
        res = []
        for sp in (1, 2, 3, 4, 6, 8, 12, 16):
            os.environ["M3R_ATTN_SPLITS"] = str(sp)
            ms = timeit(lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk), iters=7)
            res.append((ms, sp))
        os.environ.pop("M3R_ATTN_SPLITS")
        ms0 = timeit(lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk), iters=7)
        res.sort()
        print(f"sweep {name:20s} default {ms0*1e3:7.1f} us | best " + "  ".join(f"s{s_}:{m*1e3:.1f}" for m, s_ in res[:5]), flush=True)

if "longmem" in which:       # one-view update cross-attention against long memories (C4: up to 100 views, C5: ~360)
    for M_ in (20, 50, 100, 200):
        B, H, Nq, Nk = 1, 12, 768, 768 * M_
        D = H * 64
        q = torch.randn(B * Nq, D, device="cuda").to(dt)
        kv = torch.randn(B * Nk, 2 * D, device="cuda").to(dt)
        res = []
        for sp in (2, 4, 6, 8, 12, 16, 24):
            os.environ["M3R_ATTN_SPLITS"] = str(sp)
            ms = timeit(lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk), iters=5)
            res.append((ms, sp))
        os.environ.pop("M3R_ATTN_SPLITS")
        ms0 = timeit(lambda: ops.attention(q, kv[:, :D], kv[:, D:], B=B, H=H, Nq=Nq, Nk0=Nk), iters=5)
        res.sort()
        fl = 4.0 * B * H * Nq * Nk * 64
        print(f"longmem 1v x M={M_:3d} default {ms0*1e3:8.1f} us ({fl/ms0/1e9:6.1f} TF/s) | best " + "  ".join(f"s{s_}:{m*1e3:.1f}us({fl/m/1e9:.0f})" for m, s_ in res[:4]), flush=True)

if "bnsweep" in which:       # tile width of the one-wave GEMMs of the one-view / two-view steps (warm L2, like inside a step)
    import os as _os
    for name, (M, N, K, act) in {"merged qkv|kv 1v": (768, 3840, 768, "none"), "fc1 1v": (768, 3072, 768, "gelu"), "q 1v": (768, 768, 768, "none"),
                                 "head 1v": (768, 1792, 768, "none"), "merged 2v": (1536, 3840, 768, "none"), "fc1 2v": (1536, 3072, 768, "gelu"),
                                 "merged 224 1v": (196, 3840, 768, "none"), "fc1 224 1v": (196, 3072, 768, "gelu")}.items():
        a = torch.randn(M, K, device="cuda").to(dt); w = (torch.randn(N, K, device="cuda") / 28).to(dt)
        out = torch.empty(M, N, device="cuda", dtype=torch.float32 if name.startswith("head") else dt)
        res = []
        for bn in (32, 64, 128, 160, 192, 256):
            if N % bn: continue
            _os.environ["M3R_GEMM_BN"] = str(bn)
            res.append((timeit(lambda: ops.linear(a, w, None, act=act, out=out, w_static=True), iters=15), bn))
        _os.environ.pop("M3R_GEMM_BN")
        ms0 = timeit(lambda: ops.linear(a, w, None, act=act, out=out, w_static=True), iters=15)
        print(f"bnsweep {name:16s} M={M} N={N} K={K}: default {ms0*1e3:.1f}us | " + "  ".join(f"BN{b}:{m*1e3:.1f}" for m, b in res), flush=True)

if "small" in which:
    import os as _os
    for name, (M, N, K) in {"dec qkv 1v": (768, 2304, 768), "dec proj 1v": (768, 768, 768), "dec kv 1v": (768, 1536, 768),
                            "dec fc1 1v": (768, 3072, 768), "dec fc2 1v": (768, 768, 3072), "224 proj 1v": (196, 768, 768), "224 fc1 1v": (196, 3072, 768)}.items():
        a = torch.randn(M, K, device="cuda").to(dt); w = torch.randn(N, K, device="cuda").to(dt)
        out = torch.empty(M, N, device="cuda", dtype=dt)
        res = []
        for bn in (64, 128, 256):
            if N % bn: continue
            _os.environ["M3R_GEMM_BN"] = str(bn)
            res.append((timeit(lambda: ops.linear(a, w, None, out=out, w_static=True), iters=15), bn))
        _os.environ.pop("M3R_GEMM_BN")
        print(f"small gemm {name:12s} M={M} N={N} K={K}: " + "  ".join(f"BN{b}:{m*1e3:.1f}us" for m, b in res), flush=True)
    x = torch.randn(768, 768, device="cuda"); g = torch.ones(768, device="cuda"); b = torch.zeros(768, device="cuda")
    print(f"layernorm 768x768 -> 16 bit: {timeit(lambda: ops.layernorm(x, g, b, 1e-6, out_dtype=dt), iters=15)*1e3:.1f} us", flush=True)
    x = torch.randn(15360, 768, device="cuda")
    print(f"layernorm 15360x768 -> 16 bit: {timeit(lambda: ops.layernorm(x, g, b, 1e-6, out_dtype=dt), iters=15)*1e3:.1f} us", flush=True)
