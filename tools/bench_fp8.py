"""FP8 (e4m3) mode against bf16 / fp16 on the GPU, in one run:

    python tools/bench_fp8.py [--rounds 3]

1. the card and its power limit (a read-only nvidia-smi query);
2. the GEMM alone at the C3 shapes of each layer the fp8 mode changes (M = 15360 encoder / render tokens, M = 768 for a
   one-view update): m3r_gemm_e4m3 against m3r_gemm with fp16 operands, L2 flushed before every launch, CUDA events,
   TFLOP/s from 2 M N K;
3. C3 (20 views 512x384, bench.py's schedule: init 2 + 18 one-view updates + render 20 + activation) views/s in bf16 and
   fp8, alternated over --rounds rounds;
4. rel-L2 of the raw head, pts3d and conf of C3 against the unmodified reference run in fp32 on the same GPU (as
   tools/ref_gpu_parity.py), for bf16 and fp8.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from must3r_b200 import _lib, engine, synthetic as syn  # noqa: E402
from must3r_b200.model import Dust3rEncoder, MUSt3R, set_precision, ActivationType  # noqa: E402
from must3r_b200.model.common import quantize_e4m3_rows  # noqa: E402

dev = torch.device("cuda", 0)
V, H, W, SIZE = 20, 384, 512, 512
# (layer, M, N, K) of the GEMMs that take e4m3 operands in fp8 mode
SHAPES = [("enc qkv", 15360, 3072, 1024), ("enc fc1", 15360, 4096, 1024), ("dec qkv|kv (render)", 15360, 2304, 768),
          ("dec projq (render)", 15360, 768, 768), ("dec fc1 (render)", 15360, 3072, 768),
          ("dec qkv|kv (update)", 768, 3840, 768), ("dec fc1 (update)", 768, 3072, 768)]


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())


def gemm_time(M, N, K, fp8, reps=20):
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(M, K, generator=g, device=dev)
    w = torch.randn(N, K, generator=g, device=dev) / K ** 0.5
    bias = torch.zeros(N, device=dev)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    flush = torch.empty(64 << 20, dtype=torch.uint8, device=dev)           # 64 MB > the 50 MB L2
    a = _lib.GemmArgs()
    if fp8:
        A = x.clamp(-448, 448).to(torch.float8_e4m3fn)
        Wq, s = quantize_e4m3_rows(w)
        e8 = _lib.GemmE4M3Args()
        e8.a_e4m3, e8.w_scale = 1, s.data_ptr()
    else:
        A, Wq = x.half(), w.half()
    a.A, a.lda, a.W, a.ldw, a.M, a.N, a.K, a.is_bf16 = A.data_ptr(), K, Wq.data_ptr(), K, M, N, K, int(fp8)
    a.bias, a.out, a.ldc, a.out_dtype, a.w_static = bias.data_ptr(), out.data_ptr(), N, 1, 1
    lib, sp = _lib.lib(), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = (lambda: lib.m3r_gemm_e4m3(C.byref(a), C.byref(e8), sp)) if fp8 else (lambda: lib.m3r_gemm(C.byref(a), sp))
    for _ in range(3):
        _lib.check(call(), "gemm")
    ts = []
    for _ in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2] * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True).stdout.strip(), flush=True)
    torch.cuda.set_device(0)
    print("\nGEMM alone (L2 flushed, median of 20, bf16 output + bias epilogue):")
    for name, M, N, K in SHAPES:
        t16, t8 = gemm_time(M, N, K, False), gemm_time(M, N, K, True)
        f = 2.0 * M * N * K
        print(f"  {name:22s} M={M:5d} N={N:4d} K={K:4d}: fp16 {t16:7.1f} us = {f / t16 / 1e6:6.1f} TFLOP/s   "
              f"e4m3 {t8:7.1f} us = {f / t8 / 1e6:6.1f} TFLOP/s   x{t16 / t8:.2f}", flush=True)

    enc = Dust3rEncoder(img_size=(SIZE, SIZE))
    dec = MUSt3R(img_size=(SIZE, SIZE), feedback_type="single_mlp", memory_mode="kv", landscape_only=False)
    enc.load_state_dict(syn.encoder_state_dict(0))
    dec.load_state_dict(syn.decoder_state_dict(0))
    enc, dec = enc.to(dev).eval(), dec.to(dev).eval()
    imgs, ts = syn.synthetic_views(V, H, W, seed=2)
    views, tss = list(imgs.to(dev).unbind(0)), list(ts.unbind(0))
    ids = [torch.tensor(i) for i in range(V)]
    sched = [2] + [1] * (V - 2)
    raw = lambda pm: {"raw": pm}  # noqa: E731

    def job():
        feats = engine.encoder_multi_ar(enc, views, ts, device=dev, max_bs=50)
        _, pm = engine.inference_multi_ar(enc, dec, views, ids, tss, sched, encoder_precomputed_features=feats,
                                          post_process_function=raw, device=dev)
        return torch.stack([d["raw"] for d in pm]).float()

    print(f"\nC3 views/s ({V} views {W}x{H}, 5 timed jobs after 3 warm-up jobs per mode and round):")
    outs, rates = {}, {"bf16": [], "fp8": []}
    for r in range(args.rounds):
        for mode in ("bf16", "fp8"):
            set_precision(mode)
            for _ in range(3):
                outs[mode] = job()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                job()
            e1.record()
            torch.cuda.synchronize()
            rates[mode].append(V * 5 / (e0.elapsed_time(e1) / 1e3))
            print(f"  round {r} {mode}: {rates[mode][-1]:.1f} views/s", flush=True)
    for mode, v in rates.items():
        v = sorted(v)
        print(f"  {mode}: median {v[len(v) // 2]:.1f} views/s (min {v[0]:.1f}, max {v[-1]:.1f})")
    print(f"  fp8 / bf16 (medians): x{sorted(rates['fp8'])[len(v) // 2] / sorted(rates['bf16'])[len(v) // 2]:.3f}")
    set_precision(torch.float16)

    if args.no_reference:
        return
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from baseline.ref_loader import load_reference
    ref = load_reference(curope_shim=True)
    del enc, dec
    torch.cuda.empty_cache()
    renc = ref.Dust3rEncoder(img_size=(SIZE, SIZE)).eval()
    rdec = ref.MUSt3R(img_size=(SIZE, SIZE), feedback_type="single_mlp", memory_mode="kv", landscape_only=False).eval()
    renc.load_state_dict(syn.encoder_state_dict(0))
    rdec.load_state_dict(syn.decoder_state_dict(0))
    renc, rdec = renc.to(dev), rdec.to(dev)
    with torch.no_grad():
        _, rpm = ref.engine.inference_multi_ar(renc, rdec, views, ids, [t.to(dev) for t in tss], sched, max_bs=None,
                                               post_process_function=raw, device=dev)
    r_raw = torch.stack([d["raw"] for d in rpm]).float()
    r_post = ref.engine.postprocess(r_raw, ref.model.ActivationType.NORM_EXP)
    print("\nC3 against the reference in fp32 on the same GPU (rel-L2):")
    for mode in ("bf16", "fp8"):
        o = engine.postprocess(outs[mode], ActivationType.NORM_EXP)
        print(f"  {mode:5s} raw head {rel(outs[mode], r_raw):.2e}  pts3d {rel(o['pts3d'], r_post['pts3d']):.2e}  "
              f"conf {rel(o['conf'], r_post['conf']):.2e}", flush=True)


if __name__ == "__main__":
    main()
