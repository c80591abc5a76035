"""Streaming (video) schedule on one GPU: frames/s of engine.inference_video_multi_ar at 512x384 with the reference's
defaults (keyframe iff id % 3 == 0, rolling window of 25 frames), with and without the host label shadow that turns
the engine's memory edits into slice operations.

    python tools/bench_stream.py [frames=60] [window=25]
"""
import importlib
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import engine, synthetic as syn  # noqa: E402
from must3r_b200.model import Dust3rEncoder, MUSt3R, ActivationType, set_precision  # noqa: E402

inf = importlib.import_module("must3r_b200.engine.inference")
F = int(sys.argv[1]) if len(sys.argv) > 1 else 60
WIN = int(sys.argv[2]) if len(sys.argv) > 2 else 25
H, W = 384, 512
dev = torch.device("cuda", 0)
set_precision(torch.bfloat16)
enc = Dust3rEncoder(img_size=(512, 512))
dec = MUSt3R(img_size=(512, 512), feedback_type="single_mlp", memory_mode="kv", landscape_only=False)
enc.load_state_dict(syn.encoder_state_dict(0))
dec.load_state_dict(syn.decoder_state_dict(0))
enc, dec = enc.to(dev).eval(), dec.to(dev).eval()
imgs, ts = syn.synthetic_views(F, H, W, seed=3)
imgs = imgs.to(dev)
views, tss = list(imgs.unbind(0)), list(ts.unbind(0))
pp = lambda pm: engine.postprocess(pm, ActivationType.NORM_EXP)  # noqa: E731


def run():
    x, pos = engine.encoder_multi_ar(enc, views, ts, device=dev)
    return engine.inference_video_multi_ar(enc, dec, views, tss, [2] + [1] * (F - 2), encoder_precomputed_features=(x, pos),
                                           post_process_function=pp, device=dev, return_mem=True, local_context_size=WIN)


def timed(tag):
    run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    mem, out = run()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"{tag:34s} {F / dt:8.1f} frames/s  ({dt * 1e3 / F:.2f} ms/frame, {mem[1].shape[1] // 768} views left in memory)", flush=True)
    return mem, out


mem_a, out_a = timed("host label shadow (slice edits)")
real = inf._shadow_after_call
inf._shadow_after_call = lambda mem_before, new_mem, idx_st, x_st: new_mem
mem_b, out_b = timed("device masks (reference's edits)")
inf._shadow_after_call = real
same = torch.equal(mem_a[1], mem_b[1]) and all(torch.equal(a, b) for a, b in zip(mem_a[0], mem_b[0])) \
    and all(torch.equal(a[k], b[k]) for a, b in zip(out_a, out_b) for k in a)
print("identical results:", same)
