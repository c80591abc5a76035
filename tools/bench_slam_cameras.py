#!/usr/bin/env python
"""One SLAM map built by K = 1, 2, 4 cameras on one GPU: seeded 640x480 frames per camera (each its own sliding synthetic
scene), the full-size random-weight model in bf16 at res 512 with the defaults of tools/bench_slam.py, in two modes that
alternate in one run:

  batched    MultiCameraSLAM.step over every camera each step (one encoder, one decoder call against the one memory,
             one ordered keyframe commit and one wait per step)
  sequential SLAM_MUSt3R with one agent per camera, fed the same frames in the reference's order, one at a time

    python tools/bench_slam_cameras.py [--frames 200] [--warmup 10] [--cameras 1 2 4] [--rounds 2]

Prints the aggregate frames/s of each mode (the best of --rounds alternated runs, and every run); for the batched mode
the median device time of a step (CUDA events) split into encoder, decoder, the per-frame tails and the commit, up to the
step's one wait; the keyframe counts of both modes; the card and its power limit.  One JSON line at the end.  Writes only
to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_slam import card, frames  # noqa: E402
from must3r_b200 import synthetic as syn  # noqa: E402
from must3r_b200.engine import slam  # noqa: E402
from must3r_b200.engine import slam_cameras as scm  # noqa: E402
from must3r_b200.model import set_precision  # noqa: E402


def ev():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def run_batched(chkpt, seqs, warmup, res):
    K, n = len(seqs), len(seqs[0])
    mc = scm.MultiCameraSLAM(chkpt, K, device="cuda:0", res=res)
    enc = mc.model[0]
    marks = []
    fwd, dec, com = enc.forward, scm.MultiCameraSLAM._decode_shared, scm.commit_ordered

    def timed_encoder(*a, **k):
        marks.append([ev()])
        out = fwd(*a, **k)
        marks[-1].append(ev())
        return out

    def timed_decode(self, *a, **k):
        out = dec(self, *a, **k)
        marks[-1].append(ev())
        return out

    def timed_commit(*a, **k):
        marks[-1].append(ev())
        com(*a, **k)
        marks[-1].append(ev())

    enc.forward, scm.MultiCameraSLAM._decode_shared, scm.commit_ordered = timed_encoder, timed_decode, timed_commit
    try:
        for k in range(warmup):
            mc.step({c: (seq[k], k * K + c) for c, seq in enumerate(seqs)})
        torch.cuda.synchronize()
        marks.clear()
        t0 = time.perf_counter()
        for k in range(warmup, n):
            mc.step({c: (seq[k], k * K + c) for c, seq in enumerate(seqs)})
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        del enc.forward
        scm.MultiCameraSLAM._decode_shared, scm.commit_ordered = dec, com
    full = [m for m in marks if len(m) == 5]
    split = {name: round(float(np.median([m[i].elapsed_time(m[i + 1]) for m in full])), 3) if full else None
             for i, name in enumerate(("encoder_ms", "decoder_ms", "tail_ms", "commit_ms"))}
    return (n - warmup) * K / wall, split, mc


def run_sequential(chkpt, seqs, warmup, res):
    K, n = len(seqs), len(seqs[0])
    mc = scm.MultiCameraSLAM(chkpt, K, device="cuda:0", res=res)        # its SLAM_MUSt3R, on the same model
    for k in range(warmup):
        for c, seq in enumerate(seqs):
            slam.SLAM_MUSt3R.__call__(mc.slam, seq[k], k * K + c, c)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(warmup, n):
        for c, seq in enumerate(seqs):
            slam.SLAM_MUSt3R.__call__(mc.slam, seq[k], k * K + c, c)
    torch.cuda.synchronize()
    return (n - warmup) * K / (time.perf_counter() - t0), mc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--cameras", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_slam_cameras needs a CUDA device"
    set_precision(torch.bfloat16)
    name, limit = card()
    print(f"{name} (power limit {limit})", flush=True)
    results = []
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "random.pth")
        dsd = syn.camera_like_head_bias(syn.decoder_state_dict(0))
        torch.save({"args": argparse.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                               decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                    "encoder": syn.encoder_state_dict(0), "decoder": dsd}, chkpt)
        all_seqs = [frames(args.frames + args.warmup, seed=i) for i in range(max(args.cameras))]
        for K in args.cameras:
            seqs = all_seqs[:K]
            fbs, fss = [], []
            for _ in range(args.rounds):
                fb, split, mb = run_batched(chkpt, seqs, args.warmup, args.res)
                fbs.append(round(fb, 2))
                print(f"K={K} batched: {fb:.2f} frames/s", flush=True)
                fs, ms = run_sequential(chkpt, seqs, args.warmup, args.res)
                fss.append(round(fs, 2))
                print(f"K={K} sequential: {fs:.2f} frames/s", flush=True)
                kb, ks = len(mb.keyframes), len(ms.keyframes)
                alone = mb.stats["alone"]
                del mb, ms
                torch.cuda.empty_cache()
            r = {"cameras": K, "batched_fps": max(fbs), "sequential_fps": max(fss), "batched_runs": fbs,
                 "sequential_runs": fss, **split, "keyframes_batched": kb, "keyframes_sequential": ks,
                 "batched_alone_frames": alone}
            results.append(r)
            print(f"K={K}: batched {r['batched_fps']} frames/s (runs {fbs}), sequential {r['sequential_fps']} (runs {fss}); "
                  f"batched step device ms: encoder {split['encoder_ms']}, decoder {split['decoder_ms']}, tail "
                  f"{split['tail_ms']}, commit {split['commit_ms']}; keyframes {kb} (sequential {ks})", flush=True)
    print(f"{name} (power limit {limit}), {args.frames} timed frames per camera at res {args.res}, bf16")
    print(json.dumps({"metric": "slam_cameras_frames_per_s", "results": results, "gpu": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
