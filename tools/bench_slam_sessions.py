#!/usr/bin/env python
"""Several SLAM sessions on one GPU: S = 1, 2, 4, 8 sessions of seeded 640x480 frames (each its own sliding synthetic
scene), the full-size random-weight model in bf16 at res 512 with the defaults of tools/bench_slam.py, in three modes:

  batched    SLAMSessions.step over every session each step (one encoder and one ragged decoder call per step)
  sequential the same sessions stepped one after another in one thread (SLAM_MUSt3R.__call__ per frame)
  threads    S host threads, each on its own CUDA stream, each running its session's frames

    python tools/bench_slam_sessions.py [--frames 200] [--warmup 10] [--sessions 1 2 4 8]

Prints the aggregate frames/s of each mode; for the batched mode the median device time of a step (CUDA events) split
into encoder, decoder and the per-session tail up to the step's one wait; keyframes and memory tokens per session at the
end; the card and its power limit.  One JSON line at the end.  Writes only to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import threading
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_slam import card, frames  # noqa: E402
from must3r_b200 import synthetic as syn  # noqa: E402
from must3r_b200.engine import slam  # noqa: E402
from must3r_b200.engine.inference import _PENDING_HOST_COPIES, _d2h_stream  # noqa: E402
from must3r_b200.engine import slam_sessions as ssm  # noqa: E402
from must3r_b200.model import set_precision  # noqa: E402


def tokens(s):
    return 0 if s.memory is None else int(s.memory[0][0].shape[1])


def run_batched(chkpt, seqs, warmup, res):
    ss = ssm.SLAMSessions(chkpt, len(seqs), device="cuda:0", res=res)
    enc = ss.model[0]
    marks = []
    fwd, dec, wait = enc.forward, ssm.SLAMSessions._decode, slam._wait_host_copies

    def ev():
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        return e

    def timed_encoder(*a, **k):
        marks.append([ev()])
        out = fwd(*a, **k)
        marks[-1].append(ev())
        return out

    def timed_decode(self, *a, **k):
        out = dec(self, *a, **k)
        marks[-1].append(ev())
        return out

    def timed_wait():
        if len(marks[-1]) == 3:                 # a batched step's wait, not that of a frame run alone (no decode mark)
            marks[-1].append(ev())
        wait()

    enc.forward, ssm.SLAMSessions._decode, slam._wait_host_copies = timed_encoder, timed_decode, timed_wait
    try:
        n = len(seqs[0])
        for k in range(warmup):
            ss.step({i: (seq[k], k, 0) for i, seq in enumerate(seqs)})
        torch.cuda.synchronize()
        marks.clear()
        t0 = time.perf_counter()
        for k in range(warmup, n):
            ss.step({i: (seq[k], k, 0) for i, seq in enumerate(seqs)})
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        del enc.forward
        ssm.SLAMSessions._decode, slam._wait_host_copies = dec, wait
    full = [m for m in marks if len(m) == 4]
    split = {name: round(float(np.median([m[i].elapsed_time(m[i + 1]) for m in full])), 3) if full else None
             for i, name in enumerate(("encoder_ms", "decoder_ms", "tail_ms"))}
    return (n - warmup) * len(seqs) / wall, split, ss


def run_sequential(chkpt, seqs, warmup, res):
    ss = ssm.SLAMSessions(chkpt, len(seqs), device="cuda:0", res=res)
    n = len(seqs[0])
    for k in range(warmup):
        for i, seq in enumerate(seqs):
            slam.SLAM_MUSt3R.__call__(ss[i], seq[k], k, 0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(warmup, n):
        for i, seq in enumerate(seqs):
            slam.SLAM_MUSt3R.__call__(ss[i], seq[k], k, 0)
    torch.cuda.synchronize()
    return (n - warmup) * len(seqs) / (time.perf_counter() - t0), ss


def run_threads(chkpt, seqs, warmup, res):
    ss = ssm.SLAMSessions(chkpt, len(seqs), device="cuda:0", res=res)
    n = len(seqs[0])
    dev = torch.device("cuda:0")
    wait = slam._wait_host_copies
    # the read-back bookkeeping is one process-wide list: each thread waits for the (shared) read-back stream itself
    slam._wait_host_copies = lambda: _d2h_stream(dev).synchronize()
    barrier = threading.Barrier(len(seqs) + 1)

    errors = []

    def worker(i):
        try:
            st = torch.cuda.Stream(device=dev)
            with torch.cuda.device(dev), torch.cuda.stream(st):
                for k in range(warmup):
                    slam.SLAM_MUSt3R.__call__(ss[i], seqs[i][k], k, 0)
                st.synchronize()
                barrier.wait()
                barrier.wait()
                for k in range(warmup, n):
                    slam.SLAM_MUSt3R.__call__(ss[i], seqs[i][k], k, 0)
                st.synchronize()
        except BaseException as e:                     # noqa: BLE001  (reported by the main thread)
            errors.append(e)
            barrier.abort()

    th = [threading.Thread(target=worker, args=(i,)) for i in range(len(seqs))]
    try:
        for t in th:
            t.start()
        barrier.wait()
        t0 = time.perf_counter()
        barrier.wait()
        for t in th:
            t.join()
        wall = time.perf_counter() - t0
    except threading.BrokenBarrierError:
        for t in th:
            t.join()
        raise errors[0] if errors else RuntimeError("a worker thread failed")
    finally:
        slam._wait_host_copies = wait
        _PENDING_HOST_COPIES.clear()
    return (n - warmup) * len(seqs) / wall, ss


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--sessions", type=int, nargs="+", default=[1, 2, 4, 8])
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_slam_sessions needs a CUDA device"
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
        all_seqs = [frames(args.frames + args.warmup, seed=i) for i in range(max(args.sessions))]
        for S in args.sessions:
            seqs = all_seqs[:S]
            fb, split, sb = run_batched(chkpt, seqs, args.warmup, args.res)
            print(f"S={S} batched: {fb:.2f} frames/s", flush=True)
            fs, sq = run_sequential(chkpt, seqs, args.warmup, args.res)
            print(f"S={S} sequential: {fs:.2f} frames/s", flush=True)
            ft, stt = run_threads(chkpt, seqs, args.warmup, args.res)
            print(f"S={S} threads: {ft:.2f} frames/s", flush=True)
            r = {"sessions": S, "batched_fps": round(fb, 2), "sequential_fps": round(fs, 2), "threads_fps": round(ft, 2),
                 **split, "keyframes": [len(s.keyframes) for s in sb.sessions],
                 "memory_tokens": [tokens(s) for s in sb.sessions],
                 "keyframes_sequential": [len(s.keyframes) for s in sq.sessions],
                 "batched_alone_frames": sb.stats["alone"]}
            results.append(r)
            print(f"S={S}: batched {r['batched_fps']} frames/s, sequential {r['sequential_fps']}, threads {r['threads_fps']}; "
                  f"batched step device ms: encoder {split['encoder_ms']}, decoder {split['decoder_ms']}, tail "
                  f"{split['tail_ms']}; keyframes {r['keyframes']} (sequential {r['keyframes_sequential']}), "
                  f"memory tokens {r['memory_tokens']}", flush=True)
            del sb, sq, stt
            torch.cuda.empty_cache()
    print(f"{name} (power limit {limit}), {args.frames} timed frames per session at res {args.res}, bf16")
    print(json.dumps({"metric": "slam_sessions_frames_per_s", "results": results, "gpu": name, "power_limit": limit}))


if __name__ == "__main__":
    main()
