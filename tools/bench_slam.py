#!/usr/bin/env python
"""SLAM front end throughput on one GPU: SLAM_MUSt3R.__call__ over seeded 640x480 frames of a sliding synthetic scene
with the full-size random-weight model in bf16 at res=512 and the reference's defaults (searcher
'kdtree-scipy-quadrant_x2', overlap 'nn-norm', kf_x_subsamp=4).

    python tools/bench_slam.py [--frames 200] [--warmup 10]

Prints frames/s; the per-frame tail after the prediction (pose kernel, quadrant ids, grid query, keyframe kernel, the
record's read-back) as host time and as device time between CUDA events; the same tail composed of the existing torch
ops (engine/camera.py focal + Procrustes, keyframes.get_overlap_score) on the same predictions and map; the keyframes
and memory tokens at the end; the card's name and power limit.  One JSON line at the end.  Writes only to a temporary
directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from must3r_b200 import synthetic as syn  # noqa: E402
from must3r_b200.engine import camera, keyframes, slam  # noqa: E402
from must3r_b200.model import set_precision  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def frames(n, seed=0, H=480, W=640, step=6):
    pano = syn.synthetic_frame(H, W + step * n, seed=seed)
    return [np.ascontiguousarray(pano[:, step * i:step * i + W]) for i in range(n)]


def torch_tail(res, tree, kw):
    """The same work with the existing torch ops: focal, rectification, Procrustes, overlap score (syncs included)."""
    H, W = res['conf'].shape[-2:]
    loc = res['pts3d_local'][0]
    pp = torch.tensor((W / 2, H / 2), device=loc.device)
    focal = camera.estimate_focal_weiszfeld(loc, pp)
    loc[..., 2] *= (focal.mean() / focal)[:, None, None]
    R, t = camera.rigid_points_registration(loc.reshape(1, -1, 3), res['pts3d'][0].reshape(1, -1, 3), res['conf'][0].reshape(1, -1) - 1)
    score = keyframes.get_overlap_score(res, tree, t[0], mode=kw['overlap_mode'], kf_x_subsamp=kw['kf_x_subsamp'],
                                        min_conf_keyframe=kw['min_conf_keyframe'], percentile=kw['overlap_percentile'])
    return float(focal[0].cpu()), score, bool(res['conf'][0, 0].median() > kw['min_conf_keyframe'])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--res", type=int, default=512)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_slam needs a CUDA device"
    set_precision(torch.bfloat16)
    name, limit = card()
    imgs = frames(args.frames + args.warmup)
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "random.pth")
        dsd = syn.camera_like_head_bias(syn.decoder_state_dict(0))
        torch.save({"args": argparse.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                               decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                    "encoder": syn.encoder_state_dict(0), "decoder": dsd}, chkpt)
        s = slam.SLAM_MUSt3R(chkpt, res=args.res, device="cuda:0")

    # per-frame tail: from the prediction (forward_must3r returned) to the record on the host
    marks, keep = [], []
    fwd, wait = slam.forward_must3r, slam._wait_host_copies

    def timed_forward(*a, **k):
        out = fwd(*a, **k)
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        marks.append([time.perf_counter(), ev])
        if len(keep) < 32:
            keep.append({n: out[0][-1][n].clone() for n in ('pts3d', 'pts3d_local', 'conf')})
        return out

    def timed_wait():
        wait()
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        marks[-1] += [time.perf_counter(), ev]

    slam.forward_must3r, slam._wait_host_copies = timed_forward, timed_wait
    try:
        for i in range(args.warmup):
            s(imgs[i], i, 0)
        torch.cuda.synchronize()
        marks.clear()
        keep.clear()
        t0 = time.perf_counter()
        for i in range(args.warmup, args.warmup + args.frames):
            s(imgs[i], i, 0)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        slam.forward_must3r, slam._wait_host_copies = fwd, wait
    host_ms = [1e3 * (m[2] - m[0]) for m in marks if len(m) == 4]
    dev_ms = [m[1].elapsed_time(m[3]) for m in marks if len(m) == 4]

    # the same predictions through the torch composition, against the final map
    kw = dict(overlap_mode=s.overlap_mode, kf_x_subsamp=s.kf_x_subsamp, min_conf_keyframe=s.min_conf_keyframe,
              overlap_percentile=s.overlap_percentile)
    torch_ms = []
    for res in keep * 2:
        r = {n: v.clone() for n, v in res.items()}
        torch.cuda.synchronize()
        t = time.perf_counter()
        torch_tail(r, s.overlap_tree, kw)
        torch.cuda.synchronize()
        torch_ms.append(1e3 * (time.perf_counter() - t))
    torch_ms = torch_ms[len(keep):]
    tokens = 0 if s.memory is None else int(s.memory[0][0].shape[1])
    out = {"metric": "slam_frames_per_s", "value": round(args.frames / wall, 2), "frames": args.frames, "res": args.res,
           "tail_host_ms_median": round(float(np.median(host_ms)), 3), "tail_device_ms_median": round(float(np.median(dev_ms)), 3),
           "torch_tail_ms_median": round(float(np.median(torch_ms)), 3), "keyframes": len(s.keyframes),
           "memory_tokens": tokens, "gpu": name, "power_limit": limit}
    print(f"{name} (power limit {limit}): {out['value']} frames/s over {args.frames} frames at res {args.res}, bf16")
    print(f"tail after the prediction: {out['tail_host_ms_median']} ms host, {out['tail_device_ms_median']} ms device "
          f"(median); torch composition on the same predictions: {out['torch_tail_ms_median']} ms")
    print(f"{len(s.keyframes)} keyframes, {tokens} memory tokens")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
