"""Keyframe point-map query: the grid index (engine/keyframes.py PointGrid) against the brute-force scan (nn_min_dist).

The map is what the SLAM front end accumulates: per keyframe, the 256x192 points (512x384 frames at kf_x_subsamp=2) a
camera sees of the walls of an 8 x 6 x 3 m room, with depth-proportional noise, along a circular camera path.  The
query is the next frame on the path (overlapping the last keyframes), with all its points (Q = 49152) or a quarter of
them (Q = 12288).  P ~ 49k to 4.9M = 1 to 100 keyframes.  Times are CUDA events around the query only; the
index build (on each add, once per keyframe) is timed separately.  Every index result is checked bitwise against the
brute force.  The same sizes are also run on maps made of the pointmaps of the full-size model with random weights
(one bucket), whose distribution is nothing like a room: the cell size is chosen from the data.  For one bucket the
table also times `DeviceNN.query`, which picks brute force or the index from the map size.

Usage: python tools/bench_pointgrid.py [--reps 10] [--sizes 1,2,4,10,100] [--no-model]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200.engine import keyframes as kf  # noqa: E402

ROOM = (8.0, 6.0, 3.0)
W, H = 256, 192


def camera(k):
    phi = 2 * math.pi * k / 40.0
    c = torch.tensor([ROOM[0] / 2 + 1.5 * math.cos(phi), ROOM[1] / 2 + 1.5 * math.sin(phi), 1.5 + 0.2 * math.sin(3 * phi)])
    return c, phi + math.pi / 2 + 0.3 * math.sin(2 * phi)


def frame(k, seed):
    """Points of the room's walls seen by camera k (pinhole, 60 degree horizontal field of view)."""
    c, yaw = camera(k)
    f = (W / 2) / math.tan(math.radians(30))
    v, u = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    dc = torch.stack([(u - W / 2) / f, (v - H / 2) / f, torch.ones_like(u)], -1).reshape(-1, 3)
    right = torch.tensor([math.sin(yaw), -math.cos(yaw), 0.0], dtype=torch.float64)
    down = torch.tensor([0.0, 0.0, -1.0], dtype=torch.float64)
    fwd = torch.tensor([math.cos(yaw), math.sin(yaw), 0.0], dtype=torch.float64)
    d = dc[:, :1] * right + dc[:, 1:2] * down + dc[:, 2:] * fwd
    lim = torch.where(d > 0, torch.tensor(ROOM, dtype=torch.float64), torch.zeros(3, dtype=torch.float64))
    t = ((lim - c.double()) / d).masked_fill(d == 0, math.inf).amin(-1)
    p = c.double() + t[:, None] * d
    g = torch.Generator().manual_seed(seed)
    p = p + torch.randn(p.shape, generator=g, dtype=torch.float64) * (0.005 * t[:, None])
    return p.float(), c


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    ms.sort()
    return ms[len(ms) // 2]


def card():
    r = {"gpu": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        r["power_limit_and_max_sm_clock"] = out[0] if out else "not reported"
    except (OSError, subprocess.SubprocessError):
        r["power_limit_and_max_sm_clock"] = "not reported"
    return r


def model_frames(n):
    """Pointmaps (pts3d at kf_x_subsamp=2) of n synthetic 512x384 frames from the full-size model with random weights,
    run through the streaming schedule in bf16."""
    from must3r_b200 import engine, synthetic as syn
    from must3r_b200.model import ActivationType, Dust3rEncoder, MUSt3R, set_precision
    dev = torch.device("cuda", 0)
    set_precision(torch.bfloat16)
    enc = Dust3rEncoder(img_size=(512, 512))
    dec = MUSt3R(img_size=(512, 512), feedback_type="single_mlp", memory_mode="kv", landscape_only=False)
    enc.load_state_dict(syn.encoder_state_dict(0))
    dec.load_state_dict(syn.decoder_state_dict(0))
    enc, dec = enc.to(dev).eval(), dec.to(dev).eval()
    imgs, ts = syn.synthetic_views(n, 2 * H, 2 * W, seed=3)
    views, tss = list(imgs.to(dev).unbind(0)), list(ts.unbind(0))
    out = engine.inference_video_multi_ar(enc, dec, views, tss, [2] + [1] * (n - 2),
                                          post_process_function=lambda pm: engine.postprocess(pm, ActivationType.NORM_EXP),
                                          device=dev)
    frames = [r["pts3d"].to(dev).reshape(-1, 2 * H, 2 * W, 3)[0, ::2, ::2].reshape(-1, 3).float().contiguous() for r in out]
    del enc, dec
    return frames


def run_case(name, frames, qall, reps, cams=None, cq=None):
    """Index (one bucket; and 32 quadrant buckets when camera centres are given) against brute force, Q = 49152 / 12288."""
    pts = torch.cat(frames)
    for quads in ((0, 4) if cams is not None else (0,)):
        grid = kf.PointGrid(2 * quads ** 2 if quads else 1)
        ids_of = (lambda x, c: kf.get_quadrant_id(x - c[None], quads)) if quads else None
        for i, f in enumerate(frames):
            grid.add(f, ids_of(f, cams[i]) if quads else None)

        def build():
            grid._grid = None
            grid._build(pts.device)
        build_ms = timed(build, max(3, reps // 3))
        for Q in (49152, 12288):
            q = qall[:: 49152 // Q].contiguous()
            qid = ids_of(q, cq) if quads else None
            got = grid.query(q, qid)
            if quads:
                pid = torch.cat([ids_of(f, c) for f, c in zip(frames, cams)])
                want = torch.empty_like(got)
                for b in range(grid.nb):
                    sel = qid == b
                    if sel.any():
                        want[sel] = kf.nn_min_dist(q[sel], pts[pid == b])
            else:
                want = kf.nn_min_dist(q, pts)
            exact = bool(torch.equal(got.view(torch.int32), want.view(torch.int32)))
            row = {"map": name, "P": pts.shape[0], "Q": Q, "buckets": grid.nb,
                   "index_ms": round(timed(lambda: grid.query(q, qid), reps), 4), "build_ms": round(build_ms, 3),
                   "cell_size": grid._grid[4], "cells": grid._grid[1].shape[0], "exact": exact,
                   "median_dist": float(got.median())}
            if not quads:
                row["brute_ms"] = round(timed(lambda: kf.nn_min_dist(q, pts), max(3, reps // 3)), 4)
                nn = kf.DeviceNN()
                for f in frames:
                    nn.add_pts(f)
                row["DeviceNN_ms"] = round(timed(lambda: nn.query(q), reps), 4)
                row["DeviceNN_uses"] = "brute force" if nn.uses_brute_force() else "index"
            print(json.dumps(row), flush=True)
            if not exact:
                raise SystemExit("index and brute force disagree")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--sizes", default="1,2,4,10,100", help="keyframes in the map (x 49152 points)")
    ap.add_argument("--no-model", action="store_true", help="skip the maps made of the random-weight model's pointmaps")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pointgrid needs a CUDA device")
    print(json.dumps(card()), flush=True)
    sizes = [int(s) for s in args.sizes.split(",")]
    for K in sizes:
        frames = [frame(k, k) for k in range(K)]
        qall, cq = frame(K, 10_000 + K)
        run_case("room", [p.cuda() for p, _ in frames], qall.cuda(), args.reps, [c.cuda() for _, c in frames], cq.cuda())
    if not args.no_model:
        mf = model_frames(max(sizes) + 1)
        for K in sizes:
            run_case("model", mf[:K], mf[K], args.reps)


if __name__ == "__main__":
    main()
