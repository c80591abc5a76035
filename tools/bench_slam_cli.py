#!/usr/bin/env python
"""`python -m must3r_b200.slam` throughput on one GPU: 200 seeded 640x480 JPEG frames of a sliding synthetic scene, the
full-size random-weight model in bf16, --res 512 --subsamp 4 and the other defaults of the reference's slam.py.

    python tools/bench_slam_cli.py [--frames 200] [--rounds 2]

Reports the run's own `fps` (frames over the wall time of the frame loop) with the frames decoded on a host thread
ahead of use (ReadAhead, the command line's default) and with every frame decoded before the clock starts (the
reference's preload), alternating the two in each round after one untimed warm-up run; for the read-ahead, the share of
the frame loop the consumer spent waiting for the decoder thread (ReadAhead.wait_s); whether the poses of two runs are
equal, across the two modes and across two runs of one mode; the card's name and power limit.  One JSON line at the end.
Writes only to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_slam import card, frames  # noqa: E402
from must3r_b200 import slam as cli, synthetic as syn  # noqa: E402
from must3r_b200.model import set_precision  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_slam_cli needs a CUDA device"
    set_precision(torch.bfloat16)
    name, limit = card()
    import PIL.Image
    with tempfile.TemporaryDirectory() as d:
        img_dir = os.path.join(d, "frames")
        os.makedirs(img_dir)
        for i, im in enumerate(frames(args.frames)):
            PIL.Image.fromarray(im).save(os.path.join(img_dir, f"{i:05d}.jpg"), quality=90)
        chkpt = os.path.join(d, "random.pth")
        dsd = syn.camera_like_head_bias(syn.decoder_state_dict(0))
        torch.save({"args": argparse.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                               decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                    "encoder": syn.encoder_state_dict(0), "decoder": dsd}, chkpt)

        readers = []

        class Recorded(cli.ReadAhead):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                readers.append(self)
        cli.ReadAhead = Recorded

        def run(read_ahead):
            out = os.path.join(d, "out")
            path = cli.main(["--chkpt", chkpt, "--input", img_dir, "--output", out, "--res", "512", "--subsamp", "4"],
                            read_ahead=read_ahead)
            z = np.load(path, allow_pickle=True)
            return float(z["fps"]), z["poses"]

        run(True)                                   # warm-up: module loads, tables, allocator
        fps = {"read_ahead": [], "preload": []}
        waits = []
        poses = {"read_ahead": [], "preload": []}
        for r in range(args.rounds):
            for mode in (("read_ahead", "preload") if r % 2 == 0 else ("preload", "read_ahead")):
                f, p = run(mode == "read_ahead")
                poses[mode].append(p)
                fps[mode].append(round(f, 2))
                if mode == "read_ahead":        # waiting time over the loop's wall time (frames / fps)
                    waits.append(round(readers[-1].wait_s / (args.frames / f), 4))
    same = bool(np.array_equal(poses["read_ahead"][0], poses["preload"][0]))
    repeat = bool(np.array_equal(poses["preload"][0], poses["preload"][-1]))
    res = {"metric": "slam_cli_frames_per_s", "value": float(np.median(fps["read_ahead"])),
           "preload_value": float(np.median(fps["preload"])), "runs": fps, "read_ahead_wait_share": waits,
           "frames": args.frames, "res": 512, "subsamp": 4, "poses_equal": same, "preload_repeat_poses_equal": repeat, "gpu": name, "power_limit": limit}
    print(f"{name} (power limit {limit}): {args.frames} 640x480 JPEG frames at res 512, bf16: "
          f"{res['value']} frames/s with read-ahead, {res['preload_value']} frames/s decoding every frame first "
          f"(runs {fps}); share of the loop waiting for the decoder thread: {waits}; poses equal across modes: {same}, across two preload runs: {repeat}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
