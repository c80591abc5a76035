"""Reconstruct several videos (image folders in sequence order) at once on one GPU (engine/videos.py), batching their
frames, memory updates and rolling-window edits:

    python -m must3r_b200.reconstruct_videos --weights CHECKPOINT --scenes DIR [DIR ...] --output OUT \
        --execution_mode vidseq|vidslam [...]

For folder i it writes OUT/scene_{i}/scene_{thr}.ply and OUT/scene_{i}/scene.pkl, the files
`python -m must3r_b200.reconstruct --image_dir DIR_i --output OUT/scene_{i} --execution_mode M` writes.  The other
arguments are reconstruct's.  --execution_mode linseq is batched by must3r_b200.reconstruct_scenes instead, and the
decoder's memory_mode must be 'kv'.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

from .model import load_model
from .reconstruct import add_args, check_args, list_images, write_scene


def get_args_parser():
    parser = argparse.ArgumentParser(prog="python -m must3r_b200.reconstruct_videos")
    return add_args(parser, lambda p: p.add_argument("--scenes", required=True, nargs="+", type=str,
                                                     help="image dirs, one per video"))


def parse_args(argv=None):
    parser = get_args_parser()
    args = check_args(parser, parser.parse_args(argv))
    if args.execution_mode not in ("vidseq", "vidslam"):
        parser.error(f"--execution_mode {args.execution_mode}: videos are batched in vidseq or vidslam (pass "
                     "--execution_mode vidseq|vidslam); python -m must3r_b200.reconstruct_scenes batches linseq")
    if args.memory_mode not in (None, "kv"):
        parser.error(f"--memory_mode {args.memory_mode}: videos are batched with memory_mode kv only")
    return args


def main(argv=None):
    from .engine.videos import reconstruct_videos
    args = parse_args(argv)
    filelists = [list_images(d) for d in args.scenes]
    model = load_model(args.weights, encoder=args.encoder, decoder=args.decoder, device=args.device,
                       img_size=args.image_size, memory_mode=args.memory_mode)
    scenes = reconstruct_videos(model, args.device, args.image_size, args.amp, filelists, args.execution_mode,
                                args.max_bs, local_context_size=args.local_context_size,
                                keyframe_interval=args.keyframe_interval, subsample=args.subsample,
                                min_conf_keyframe=args.min_conf_keyframe, keyframe_overlap_thr=args.keyframe_overlap_thr,
                                overlap_percentile=args.overlap_percentile,
                                num_refinements_iterations=args.num_refinements_iterations, verbose=True)
    for i, scene in enumerate(scenes):
        out = os.path.join(args.output, f"scene_{i}")
        os.makedirs(out, exist_ok=True)
        write_scene(scene, out, args.file_type)
    return 0


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = True
    sys.exit(main())
