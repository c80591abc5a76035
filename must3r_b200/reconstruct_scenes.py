"""Reconstruct several image folders at once on one GPU (engine/scenes.py), batching their memory updates and renders:

    python -m must3r_b200.reconstruct_scenes --weights CHECKPOINT --scenes DIR [DIR ...] --output OUT [...]

For folder i it writes OUT/scene_{i}/scene_{thr}.ply and OUT/scene_{i}/scene.pkl, the files
`python -m must3r_b200.reconstruct --image_dir DIR_i --output OUT/scene_{i}` writes.  The other arguments are
reconstruct's.  Only --execution_mode linseq is batched here (must3r_b200.reconstruct_videos batches vidseq and vidslam),
and the decoder's memory_mode must be 'kv'.  --max_bs is per scene:
a decoder call over S folders holds up to S * max_bs views.
"""
from __future__ import annotations

import argparse
import os
import sys

import torch

from .model import load_model
from .reconstruct import add_args, check_args, list_images, write_scene


def get_args_parser():
    parser = argparse.ArgumentParser(prog="python -m must3r_b200.reconstruct_scenes")
    return add_args(parser, lambda p: p.add_argument("--scenes", required=True, nargs="+", type=str,
                                                     help="image dirs, one per scene"))


def parse_args(argv=None):
    parser = get_args_parser()
    args = check_args(parser, parser.parse_args(argv))
    if args.execution_mode != "linseq":
        parser.error(f"--execution_mode {args.execution_mode} is not batched here: "
                     "python -m must3r_b200.reconstruct_videos batches vidseq / vidslam")
    if args.memory_mode not in (None, "kv"):
        parser.error(f"--memory_mode {args.memory_mode}: scenes are batched with memory_mode kv only")
    return args


def main(argv=None):
    from .engine.scenes import reconstruct_scenes
    args = parse_args(argv)
    filelists = [list_images(d) for d in args.scenes]
    model = load_model(args.weights, encoder=args.encoder, decoder=args.decoder, device=args.device,
                       img_size=args.image_size, memory_mode=args.memory_mode)
    scenes = reconstruct_scenes(model, args.device, args.image_size, args.amp, filelists, args.num_mem_imgs, args.max_bs,
                                init_num_images=2, batch_num_views=1, render_once=args.render_once,
                                num_refinements_iterations=args.num_refinements_iterations, verbose=True)
    for i, scene in enumerate(scenes):
        out = os.path.join(args.output, f"scene_{i}")
        os.makedirs(out, exist_ok=True)
        write_scene(scene, out, args.file_type)
    return 0


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = True
    sys.exit(main())
