"""Reconstruct a folder of images (the reference's get_reconstruction.py) on the CUDA model:

    python -m must3r_b200.reconstruct --weights CHECKPOINT --image_dir DIR --output OUT [--execution_mode linseq|vidseq|vidslam]

Writes OUT/scene_{thr}.ply, the confidence-filtered point cloud at each threshold of get_reconstruction.py (all of them
gathered on the GPU in one pass), and OUT/scene.pkl, the pickled SceneState.  The arguments are get_reconstruction.py's;
--retrieval is rejected (retrieval needs asmk and faiss, which are not vendored) and --file_type is 'ply' only (GLB
export needs trimesh).  --cam_size and --camera_conf_thr only concern the GLB's camera meshes and have no effect.
"""
from __future__ import annotations

import argparse
import os
import pickle
import sys

import torch

from .model import MEMORY_MODES, load_model


def get_args_parser():
    parser = argparse.ArgumentParser(prog="python -m must3r_b200.reconstruct")
    return add_args(parser, lambda p: p.add_argument("--image_dir", required=True, type=str, help="image dir"))


def add_args(parser, add_input):
    """get_reconstruction.py's arguments; `add_input(parser)` adds the input argument(s) after --image_size."""
    parser.add_argument("--image_size", type=int, default=512, choices=[512, 224], help="image size")

    add_input(parser)
    parser.add_argument("--output", required=True, type=str, help="output dir")

    parser.add_argument("--weights", type=str, help="path to the model weights", default=None)
    parser.add_argument("--encoder", type=str, default=None, help="encoder class instantiation")
    parser.add_argument("--decoder", type=str, default=None, help="decoder class instantiation")
    parser.add_argument("--memory_mode", type=str, default=None, choices=MEMORY_MODES,
                        help="decoder memory_mode override")

    parser.add_argument("--retrieval", type=str, default=None,
                        help="not supported: retrieval needs asmk and faiss, which are not vendored")

    parser.add_argument("--device", type=str, default='cuda', help="pytorch device")
    parser.add_argument("--amp", type=str, default=False)

    parser.add_argument("--execution_mode", type=str, default="linseq",
                        choices=["linseq", "retrieval", "vidseq", "vidslam"])

    parser.add_argument("--max_bs", type=int, default=1)
    parser.add_argument("--num_refinements_iterations", type=int, default=0)
    parser.add_argument('--render_once', action='store_true', default=False, help="skip the final rendering step")

    # linseq / retrieval params
    parser.add_argument("--num_mem_imgs", type=int, default=50)

    # vidseq /vidslam params
    parser.add_argument("--local_context_size", type=int, default=0)
    # vidseq params
    parser.add_argument("--keyframe_interval", type=int, default=3)
    # vidslam params
    parser.add_argument("--subsample", type=int, default=2)
    parser.add_argument("--min_conf_keyframe", type=float, default=1.5)
    parser.add_argument("--keyframe_overlap_thr", type=float, default=0.05)
    parser.add_argument("--overlap_percentile", type=float, default=85)

    # viz params
    parser.add_argument("--cam_size", type=float, default=0.05)
    parser.add_argument("--camera_conf_thr", type=float, default=0.0)

    parser.add_argument("--file_type", type=str, default="ply", choices=["ply"])
    return parser


def parse_args(argv=None):
    parser = get_args_parser()
    return check_args(parser, parser.parse_args(argv))


def check_args(parser, args):
    if args.retrieval is not None:
        parser.error("--retrieval is not supported: retrieval keyframes need asmk and faiss, which are not vendored")
    if args.execution_mode == "retrieval":
        parser.error("You need to provide --retrieval for execution_mode==retrieval (and --retrieval is not supported)")
    if args.amp in ("False", "false", "0", ""):
        args.amp = False
    return args


def list_images(image_dir):
    """get_reconstruction.py:75-77: every file of the directory, sorted."""
    return sorted([os.path.join(image_dir, f) for f in os.listdir(image_dir)
                   if os.path.isfile(os.path.join(image_dir, f))])


def main(argv=None):
    from .engine import demo
    args = parse_args(argv)
    images = list_images(args.image_dir)
    os.makedirs(args.output, exist_ok=True)
    model = load_model(args.weights, encoder=args.encoder, decoder=args.decoder, device=args.device,
                       img_size=args.image_size, memory_mode=args.memory_mode)
    num_mem_imgs = min(args.num_mem_imgs, len(images))
    min_conf_thr = demo.THRESHOLDS[-1]
    scene, _ = demo.get_reconstructed_scene(
        outdir=args.output, viser_server=None, should_save_glb=False, model=model, retrieval=None, device=args.device,
        verbose=True, image_size=args.image_size, amp=args.amp, filelist=images, min_conf_thr=min_conf_thr,
        as_pointcloud=True, transparent_cams=False, local_pointmaps=False, cam_size=args.cam_size,
        num_mem_images=num_mem_imgs, max_bs=args.max_bs, render_once=args.render_once,
        camera_conf_thr=args.camera_conf_thr, num_refinements_iterations=args.num_refinements_iterations,
        execution_mode=args.execution_mode, vidseq_local_context_size=args.local_context_size,
        keyframe_interval=args.keyframe_interval, slam_local_context_size=args.local_context_size,
        subsample=args.subsample, min_conf_keyframe=args.min_conf_keyframe,
        keyframe_overlap_thr=args.keyframe_overlap_thr, overlap_percentile=args.overlap_percentile)
    write_scene(scene, args.output, args.file_type)
    return 0


def write_scene(scene, output, file_type):
    """OUT/scene_{thr}.ply at every threshold of get_reconstruction.py and OUT/scene.pkl."""
    from .engine import demo
    clouds = demo.get_3D_models_from_scene(scene, demo.THRESHOLDS)
    for thr, (pts, col) in zip(demo.THRESHOLDS, clouds):
        path = os.path.join(output, f'scene_{thr}.{file_type}')
        print('(exporting 3D scene to', path, f': {pts.shape[0]} points)')
        demo.write_ply(path, pts, col)
    with open(os.path.join(output, 'scene.pkl'), 'wb') as f:
        pickle.dump(scene, f)


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = True
    sys.exit(main())
