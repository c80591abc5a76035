"""Run one online SLAM map built by several cameras headless, their frames batched into one encoder and one decoder call
per step (engine/slam_cameras.py):

    python -m must3r_b200.slam_cameras --chkpt CHECKPOINT --input DIR [DIR ...] --output OUT [--res 512] ...

The arguments, their defaults, their checks, the frame schedule, the read-ahead, the output files and `fps` are those of
`python -m must3r_b200.slam`: one camera per --input folder, its frames taken in the reference's order (camera 0, 1, ...,
skipping a camera that has run out), timestamps frame_id * skip_every over that order.  A step is the next frame of
every camera that still has frames (engine/slam_cameras.py steps_of).  The run writes OUT/all_poses.npz (or the --filter
file) with `fps` (frames over the wall time of the loop), `gpumem` and `imgHWs`, then OUT/memory.pkl (memory_path).

Rejected besides what `python -m must3r_b200.slam` rejects: --rerender with more than one folder, which the reference
rejects too (rerender_all_frames supports one agent only).  The one difference from `python -m must3r_b200.slam` over
the same folders is the step semantics of engine/slam_cameras.py: a frame does not see a keyframe taken earlier in its
step.
"""
from __future__ import annotations

import os
import sys
import time

import torch

from . import slam as single
from .engine.frames import AutoMultiLoader, ReadAhead, image_size, schedule
from .engine.slam_cameras import MAX_CAMERAS, MultiCameraSLAM, steps_of


def parse_args(argv=None):
    """`python -m must3r_b200.slam`'s parser and checks, then the checks of a shared-map run."""
    args = single.parse_args(argv)
    if len(args.input) > MAX_CAMERAS:
        single.get_args_parser().error(f"--input: at most {MAX_CAMERAS} folders")
    if args.rerender and len(args.input) > 1:
        single.get_args_parser().error("--rerender with several --input folders is not supported (the reference's "
                                       "rerender_all_frames takes one agent only)")
    return args


def run_steps(model, items, frames, trailing=None):
    """Feed `items` [(path, cam_id, timestamp)] to `model` (MultiCameraSLAM) step by step, taking the frames from
    `frames` in item order -> the frame sizes (H, W), as single.run_frames records them."""
    imgHWs = []
    for step in steps_of(items):
        batch = {}
        for _, cam_id, ts in step:
            frame = frames.get()
            imgHWs.append(tuple(int(x) for x in frame.shape[:2]))
            batch[cam_id] = (frame, ts)
        model.step(batch)
    if trailing is not None:
        imgHWs.append(image_size(trailing))
    return imgHWs


def main(argv=None):
    """-> the path of the poses file."""
    args = parse_args(argv)
    device = single.resolve_device(args.device)
    model = MultiCameraSLAM(args.chkpt, len(args.input), device=str(device),
                            res=args.res,
                            kf_x_subsamp=args.subsamp,
                            searcher=args.searcher,
                            overlap_mode=args.overlap_mode,
                            keyframe_overlap_thr=args.keyframe_overlap_thr,
                            min_conf_keyframe=args.min_conf_keyframe,
                            overlap_percentile=args.overlap_percentile,
                            rerender=args.rerender,
                            keep_memory=True,
                            load_memory=args.load_memory,
                            fixed_focal=not args.varying_focals,
                            num_init_frames=args.num_init_frames)
    camera = AutoMultiLoader(args.input, args.image_string)
    for d, cam in zip(args.input, camera.CAMERAS):
        print(f"Found {len(cam)} frames in {d}")
    os.makedirs(args.output, exist_ok=True)

    items, trailing = schedule(camera, args.skip_every)
    print(f"Start processing sequence of {len(camera)} frames")
    with torch.cuda.device(device):
        frames = ReadAhead([p for p, _, _ in items], device)
        try:
            start = time.time()
            imgHWs = run_steps(model, items, frames, trailing)
        finally:
            frames.close()
        if args.rerender:
            model.rerender_all_frames(maxbs=args.rerender_bs)
        fps = len(items) / (time.time() - start)
        gpumem = torch.cuda.max_memory_allocated(device) / single.MB
    print(f"Done @{fps}fps on average using {gpumem}MB GPU Memory "
          f"({model.stats['batched']} frames batched, {model.stats['alone']} alone)")
    print(f"{len(model.keyframes)} keyframes: {model.keyframes}")
    outfile = single.write_poses(model.slam, args.output, args.filter, fps=fps, gpumem=gpumem, imgHWs=imgHWs)
    outname = single.memory_path(args.output, args.load_memory)
    print(f"Dumping memory as {outname}")
    model.save_memory(outname)
    return outfile


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = True
    main()
    sys.exit(0)
