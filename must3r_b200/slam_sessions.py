"""Run several independent online SLAM sessions headless on one GPU, one folder of frames per session, their frames
batched into one encoder and one decoder call per step (engine/slam_sessions.py):

    python -m must3r_b200.slam_sessions --chkpt CHECKPOINT --sessions DIR [DIR ...] --output OUT [--res 512] ...

Takes the processing arguments of `python -m must3r_b200.slam` with the same names and defaults (--res, --skip_every,
--rerender, --rerender_bs, --filter, --searcher, --overlap_mode, --subsamp, --keyframe_overlap_thr, --min_conf_keyframe,
--overlap_percentile, --varying_focals, --num_init_frames, --image_string).  Session i reads folder i as
`python -m must3r_b200.slam --input DIR` would (its frames in name order, the first len // skip_every of them, timestamps
multiplied by skip_every); every step gives each session that has frames left its next frame, and the run stops when
every session's frames are used up.  Each session writes what that command writes, under OUT/session_{i}/:
all_poses.npz (or the --filter file) with `fps` (all sessions' frames over the wall time of the loop and the rerenders),
`gpumem` and `imgHWs`, then memory.pkl.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch

from . import slam as single
from .engine.frames import AutoMultiLoader, ReadAhead, image_size, schedule
from .engine.slam_sessions import SLAMSessions

PROCESSING = ('chkpt', 'device', 'image_string', 'output', 'res', 'skip_every', 'rerender', 'rerender_bs', 'filter',
              'searcher', 'overlap_mode', 'subsamp', 'keyframe_overlap_thr', 'min_conf_keyframe', 'overlap_percentile',
              'varying_focals', 'num_init_frames')


def get_args_parser():
    parser = argparse.ArgumentParser(prog="python -m must3r_b200.slam_sessions")
    for action in single.get_args_parser()._actions:
        if action.dest in PROCESSING:
            parser._add_action(action)
    parser.add_argument('--sessions', required=True, nargs='+', help="One folder of frames per session.")
    return parser


def parse_args(argv=None):
    parser = get_args_parser()
    args = parser.parse_args(argv)
    if args.output is None:
        parser.error("--output is required: the run only writes its results")
    for d in args.sessions:
        if not os.path.isdir(d):
            parser.error(f"--sessions {d}: no such folder")
    single.check_device_and_skip(parser, args)
    return args


def main(argv=None):
    """-> the poses file of every session."""
    args = parse_args(argv)
    device = single.resolve_device(args.device)
    S = len(args.sessions)
    model = SLAMSessions(args.chkpt, S, device=str(device), res=args.res, kf_x_subsamp=args.subsamp,
                         searcher=args.searcher, overlap_mode=args.overlap_mode,
                         keyframe_overlap_thr=args.keyframe_overlap_thr, min_conf_keyframe=args.min_conf_keyframe,
                         overlap_percentile=args.overlap_percentile, rerender=args.rerender, keep_memory=True,
                         fixed_focal=not args.varying_focals, num_agents=1, num_init_frames=args.num_init_frames)
    plans = []
    for d in args.sessions:
        items, trailing = schedule(AutoMultiLoader([d], args.image_string), args.skip_every)
        print(f"Found {len(items)} frames to process in {d}")
        plans.append((items, trailing))
    outdirs = [os.path.join(args.output, f"session_{i}") for i in range(S)]
    for o in outdirs:
        os.makedirs(o, exist_ok=True)
    imgHWs = [[] for _ in range(S)]
    n_frames = sum(len(items) for items, _ in plans)
    with torch.cuda.device(device):
        readers = [ReadAhead([p for p, _, _ in items], device) for items, _ in plans]
        try:
            start = time.time()
            for k in range(max(len(items) for items, _ in plans)):
                step = {}
                for i, (items, _) in enumerate(plans):
                    if k < len(items):
                        _, cam_id, ts = items[k]
                        frame = readers[i].get()
                        imgHWs[i].append(tuple(int(x) for x in frame.shape[:2]))
                        step[i] = (frame, ts, cam_id)
                model.step(step)
        finally:
            for r in readers:
                r.close()
        for i, (_, trailing) in enumerate(plans):
            if trailing is not None:
                imgHWs[i].append(image_size(trailing))
        if args.rerender:
            for s in model.sessions:
                s.rerender_all_frames(maxbs=args.rerender_bs)
        fps = n_frames / (time.time() - start)
        gpumem = torch.cuda.max_memory_allocated(device) / single.MB
    print(f"Done @{fps}fps on average over {S} sessions using {gpumem}MB GPU Memory "
          f"({model.stats['batched']} frames batched, {model.stats['alone']} alone)")
    outfiles = []
    for i, s in enumerate(model.sessions):
        print(f"session {i}: {len(s.keyframes)} keyframes: {s.keyframes}")
        outfiles.append(single.write_poses(s, outdirs[i], args.filter, fps=fps, gpumem=gpumem, imgHWs=imgHWs[i]))
        s.save_memory(os.path.join(outdirs[i], "memory.pkl"))
    return outfiles


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = True
    main()
    sys.exit(0)
