"""Run the online SLAM front end headless over folders of frames (the reference's slam.py without its GUI) on the CUDA
model:

    python -m must3r_b200.slam --chkpt CHECKPOINT --input DIR [DIR ...] --output OUT [--res 512] [--subsamp 4]
                               [--skip_every K] [--rerender] [--filter] [--load_memory MEM.pkl] [--varying_focals]

Writes OUT/all_poses.npz (or, with --filter, OUT/all_poseslaplacian_256-steps_0.1-alpha.npz: the camera centres after 256
Laplacian smoothing sweeps with alpha 0.1) through SLAM_MUSt3R.write_all_poses, with the extra arrays `fps`, `gpumem`
(peak allocated device memory in MB) and `imgHWs` (frame sizes), then the final memory, OUT/memory.pkl, through
save_memory, which --load_memory reads back in a later run.

The arguments, their defaults and the run are those of must3r/slam/slam.py:main.  SLAM_MUSt3R gets keep_memory=True,
fixed_focal=not --varying_focals and one agent per --input folder.  With several folders the frames alternate between
them (engine/frames.py); frame_id * skip_every is each frame's timestamp.  As in the reference, whose main assigns
SKIP_EVERY to a local name that its grab_frame never sees, --skip_every skips no frame: the run takes the first
len(frames) // skip_every frames in order and multiplies their timestamps by skip_every.

`fps` is the reference's: the frames processed over the wall time of the frame loop plus --rerender.  The reference
decodes every frame before the clock starts; here one host thread decodes a few frames ahead into pinned buffers
(engine/frames.py ReadAhead) while the GPU works, so decoding overlaps inside that window and host memory does not grow
with the sequence.  The loop adds no synchronisation to SLAM_MUSt3R's one wait per frame.

Rejected with a message: --gui (the viewer needs open3d), a missing --output (the reference asserts it without the GUI),
camera streams (cam:N) and video files (decoding them needs cv2, which this package does not use), a --device that is not
CUDA.  --viz_conf and --hide_cameras only concern the GUI and have no effect; --force_first_keyframes is parsed and
never read, as in the reference.

Deliberate difference: when --load_memory is OUT/memory.pkl, the reference writes the memory to OUT/memory_0.pkl, over
an earlier memory_0.pkl if there is one, and it only recognises the loaded file by the exact string OUT/memory.pkl.  Here
the two paths are compared after resolving them (so ./OUT/memory.pkl or a link to it count too), and the memory goes to
OUT/memory_{count}.pkl with the first count whose file does not exist, so no earlier memory file is overwritten.
"""
from __future__ import annotations

import argparse
import os
import sys
import time

import torch

from .engine.frames import AutoMultiLoader, ReadAhead, decode, image_size, schedule
from .engine.slam import SLAM_MUSt3R

MB = 1024. ** 2
FILTERING_MODE, FILTERING_ALPHA, FILTERING_STEPS = 'laplacian', .1, 256


def get_args_parser():
    parser = argparse.ArgumentParser(prog="python -m must3r_b200.slam")
    parser.add_argument('--chkpt', required=True, help='Path to checkpoint.')
    parser.add_argument('--device', default='cuda:0', help='CUDA device to run on (e.g. "cuda:0").')
    parser.add_argument('--input', default='cam:0', nargs='+',
                        help="Folders of frames, one per camera (camera streams and video files are not supported).")
    parser.add_argument('--image_string', default=None, type=str,
                        help="In the case of an image collection, string to identify image files.")
    parser.add_argument('--load_memory', default=None, type=str, help="Load memory from another run.")
    parser.add_argument('--output', default=None, type=str, help="Output directory to write predictions")

    # Processing related opts
    parser.add_argument('--res', default=224, choices=[224, 512],
                        type=int, help="Image resolution that works for the model used.")
    parser.add_argument('--skip_every', default=1, type=int,
                        help="Timestamp step; as in the reference, the first len(frames) // skip_every frames are used.")
    parser.add_argument('--rerender', action='store_true', default=False, help="Rerender all frames at the end.")
    parser.add_argument('--rerender_bs', default=64, type=int, help="Re-rendering batch size")
    parser.add_argument('--filter', action='store_true', default=False, help="Minimal Laplacian filtering after rerender.")

    # Hyperparams
    parser.add_argument('--searcher', default="kdtree-scipy-quadrant_x2", type=str,
                        help="Method for overlap prediction")
    parser.add_argument('--overlap_mode', default="nn-norm", type=str,
                        help="How to estimate overlap")
    parser.add_argument('--subsamp', default=2, type=int)
    parser.add_argument('--keyframe_overlap_thr', default=.1, type=float,
                        help="At least this overlap to add incoming image in memory")
    parser.add_argument('--min_conf_keyframe', default=1.2, type=float, help="Ignore 3D points below this confidence.")
    parser.add_argument('--overlap_percentile', default=85., type=float,
                        help="Percentile of image distances to compute overlap")
    parser.add_argument('--varying_focals', action='store_true', default=False,
                        help="Focals may vary along sequence (e.g. zoom-in/out).")

    parser.add_argument('--force_first_keyframes', default=None, type=int, help="Parsed and not used (as in the reference).")
    parser.add_argument('--num_init_frames', default=2, type=int)

    # GUI related opts
    parser.add_argument('--viz_conf', default=4., type=float, help="GUI only: no effect.")
    parser.add_argument('--gui', action='store_true', default=False, help="Not supported: the viewer needs open3d.")
    parser.add_argument('--hide_cameras', action='store_true', default=False, help="GUI only: no effect.")
    return parser


def parse_args(argv=None):
    parser = get_args_parser()
    args = parser.parse_args(argv)
    if args.gui:
        parser.error("--gui is not supported: the viewer needs open3d")
    if args.output is None:
        parser.error("--output is required: without the GUI the run only writes its results (You should define an "
                     "output folder)")
    inputs = [args.input] if isinstance(args.input, str) else args.input
    for inp in inputs:
        if 'cam:' in inp:
            parser.error(f"--input {inp}: camera streams are not supported (they need cv2)")
        if os.path.isfile(inp):
            parser.error(f"--input {inp}: video files are not supported (they need cv2); give a folder of frames")
        if not os.path.isdir(inp):
            parser.error(f"--input {inp}: no such folder")
    check_device_and_skip(parser, args)
    return args


def check_device_and_skip(parser, args):
    """Reject through `parser` a --device that is not a CUDA device and a --skip_every below 1."""
    try:
        dev = torch.device(args.device)
    except RuntimeError:
        parser.error(f"--device {args.device}: not a device")
    if dev.type != 'cuda':
        parser.error(f"--device {args.device}: must3r_b200 runs on CUDA devices only")
    if args.skip_every < 1:
        parser.error("--skip_every must be at least 1")


def resolve_device(name):
    """The CUDA device `name` names, with the current device's index when it has none."""
    device = torch.device(name)
    if device.index is None:
        device = torch.device('cuda', torch.cuda.current_device())
    return device


def write_poses(model, output, filtered, **tolog):
    """model.write_all_poses into OUTPUT/all_poses.npz, or when `filtered` the Laplacian-smoothed poses into
    OUTPUT/all_poses{mode}_{steps}-steps_{alpha}-alpha.npz -> the file's path."""
    if not filtered:
        outfile = os.path.join(output, 'all_poses.npz')
        model.write_all_poses(outfile, **tolog)
    else:
        outfile = os.path.join(output, f"all_poses{FILTERING_MODE}_{FILTERING_STEPS}-steps_{FILTERING_ALPHA}-alpha.npz")
        model.write_all_poses(outfile, filtering_mode=FILTERING_MODE, filtering_steps=FILTERING_STEPS,
                              filtering_alpha=FILTERING_ALPHA, **tolog)
    return outfile


def memory_path(output, load_memory=None):
    """OUT/memory.pkl, or OUT/memory_{count}.pkl with the first count whose file does not exist when the memory was
    loaded from OUT/memory.pkl (compared as resolved paths).  The reference writes OUT/memory_0.pkl in that case, over an
    earlier one, and compares the path strings."""
    outname = os.path.join(output, "memory.pkl")
    if load_memory is None or os.path.realpath(load_memory) != os.path.realpath(outname):
        return outname
    count = 0
    while os.path.exists(os.path.join(output, f"memory_{count}.pkl")):
        count += 1
    return os.path.join(output, f"memory_{count}.pkl")


class Preloaded:
    """Every frame decoded up front, as the reference's ImageCollection preloads them; `get()` returns the next one.
    Only `main(read_ahead=False)` uses it, for tools/bench_slam_cli.py's comparison: no command-line option selects it."""

    def __init__(self, paths):
        self.frames = [decode(p) for p in paths]
        self._next = 0

    def get(self):
        self._next += 1
        return self.frames[self._next - 1]

    def close(self):
        pass


def run_frames(model, items, frames, trailing=None):
    """Feed `items` [(path, cam_id, timestamp)] to `model` (SLAM_MUSt3R) in order, taking the frames from `frames`
    (ReadAhead or Preloaded over the items' paths) -> the frame sizes (H, W) the reference records: every fed frame's,
    then that of `trailing`, the frame read after the last one, if there is one (read from its header, not decoded)."""
    imgHWs = []
    for _, cam_id, ts in items:
        frame = frames.get()
        imgHWs.append(tuple(int(x) for x in frame.shape[:2]))
        model(frame, ts, cam_id)
    if trailing is not None:
        imgHWs.append(image_size(trailing))
    return imgHWs


def main(argv=None, read_ahead=True):
    """The reference's headless main (must3r/slam/slam.py:568-693) -> the path of the poses file.  read_ahead=False
    decodes every frame before the clock starts, as the reference does; it exists for tools/bench_slam_cli.py's
    comparison, and no command-line option selects it."""
    args = parse_args(argv)
    device = resolve_device(args.device)
    model = SLAM_MUSt3R(chkpt=args.chkpt,
                        res=args.res,
                        kf_x_subsamp=args.subsamp,
                        searcher=args.searcher,
                        overlap_mode=args.overlap_mode,
                        keyframe_overlap_thr=args.keyframe_overlap_thr,
                        min_conf_keyframe=args.min_conf_keyframe,
                        overlap_percentile=args.overlap_percentile,
                        rerender=args.rerender,
                        keep_memory=args.output is not None,
                        load_memory=args.load_memory,
                        fixed_focal=not args.varying_focals,
                        num_agents=len(args.input),
                        device=str(device),
                        num_init_frames=args.num_init_frames,
                        )
    camera = AutoMultiLoader(args.input, args.image_string)
    for d, cam in zip(args.input, camera.CAMERAS):
        print(f"Found {len(cam)} frames in {d}")
    os.makedirs(args.output, exist_ok=True)

    items, trailing = schedule(camera, args.skip_every)
    print(f"Start processing sequence of {len(camera)} frames")
    paths = [p for p, _, _ in items]
    with torch.cuda.device(device):
        frames = ReadAhead(paths, device) if read_ahead else Preloaded(paths)
        try:
            start = time.time()
            imgHWs = run_frames(model, items, frames, trailing)
        finally:
            frames.close()
        if args.rerender:
            model.rerender_all_frames(maxbs=args.rerender_bs)
        wallclock_time = time.time() - start
        fps = len(items) / wallclock_time
        gpumem = torch.cuda.max_memory_allocated(device) / MB
    print(f"Done @{fps}fps on average using {gpumem}MB GPU Memory")
    print(f"{len(model.keyframes)} keyframes: {model.keyframes}")
    outfile = write_poses(model, args.output, args.filter, fps=fps, gpumem=gpumem, imgHWs=imgHWs)
    outname = memory_path(args.output, args.load_memory)
    print(f"Dumping memory as {outname}")
    model.save_memory(outname)
    return outfile


if __name__ == '__main__':
    torch.backends.cuda.matmul.allow_tf32 = True
    main()
    sys.exit(0)
