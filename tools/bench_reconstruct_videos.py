#!/usr/bin/env python
"""Several videos on one GPU (must3r_b200/engine/videos.py) against one video after another.

    python tools/bench_reconstruct_videos.py [--scenes 1 2 4 8] [--frames 200] [--rounds 2] [--modes ...]

Per video count S: S folders of seeded synthetic 512x384 PNG frames (a panorama sliding right, each video from its own
seed), the full-size random-weight model in bf16 at image_size 512, get_reconstruction.py's defaults otherwise (max_bs 1,
no refinement).  Modes: vidseq at local_context_size 0 and 25 (keyframe_interval 3), and vidslam with the command line's
defaults.  Per mode, two runs alternate in rounds: `reconstruct_videos` over all S videos, and
`get_reconstructed_scene` once per video in one thread.  Reports the aggregate frames/s of each (best round, from the
file lists to the SceneStates on the host), the median device time of the batched run's encoder, memory steps (decoder
calls and commits), compaction, keyframe tail (vidslam: searcher queries, keyframe kernels, the read-back wait and the
searcher updates) and postprocess (CUDA events at the engine's phase boundaries, summed over the steps), per video the
keyframe counts of both runs and the largest pts3d relative L2 between them, the card's name and power limit, and one
JSON line.  Writes only to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from must3r_b200 import synthetic as syn  # noqa: E402
from must3r_b200.engine import demo, videos  # noqa: E402
from must3r_b200.model import load_model, set_precision  # noqa: E402
from bench_reconstruct import card  # noqa: E402
from bench_reconstruct_scenes import write_frames  # noqa: E402

PHASES = ("encode", "memory", "compact", "keyframes", "postprocess")
MODES = {"vidseq_window0": ("vidseq", 0), "vidseq_window25": ("vidseq", 25), "vidslam": ("vidslam", 0)}


class PhaseEvents:
    """Replaces videos._phase: one CUDA event per phase boundary of a batched run; a phase's time is the sum of its
    stretches."""

    def __init__(self):
        self.marks = []

    def __call__(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.marks.append((name, e))

    def times_ms(self):
        out = {p: 0.0 for p in PHASES}
        for (name, a), (_, b) in zip(self.marks, self.marks[1:]):
            out[name] += a.elapsed_time(b)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--modes", nargs="+", default=list(MODES), choices=list(MODES))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_reconstruct_videos needs a CUDA device"
    set_precision(torch.bfloat16)
    name, limit = card()
    res = {"frames": args.frames, "gpu": name, "power_limit": limit, "runs": {}}
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "random.pth")
        dsd = syn.camera_like_head_bias(syn.decoder_state_dict(0))
        torch.save({"args": argparse.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                               decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                    "encoder": syn.encoder_state_dict(0), "decoder": dsd}, chkpt)
        model = load_model(chkpt, device="cuda", img_size=512, verbose=False)
        lists = [write_frames(os.path.join(d, f"s{i}"), args.frames, seed=i) for i in range(max(args.scenes))]
        keyframes = []

        class Recorded(videos.VideoPlan):
            def __init__(self, *a, **k):
                super().__init__(*a, **k)
                keyframes.append(self.keyframes)
        videos.VideoPlan = Recorded

        def batched(mode, context, S, phase=None):
            keyframes.clear()
            videos._phase = phase or (lambda n: None)
            try:
                out = videos.reconstruct_videos(model, "cuda", 512, False, lists[:S], mode, 1,
                                                local_context_size=context, verbose=False)
            finally:
                videos._phase = lambda n: None
            return out, [len(k) for k in keyframes]

        orig_video = demo.inference_video_multi_ar

        def sequential(mode, context, fls):
            out, counts = [], []
            for fl in fls:
                n = [min(2, len(fl))]

                def counting(*a, **k):
                    f = k["is_keyframe_function"]

                    def kf(id, r, state):
                        v = bool(f(id, r, state))
                        n[0] += v
                        return v
                    k["is_keyframe_function"] = kf
                    return orig_video(*a, **k)
                demo.inference_video_multi_ar = counting
                try:
                    scene, _ = demo.get_reconstructed_scene(
                        None, None, False, model, None, "cuda", False, 512, False, fl, 1, 0, mode, num_mem_images=50,
                        render_once=False, vidseq_local_context_size=context, keyframe_interval=3,
                        slam_local_context_size=context, subsample=2, min_conf_keyframe=1.5, keyframe_overlap_thr=0.05,
                        overlap_percentile=85.0, min_conf_thr=1.05, as_pointcloud=True, transparent_cams=False,
                        local_pointmaps=False, cam_size=0.05)
                finally:
                    demo.inference_video_multi_ar = orig_video
                out.append(scene)
                counts.append(n[0])
            return out, counts

        # warm both paths on short videos (module loads, allocator, workspaces)
        short = [fl[:8] for fl in lists[:2]]
        for mode, context in MODES.values():
            videos.reconstruct_videos(model, "cuda", 512, False, short, mode, 1, local_context_size=context, verbose=False)
            sequential(mode, context, short[:1])
        for key in args.modes:
            mode, context = MODES[key]
            for S in args.scenes:
                t_b, t_s, phases = [], [], []
                out_b = out_s = kf_b = kf_s = None
                for r in range(args.rounds):
                    for run in (("b", "s") if r % 2 == 0 else ("s", "b")):
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        if run == "b":
                            ev = PhaseEvents()
                            out_b, kf_b = batched(mode, context, S, ev)
                            torch.cuda.synchronize()
                            t_b.append(time.perf_counter() - t0)
                            phases.append(ev.times_ms())
                        else:
                            out_s, kf_s = sequential(mode, context, lists[:S])
                            torch.cuda.synchronize()
                            t_s.append(time.perf_counter() - t0)
                err = [max(syn.rel_l2(a["pts3d"], b["pts3d"]) for a, b in zip(sb.x_out, ss.x_out))
                       for sb, ss in zip(out_b, out_s)]
                frames = S * args.frames
                run = {"batched_frames_per_s": round(frames / min(t_b), 2),
                       "sequential_frames_per_s": round(frames / min(t_s), 2),
                       "batched_s": [round(v, 3) for v in t_b], "sequential_s": [round(v, 3) for v in t_s],
                       "device_ms_median": {p: round(float(np.median([ph[p] for ph in phases])), 2) for p in PHASES},
                       "keyframes_batched": kf_b, "keyframes_sequential": kf_s,
                       "max_pts3d_rel_l2_per_scene": [float(f"{e:.3g}") for e in err]}
                run["speedup"] = round(run["batched_frames_per_s"] / run["sequential_frames_per_s"], 3)
                res["runs"][f"{key}_S{S}"] = run
                print(f"{key} S={S}: batched {run['batched_frames_per_s']} frames/s, one after another "
                      f"{run['sequential_frames_per_s']} frames/s (x{run['speedup']}); device ms {run['device_ms_median']}; "
                      f"keyframes {kf_b} / {kf_s}; max pts3d rel L2 per video {run['max_pts3d_rel_l2_per_scene']}",
                      flush=True)
    print(f"{name} (power limit {limit}), {args.frames} frames 512x384 per video, bf16, max_bs 1")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
