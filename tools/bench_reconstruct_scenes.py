#!/usr/bin/env python
"""Several offline reconstructions on one GPU (must3r_b200/engine/scenes.py) against one scene after another.

    python tools/bench_reconstruct_scenes.py [--scenes 1 2 4 8] [--frames 60] [--keyframes 20] [--rounds 2]

Per scene count S: S folders of seeded synthetic 512x384 PNG frames (a panorama sliding right, each scene from its own
seed), the full-size random-weight model in bf16 at image_size 512, get_reconstruction.py's defaults (max_bs 1, the render
pass on).  Two modes alternate in rounds: `reconstruct_scenes` over all S scenes, and `must3r_inference` once per scene
in one thread.  Reports the aggregate views/s of each (best round, from the file lists to the SceneStates on the host),
the median device time of the batched run's encoder, memory steps, render and postprocess (CUDA events at the engine's
phase boundaries), per scene the largest pts3d relative L2 between the two modes, the card's name and power limit, and
one JSON line.  Writes only to a temporary directory.
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
from must3r_b200.engine import demo, scenes  # noqa: E402
from must3r_b200.model import load_model, set_precision  # noqa: E402
from bench_reconstruct import card  # noqa: E402

PHASES = ("encode", "memory", "render", "postprocess")


def write_frames(d, n, seed, H=384, W=512, step=6):
    import PIL.Image
    os.makedirs(d, exist_ok=True)
    pano = syn.synthetic_frame(H, W + step * n, seed=seed)
    paths = []
    for i in range(n):
        p = os.path.join(d, f"{i:04d}.png")
        PIL.Image.fromarray(np.ascontiguousarray(pano[:, step * i:step * i + W])).save(p)
        paths.append(p)
    return paths


class PhaseEvents:
    """Replaces scenes._phase: one CUDA event per phase boundary of a batched run."""

    def __init__(self):
        self.events = {}

    def __call__(self, name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.events[name] = e

    def times_ms(self):
        names = PHASES + ("end",)
        return {a: self.events[a].elapsed_time(self.events[b]) for a, b in zip(names, names[1:])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, nargs="+", default=[1, 2, 4, 8])
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--keyframes", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_reconstruct_scenes needs a CUDA device"
    set_precision(torch.bfloat16)
    name, limit = card()
    res = {"frames": args.frames, "keyframes": args.keyframes, "gpu": name, "power_limit": limit, "runs": {}}
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "random.pth")
        dsd = syn.camera_like_head_bias(syn.decoder_state_dict(0))
        torch.save({"args": argparse.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                               decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                    "encoder": syn.encoder_state_dict(0), "decoder": dsd}, chkpt)
        model = load_model(chkpt, device="cuda", img_size=512, verbose=False)
        lists = [write_frames(os.path.join(d, f"s{i}"), args.frames, seed=i) for i in range(max(args.scenes))]
        kw = dict(num_mem_images=args.keyframes, max_bs=1, render_once=False, verbose=False)

        def batched(S, phase=None):
            scenes._phase = phase or (lambda n: None)
            try:
                return scenes.reconstruct_scenes(model, "cuda", 512, False, lists[:S], **kw)
            finally:
                scenes._phase = lambda n: None

        def sequential(S):
            return [demo.must3r_inference(model, None, "cuda", 512, False, fl, min(args.keyframes, len(fl)), 1, 2, 1,
                                          False, is_sequence=True, verbose=False) for fl in lists[:S]]
        # warm both paths on short scenes (module loads, allocator, workspaces)
        short = [fl[:8] for fl in lists[:2]]
        scenes.reconstruct_scenes(model, "cuda", 512, False, short, 4, 1, verbose=False)
        demo.must3r_inference(model, None, "cuda", 512, False, short[0], 4, 1, 2, 1, False, is_sequence=True, verbose=False)
        for S in args.scenes:
            t_b, t_s, phases = [], [], []
            out_b = out_s = None
            for r in range(args.rounds):
                order = ("b", "s") if r % 2 == 0 else ("s", "b")
                for mode in order:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if mode == "b":
                        ev = PhaseEvents()
                        out_b = batched(S, ev)
                        torch.cuda.synchronize()
                        t_b.append(time.perf_counter() - t0)
                        phases.append(ev.times_ms())
                    else:
                        out_s = sequential(S)
                        torch.cuda.synchronize()
                        t_s.append(time.perf_counter() - t0)
            err = [max(syn.rel_l2(a["pts3d"], b["pts3d"]) for a, b in zip(sb.x_out, ss.x_out))
                   for sb, ss in zip(out_b, out_s)]
            views = S * args.frames
            run = {"batched_views_per_s": round(views / min(t_b), 2), "sequential_views_per_s": round(views / min(t_s), 2),
                   "batched_s": [round(v, 3) for v in t_b], "sequential_s": [round(v, 3) for v in t_s],
                   "device_ms_median": {p: round(float(np.median([ph[p] for ph in phases])), 2) for p in PHASES},
                   "max_pts3d_rel_l2_per_scene": [float(f"{e:.3g}") for e in err]}
            run["speedup"] = round(run["batched_views_per_s"] / run["sequential_views_per_s"], 3)
            res["runs"][str(S)] = run
            print(f"S={S}: batched {run['batched_views_per_s']} views/s, one after another "
                  f"{run['sequential_views_per_s']} views/s (x{run['speedup']}); device ms {run['device_ms_median']}; "
                  f"max pts3d rel L2 per scene {run['max_pts3d_rel_l2_per_scene']}", flush=True)
    print(f"{name} (power limit {limit}), {args.frames} frames 512x384 per scene, {args.keyframes} keyframes, bf16, max_bs 1")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
