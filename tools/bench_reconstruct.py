#!/usr/bin/env python
"""Reconstruction front end on one GPU (must3r_b200/engine/demo.py): 200 seeded synthetic 512x384 frames written as PNG
files, the full-size random-weight model in bf16 at image_size 512.

    python tools/bench_reconstruct.py [--frames 200] [--rounds 3]

Times get_reconstructed_scene in three modes: 'linseq' with 50 keyframes and the render pass, 'vidseq' and 'vidslam'
(the reference's defaults of get_reconstruction.py otherwise), each from the file list to the SceneState on the host.
Then, on the linseq scene, the point clouds at get_reconstruction.py's 8 thresholds two ways, alternating in rounds:
m3r_scene_points (one pass for all thresholds, the points copied to the host) and the reference's numpy masking of the
host tensors (gradio.py:147-151, :91-92, once per threshold), checking that both give the same arrays.  Prints the card's
name and power limit and one JSON line.  Writes only to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from must3r_b200 import synthetic as syn  # noqa: E402
from must3r_b200.engine import demo  # noqa: E402
from must3r_b200.model import load_model, set_precision  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def write_frames(d, n, H=384, W=512, step=6):
    import PIL.Image
    pano = syn.synthetic_frame(H, W + step * n, seed=0)
    paths = []
    for i in range(n):
        p = os.path.join(d, f"{i:04d}.png")
        PIL.Image.fromarray(np.ascontiguousarray(pano[:, step * i:step * i + W])).save(p)
        paths.append(p)
    return paths


def numpy_clouds(scene, thresholds):
    """gradio.py:147-151 then :91-92 on the scene's host tensors, once per threshold."""
    out = []
    for thr in thresholds:
        pts3d = [o['pts3d'].cpu() for o in scene.x_out]
        msk = [(o['conf'] >= thr).cpu() for o in scene.x_out]
        pts = np.concatenate([p.numpy()[m.numpy()] for p, m in zip(pts3d, msk)])
        col = np.concatenate([p[m.numpy()] for p, m in zip(scene.imgs, msk)])
        out.append((pts, col))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_reconstruct needs a CUDA device"
    set_precision(torch.bfloat16)
    name, limit = card()
    res = {}
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "random.pth")
        dsd = syn.camera_like_head_bias(syn.decoder_state_dict(0))
        torch.save({"args": argparse.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                               decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                    "encoder": syn.encoder_state_dict(0), "decoder": dsd}, chkpt)
        model = load_model(chkpt, device="cuda", img_size=512, verbose=False)
        paths = write_frames(d, args.frames)
        common = dict(outdir=d, viser_server=None, should_save_glb=False, model=model, retrieval=None, device="cuda",
                      verbose=False, image_size=512, amp=False, filelist=paths, max_bs=1, num_refinements_iterations=0,
                      num_mem_images=min(50, len(paths)), render_once=False, vidseq_local_context_size=0,
                      keyframe_interval=3, slam_local_context_size=0, subsample=2, min_conf_keyframe=1.5,
                      keyframe_overlap_thr=0.05, overlap_percentile=85, min_conf_thr=1.05, as_pointcloud=True,
                      transparent_cams=False, local_pointmaps=False, cam_size=0.05)
        # warm every mode once on a few frames (module loads, allocator, kernel setup)
        for mode in ("linseq", "vidseq", "vidslam"):
            demo.get_reconstructed_scene(**{**common, "filelist": paths[:8], "num_mem_images": 4}, execution_mode=mode)
        scenes = {}
        for mode in ("linseq", "vidseq", "vidslam"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            scenes[mode], _ = demo.get_reconstructed_scene(**common, execution_mode=mode)
            torch.cuda.synchronize()
            res[f"{mode}_s"] = round(time.perf_counter() - t0, 3)
            res[f"{mode}_views_per_s"] = round(args.frames / res[f"{mode}_s"], 2)
    scene = scenes["linseq"]
    thr = demo.THRESHOLDS
    kernel_s, numpy_s = [], []
    demo.get_3D_models_from_scene(scene, thr)                       # warm
    for _ in range(args.rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        k = demo.get_3D_models_from_scene(scene, thr)
        kernel_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        ref = numpy_clouds(scene, thr)
        numpy_s.append(time.perf_counter() - t0)
    for (p, c), (rp, rc) in zip(k, ref):
        assert np.array_equal(p, rp) and np.array_equal(c, rc)
    res.update({"points_8_thresholds": int(sum(p.shape[0] for p, _ in k)),
                "cloud_kernel_s_median": round(float(np.median(kernel_s)), 4),
                "cloud_numpy_s_median": round(float(np.median(numpy_s)), 4),
                "cloud_kernel_s": [round(v, 4) for v in kernel_s], "cloud_numpy_s": [round(v, 4) for v in numpy_s],
                "frames": args.frames, "gpu": name, "power_limit": limit})
    print(f"{name} (power limit {limit}), {args.frames} frames 512x384, bf16:")
    for mode in ("linseq", "vidseq", "vidslam"):
        print(f"  {mode}: {res[f'{mode}_s']} s, {res[f'{mode}_views_per_s']} views/s")
    print(f"  point clouds at 8 thresholds ({res['points_8_thresholds']} points): kernel {res['cloud_kernel_s_median']} s, "
          f"numpy masking {res['cloud_numpy_s_median']} s (median of {args.rounds} alternating rounds)")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
