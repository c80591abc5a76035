"""Input preprocessing on the GPU (must3r_b200/engine/images.py): per-frame times of the SLAM path (preproc_frame: PIL
resize, crop, ImgNorm) and the demo path (load_images: CenterCrop + antialiased bilinear Resize), against the host path
of the reference (PIL / torchvision, when importable), and a C5-style stream that starts from host uint8 frames.

    python tools/bench_preproc.py [--frames 60] [--reps 20] [--no-stream]

GPU times are CUDA events around the enqueued work ("device": frames already on the GPU; "from host": numpy frames,
pinned staging and the upload included).  Host times are wall clock on this machine's CPU (torch's thread count as
set).  Writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from must3r_b200 import engine, synthetic as syn  # noqa: E402
from must3r_b200.engine import images  # noqa: E402


def cuda_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, (time.perf_counter() - t0) * 1e3 / reps


def host_ms(fn, reps):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    return (time.perf_counter() - t0) * 1e3 / reps


def host_paths():
    """The reference's host operations (dust3r _resize_pil_image + crop + ImgNorm; ImgNorm + CenterCrop + Resize)."""
    try:
        import PIL.Image
        import torchvision.transforms as tvf
    except ImportError:
        return None
    norm = tvf.Compose([tvf.ToTensor(), tvf.Normalize((0.5, 0.5, 0.5), (0.5, 0.5, 0.5))])

    def slam(f, res):
        (h, w), filt, (x0, y0, cw, ch), _ = images._slam_geometry(f.shape[0], f.shape[1], res)
        im = PIL.Image.fromarray(f)
        if (w, h) != im.size:
            im = im.resize((w, h), PIL.Image.LANCZOS if filt == "lanczos" else PIL.Image.BICUBIC)
        return norm(im.crop((x0, y0, x0 + cw, y0 + ch)))[None]

    def demo(f, size):
        geo = images._demo_geometry(size, f.shape[0], f.shape[1])
        t = norm(PIL.Image.fromarray(f))
        if geo.out_hw == tuple(f.shape[:2]):
            return t
        return tvf.Resize(list(geo.out_hw))(tvf.CenterCrop(list(geo.crop[2:]))(t))

    return slam, demo


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=60, help="frames of the C5-style stream")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-stream", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    results = {"gpu": torch.cuda.get_device_name(dev), "host_threads": torch.get_num_threads()}
    hp = host_paths()
    rows = []
    for tag, (H, W), n in (("640x480", (480, 640), 1), ("1920x1080", (1080, 1920), 1), ("20x 2560x1440", (1440, 2560), 20)):
        host = np.stack([syn.synthetic_frame(H, W, seed=i) for i in range(n)])
        dvc = torch.from_numpy(host).to(dev)
        geo = images._demo_geometry(512, H, W)
        demo_op, _, _ = images.get_resize_function(512, 16, H, W)
        (h, w), filt, crop, _ = images._slam_geometry(H, W, 512)
        r = {"input": tag, "demo_out": list(geo.out_hw), "slam_out": [crop[3], crop[2]]}
        for path, fn_dev, fn_host in (
                ("slam", lambda: images.resize_pil(dvc, (h, w), filt, crop=crop),
                 lambda: [images.preproc_frame(f, 0, res=512) for f in host]),
                ("demo", lambda: demo_op(dvc), lambda: images.load_images(list(host), 512, verbose=False))):
            gd, _ = cuda_ms(fn_dev, args.reps)
            gh, wall = cuda_ms(fn_host, max(2, args.reps // 4))
            r[f"{path}_gpu_ms_per_frame"] = round(gd / n, 4)
            r[f"{path}_from_host_ms_per_frame"] = round(gh / n, 4)
            r[f"{path}_from_host_wall_ms_per_frame"] = round(wall / n, 4)
            if hp is not None:
                fn = hp[0] if path == "slam" else hp[1]
                r[f"{path}_host_ms_per_frame"] = round(host_ms(lambda: [fn(f, 512) for f in host], 2 if n > 1 else 5) / n, 3)
        rows.append(r)
        print(json.dumps(r), flush=True)
    results["cases"] = rows
    if not args.no_stream:
        results["stream"] = stream(dev, args.frames)
        print(json.dumps(results["stream"]), flush=True)
    print(json.dumps(results))


def stream(dev, F):
    """C5-style: 640x480 camera frames on the host -> preproc_frame (512x384) -> inference_video_multi_ar (keyframe iff
    id % 3 == 0, window 25), against the same run over frames that are already normalised on the GPU."""
    from must3r_b200.model import Dust3rEncoder, MUSt3R, ActivationType, set_precision
    set_precision(torch.bfloat16)
    enc = Dust3rEncoder(img_size=(512, 512))
    dec = MUSt3R(img_size=(512, 512), feedback_type="single_mlp", memory_mode="kv", landscape_only=False)
    enc.load_state_dict(syn.encoder_state_dict(0))
    dec.load_state_dict(syn.decoder_state_dict(0))
    enc, dec = enc.to(dev).eval(), dec.to(dev).eval()
    frames = [syn.synthetic_frame(480, 640, seed=100 + i) for i in range(F)]
    pp = lambda pm: engine.postprocess(pm, ActivationType.NORM_EXP)  # noqa: E731
    pre = [images.preproc_frame(f, i)[0]["img"][0] for i, f in enumerate(frames)]

    def run(views):
        ts = torch.tensor([[384, 512]] * F)
        x, pos = engine.encoder_multi_ar(enc, views, ts, device=dev)
        return engine.inference_video_multi_ar(enc, dec, views, list(ts.unbind(0)), [2] + [1] * (F - 2),
                                               encoder_precomputed_features=(x, pos), post_process_function=pp, device=dev,
                                               local_context_size=25)

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    with torch.no_grad():
        t_dev = timed(lambda: run(pre))
        t_host = timed(lambda: run([images.preproc_frame(f, i)[0]["img"][0] for i, f in enumerate(frames)]))
    return {"stream_frames": F, "frames_per_s_preprocessed_on_gpu_from_host_uint8": round(F / t_host, 2),
            "frames_per_s_inputs_already_on_gpu": round(F / t_dev, 2)}


if __name__ == "__main__":
    main()
