"""PNG decoding on the GPU (engine/png.py) against Pillow, and load_images on PNG paths.

Decode: for each size (640x480, 1920x1080, 2560x1440), content (smooth, uniform noise: the literal-heavy worst case),
compression (Pillow's default and compress_level=1) and batch (1 and 32 files): the GPU path's wall time (host clock
ending in a synchronise; it includes reading the files, parsing and the one status wait), the device time of the
decode's launch sequence (the library's per-launch CUDA events), and how many images the decoder handed back to Pillow,
against Pillow on one thread and on a thread pool of the host's size.
load_images: 200 1080p PNG paths, GPU decode against Pillow-decoded arrays.
SLAM command line (--slam): frames/s on 200 640x480 PNG frames in tools/bench_slam_cli.py's setup, alternating the GPU
read-ahead, the read-ahead decoding with Pillow, and the preload.
Times are the best of --reps runs after a warm-up (one run for the batches of 32).  Prints one JSON line per
measurement, with the card and its power limit.
Usage: python tools/bench_png.py [--reps 3] [--slam] [--decode-only]
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_jpeg import best, card  # noqa: E402


def save_png(img, path, level=None):
    import PIL.Image
    kw = {} if level is None else dict(compress_level=level)
    PIL.Image.fromarray(img).save(path, format="PNG", **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--slam", action="store_true")
    ap.add_argument("--decode-only", action="store_true", help="only the decode cases")
    args = ap.parse_args()
    import png_ref as pr
    from must3r_b200 import _lib
    from must3r_b200.engine import imagefiles, images, png
    dev = torch.device("cuda", 0)
    gpu = card()
    pool = ThreadPoolExecutor(os.cpu_count())
    d = tempfile.mkdtemp()
    lib = _lib.lib()

    def device_ms(items):
        lib.m3r_prof_enable(1)
        outs = png.decode_parsed(items, dev)
        buf = (C.c_double * 28)()
        lib.m3r_prof_read(buf)
        lib.m3r_prof_enable(0)
        return buf[6 * 4], sum(o is None for o in outs)         # category "other": only the decode runs here

    for (H, W) in [(480, 640), (1080, 1920), (1440, 2560)]:
        for kind in ("smooth", "noisy"):
            for level in (None, 1):
                p = os.path.join(d, f"{H}_{kind}_{level}.png")
                save_png(pr.content(H, W, kind), p, level)
                for n in (1, 32):
                    paths = [p] * n
                    reps = args.reps if n == 1 else 1
                    t_gpu = best(lambda: imagefiles.decode_files(paths, dev), reps)
                    items = [imagefiles.parse(x, False) for x in paths]
                    assert all(it.gpu for it in items)
                    png.decode_parsed(items, dev)
                    dms, fallbacks = device_ms(items)
                    t_pil1 = best(lambda: [pr.pillow(x) for x in paths], reps)
                    t_pool = best(lambda: list(pool.map(pr.pillow, paths)), reps)
                    print(json.dumps(dict(bench="decode", gpu=gpu, size=f"{W}x{H}", content=kind,
                                          compress_level="default" if level is None else level, batch=n,
                                          file_bytes=os.path.getsize(p), gpu_wall_ms=round(1e3 * t_gpu, 3),
                                          gpu_device_ms=round(dms, 3), handed_to_pillow=int(fallbacks),
                                          pillow_1thread_ms=round(1e3 * t_pil1, 3), pillow_pool_ms=round(1e3 * t_pool, 3),
                                          pool_threads=os.cpu_count())), flush=True)
    if args.decode_only:
        return
    paths = []
    for k in range(200):
        p = os.path.join(d, f"li_{k:03d}.png")
        save_png(pr.content(1080, 1920, "smooth", seed=k % 8), p)
        paths.append(p)
    t_gpu = best(lambda: images.load_images(paths, 512, verbose=False, device=dev), 1)
    t_pil = best(lambda: images.load_images([pr.pillow(p) for p in paths], 512, verbose=False, device=dev), 1)
    print(json.dumps(dict(bench="load_images", gpu=gpu, frames=200, size="1920x1080", gpu_decode_s=round(t_gpu, 3),
                          pillow_s=round(t_pil, 3))), flush=True)
    if args.slam:
        slam_fps(gpu, d)


def slam_fps(gpu, d, nframes=200, rounds=2):
    """tools/bench_slam_cli.py's run (random-weight full-size model, bf16, res 512, subsamp 4) in three modes."""
    import argparse as ap_
    import PIL.Image
    from bench_slam import frames
    from must3r_b200 import slam as cli, synthetic as syn
    from must3r_b200.engine import png
    from must3r_b200.model import set_precision
    set_precision(torch.bfloat16)
    img_dir = os.path.join(d, "slam_frames")
    os.makedirs(img_dir)
    for i, im in enumerate(frames(nframes)):
        PIL.Image.fromarray(im).save(os.path.join(img_dir, f"{i:05d}.png"))
    chkpt = os.path.join(d, "random.pth")
    torch.save({"args": ap_.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                      decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                "encoder": syn.encoder_state_dict(0), "decoder": syn.camera_like_head_bias(syn.decoder_state_dict(0))}, chkpt)
    from must3r_b200.engine import imagefiles, jpeg
    fixed = imagefiles.READ_AHEAD_ON_GPU

    def run(mode):                              # the read-ahead with PNG frames decoded on the GPU or by Pillow
        imagefiles.READ_AHEAD_ON_GPU = (jpeg.Parsed, png.Parsed) if mode == "gpu_read_ahead" else (jpeg.Parsed,)
        try:
            path = cli.main(["--chkpt", chkpt, "--input", img_dir, "--output", os.path.join(d, "out"), "--res", "512",
                             "--subsamp", "4"], read_ahead=mode != "preload")
        finally:
            imagefiles.READ_AHEAD_ON_GPU = fixed
        return float(np.load(path, allow_pickle=True)["fps"])

    modes = ["gpu_read_ahead", "pillow_read_ahead", "preload"]
    run(modes[0])                               # warm-up
    fps = {m: [] for m in modes}
    for r in range(rounds):
        for m in (modes if r % 2 == 0 else modes[::-1]):
            fps[m].append(round(run(m), 2))
    print(json.dumps(dict(bench="slam_cli", gpu=gpu, frames=nframes, size="640x480", res=512, subsamp=4, dtype="bf16",
                          runs=fps, median={m: float(np.median(v)) for m, v in fps.items()})), flush=True)


if __name__ == "__main__":
    main()
