"""JPEG decoding on the GPU (engine/jpeg.py) against Pillow, and load_images on JPEG paths.

Decode: for each size (640x480, 1920x1080, 2560x1440), quality (90, 95) and sampling (4:2:0, 4:4:4), batches of 1 and
32 files: the GPU path's wall time (host clock ending in a synchronise; it includes reading the files, parsing and the
one status wait), the device time of the decode's launch sequence (the library's per-launch CUDA events), and how many
images the decoder handed back to Pillow, against Pillow on one thread and on a thread pool of the host's size.  Smooth
content, plus uniform noise (the worst case for the synchronisation rounds) at 1080p.
load_images: 200 1080p JPEG paths, GPU decode against Pillow-decoded arrays.
SLAM command line (--slam): frames/s on 200 640x480 JPEG frames in tools/bench_slam_cli.py's setup, alternating the GPU
read-ahead, the read-ahead decoding with Pillow, and the preload.
Prints one JSON line per measurement, with the card and its power limit.
Usage: python tools/bench_jpeg.py [--reps 5] [--slam]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()[0]
    return q


def best(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--slam", action="store_true")
    args = ap.parse_args()
    import jpeg_ref as jr
    from must3r_b200.engine import images, jpeg
    dev = torch.device("cuda", 0)
    gpu = card()
    pool = ThreadPoolExecutor(os.cpu_count())
    d = tempfile.mkdtemp()
    import ctypes as C
    from must3r_b200 import _lib
    lib = _lib.lib()

    def device_ms(items):
        lib.m3r_prof_enable(1)
        outs = jpeg.decode_parsed(items, dev)
        buf = (C.c_double * 28)()
        lib.m3r_prof_read(buf)
        lib.m3r_prof_enable(0)
        return buf[6 * 4], sum(o is None for o in outs)         # category "other": only the decode runs here

    cases = [((H, W), "smooth", q, ss) for (H, W) in [(480, 640), (1080, 1920), (1440, 2560)] for q in (90, 95)
             for ss in (("420", 2), ("444", 0))] + [((1080, 1920), "noisy", q, ("420", 2)) for q in (90, 95)]
    for (H, W), kind, q, (ss, sv) in cases:
        p = os.path.join(d, f"{H}_{kind}_{q}_{ss}.jpg")
        with open(p, "wb") as f:
            f.write(jr.save(jr.content(H, W, kind), format="JPEG", quality=q, subsampling=sv))
        for n in (1, 32):
            paths = [p] * n
            t_gpu = best(lambda: jpeg.decode_files(paths, dev), args.reps)
            items = [jpeg.Parsed(x, False) for x in paths]
            jpeg.decode_parsed(items, dev)
            dms, fallbacks = device_ms(items)
            t_pil1 = best(lambda: [jr.pillow(x, False) for x in paths], args.reps)
            t_pool = best(lambda: list(pool.map(lambda x: jr.pillow(x, False), paths)), args.reps)
            print(json.dumps(dict(bench="decode", gpu=gpu, size=f"{W}x{H}", content=kind, quality=q, sampling=ss, batch=n,
                                  gpu_wall_ms=round(1e3 * t_gpu, 3), gpu_device_ms=round(dms, 3),
                                  handed_to_pillow=int(fallbacks), pillow_1thread_ms=round(1e3 * t_pil1, 3),
                                  pillow_pool_ms=round(1e3 * t_pool, 3), pool_threads=os.cpu_count())), flush=True)
    paths = []
    for k in range(200):
        p = os.path.join(d, f"li_{k:03d}.jpg")
        with open(p, "wb") as f:
            f.write(jr.save(jr.content(1080, 1920, "smooth", seed=k % 8), format="JPEG", quality=90))
        paths.append(p)
    t_gpu = best(lambda: images.load_images(paths, 512, verbose=False, device=dev), max(1, args.reps // 2))
    t_pil = best(lambda: images.load_images([jr.pillow(p, False) for p in paths], 512, verbose=False, device=dev),
                 max(1, args.reps // 2))
    print(json.dumps(dict(bench="load_images", gpu=gpu, frames=200, size="1920x1080", gpu_decode_s=round(t_gpu, 3),
                          pillow_s=round(t_pil, 3))), flush=True)
    if args.slam:
        slam_fps(gpu, d)


def slam_fps(gpu, d, nframes=200, rounds=2):
    """tools/bench_slam_cli.py's run (random-weight full-size model, bf16, res 512, subsamp 4) in three modes."""
    import argparse as ap_
    import PIL.Image
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_slam import frames
    from must3r_b200 import slam as cli, synthetic as syn
    from must3r_b200.engine import jpeg
    from must3r_b200.model import set_precision
    set_precision(torch.bfloat16)
    img_dir = os.path.join(d, "slam_frames")
    os.makedirs(img_dir)
    for i, im in enumerate(frames(nframes)):
        PIL.Image.fromarray(im).save(os.path.join(img_dir, f"{i:05d}.jpg"), quality=90)
    chkpt = os.path.join(d, "random.pth")
    torch.save({"args": ap_.Namespace(encoder="Dust3rEncoder(img_size=(512, 512))",
                                      decoder="MUSt3R(img_size=(512, 512), feedback_type='single_mlp', memory_mode='kv')"),
                "encoder": syn.encoder_state_dict(0), "decoder": syn.camera_like_head_bias(syn.decoder_state_dict(0))}, chkpt)
    gpu_parsed = jpeg.Parsed

    class PillowParsed(jpeg.Parsed):          # the read-ahead as before: every frame decoded by Pillow on the host
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.gpu = False

    def run(mode):
        jpeg.Parsed = PillowParsed if mode == "pillow_read_ahead" else gpu_parsed
        try:
            path = cli.main(["--chkpt", chkpt, "--input", img_dir, "--output", os.path.join(d, "out"), "--res", "512",
                             "--subsamp", "4"], read_ahead=mode != "preload")
        finally:
            jpeg.Parsed = gpu_parsed
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
