#!/usr/bin/env python
"""Generate tests/golden/images.npz: the reference's own input preprocessing on seeded synthetic frames.

Run where a reference checkout exists ($MUST3R_REFERENCE, or the locations oracle/install_reference.py searches):

    python tests/golden/make_images_golden.py

Frames come from ``must3r_b200.synthetic.synthetic_frame`` (integer arithmetic, regenerated identically by the tests,
which check their SHA-256).  Outputs come from the UNMODIFIED reference functions:
  * demo path: must3r/demo/inference.py load_images on the frames saved as PNG, and must3r/tools/image.py
    get_resize_function for the matrices;
  * SLAM path: must3r/slam/model.py preproc_frame, plus the PIL image of _resize_pil_image
    (dust3r/dust3r/utils/image.py) that it crops, checked to be exactly what preproc_frame normalised.
Stored, kept small (noise does not compress): the geometry of every case; for the SLAM path, SHA-256 digests of the
PIL uint8 resized images and of the fp32 images, a seeded sample of the uint8 pixels (for diagnosis when a digest
differs) and one small resized image densely; for the demo path, a seeded sample of the fp32 pixels (larger for two
cases), per-channel sums, and per-channel row and column sums.
The retrieval / rotation dependencies the reference modules import (faiss, asmk, roma) are not needed by these
functions and are replaced by empty placeholder modules when absent.
"""
import hashlib
import importlib.abc
import importlib.machinery
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from must3r_b200 import synthetic as syn  # noqa: E402
from oracle.install_reference import source  # noqa: E402

# (name, H, W, size): demo load_images cases
DEMO = [("d1080p", 1080, 1920, 512), ("d1000x700", 700, 1000, 512), ("d1000x1000", 1000, 1000, 512),
        ("dportrait", 640, 480, 512), ("dup320", 240, 320, 512), ("dpass512", 384, 512, 512), ("d224", 480, 640, 224)]
DEMO_LARGE_SAMPLE = ("d1080p", "d224")       # 16384 sampled pixels instead of 4096
SLAM_DENSE = ("s224square",)                  # resized uint8 image stored whole (224 x 224 x 3)
# (name, H, W, res): SLAM preproc_frame cases
SLAM = [("s640", 480, 640, 512), ("s1080p", 1080, 1920, 512), ("s400", 300, 400, 512), ("scopy", 384, 512, 512),
        ("sportrait", 640, 480, 512), ("ssquare", 500, 500, 512), ("s224", 480, 640, 224),
        ("s224portrait", 640, 480, 224), ("s224square", 500, 500, 224)]
SEEDS = {name: i for i, name in enumerate([c[0] for c in DEMO] + [c[0] for c in SLAM])}
N_SAMPLE = 4096


class _Placeholders(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """Empty modules (any attribute is a dummy class) for optional packages the reference imports at module level."""
    ROOTS = ("faiss", "asmk", "roma")

    def find_spec(self, name, path, target=None):
        if name.split(".")[0] in self.ROOTS:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []
        m.__getattr__ = lambda attr: type(attr, (), {})
        return m

    def exec_module(self, module):
        pass


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    ref = source()
    if ref is None:
        sys.exit("no reference checkout found: set MUST3R_REFERENCE")
    sys.path.insert(0, ref)
    sys.meta_path.append(_Placeholders())             # only consulted for modules that are not installed
    import PIL.Image
    import torchvision.transforms as tvf
    from must3r.demo.inference import load_images
    from must3r.tools.image import get_resize_function
    from must3r.slam.model import preproc_frame
    from dust3r.utils.image import _resize_pil_image, ImgNorm

    out = {}
    rng = np.random.default_rng(20261015)
    with tempfile.TemporaryDirectory() as tmp:
        for name, H, W, size in DEMO:
            frame = syn.synthetic_frame(H, W, seed=SEEDS[name])
            path = os.path.join(tmp, name + ".png")
            PIL.Image.fromarray(frame).save(path)
            d = load_images([path], size, patch_size=16, verbose=False)[0]
            img = d["img"].numpy()
            _, to_rescaled, to_orig = get_resize_function(size, 16, H, W)
            h, w = img.shape[-2:]
            crop_w, crop_h = int(round(to_orig[0, 0] * w)), int(round(to_orig[1, 1] * h))
            # the crop offsets torchvision's CenterCrop takes, read off a coordinate image
            coords = torch.stack(torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij"))
            top, left = (int(v) for v in tvf.CenterCrop([crop_h, crop_w])(coords)[:, 0, 0])
            p = f"demo.{name}."
            out[p + "input"] = np.array([H, W, size], np.int64)
            out[p + "seed"] = np.array(SEEDS[name], np.int64)
            out[p + "input_sha256"] = np.array(sha(frame))
            out[p + "crop"] = np.array([top, left, crop_h, crop_w], np.int64)
            out[p + "true_shape"] = d["true_shape"]
            out[p + "to_rescaled"] = to_rescaled
            out[p + "to_orig"] = to_orig
            out[p + "sums"] = img.astype(np.float64).sum(axis=(1, 2))
            out[p + "row_sums"] = img.astype(np.float64).sum(axis=2)
            out[p + "col_sums"] = img.astype(np.float64).sum(axis=1)
            n = 4 * N_SAMPLE if name in DEMO_LARGE_SAMPLE else N_SAMPLE
            idx = np.sort(rng.choice(img.size, n, replace=False)).astype(np.int32)
            out[p + "sample_idx"] = idx
            out[p + "sample"] = img.reshape(-1)[idx]
    for name, H1, W1, res in SLAM:
        frame = syn.synthetic_frame(H1, W1, seed=SEEDS[name])
        d, focal = preproc_frame(frame, 3, res=res)
        longsize = max(W1, H1) / min(W1, H1) * res if res in (224, 336, 448) else res
        pil = _resize_pil_image(PIL.Image.fromarray(frame), longsize)
        resized = np.asarray(pil)
        x0, y0 = (int(v) for v in d["offset"][0])
        h, w = (int(v) for v in d["true_shape"][0])
        again = ImgNorm(pil.crop((x0, y0, x0 + w, y0 + h)))[None].numpy()
        img = d["img"].numpy()
        assert again.tobytes() == img.tobytes(), name           # the stored intermediate is what preproc_frame cropped
        p = f"slam.{name}."
        out[p + "input"] = np.array([H1, W1, res], np.int64)
        out[p + "seed"] = np.array(SEEDS[name], np.int64)
        out[p + "input_sha256"] = np.array(sha(frame))
        out[p + "resized_shape"] = np.array(resized.shape, np.int64)   # [H, W, 3] uint8, PIL
        out[p + "resized_sha256"] = np.array(sha(resized))
        idx = np.sort(rng.choice(resized.size, N_SAMPLE, replace=False)).astype(np.int32)
        out[p + "resized_sample_idx"] = idx
        out[p + "resized_sample"] = resized.reshape(-1)[idx]
        if name in SLAM_DENSE:
            out[p + "resized"] = resized
        out[p + "filter"] = np.array("lanczos" if max(W1, H1) > longsize else "bicubic")
        out[p + "crop"] = np.array([x0, y0, w, h], np.int64)
        out[p + "true_shape"] = d["true_shape"]
        out[p + "offset"] = d["offset"]
        out[p + "focal"] = np.array(focal, np.float64)
        out[p + "img_shape"] = np.array(img.shape, np.int64)
        out[p + "img_sha256"] = np.array(sha(img))
        out[p + "sums"] = img.astype(np.float64).sum(axis=(0, 2, 3))
    dst = os.path.join(HERE, "images.npz")
    np.savez_compressed(dst, **out)
    print(f"wrote {dst}: {os.path.getsize(dst) / 1e6:.2f} MB, {len(DEMO)} demo and {len(SLAM)} SLAM cases")


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
