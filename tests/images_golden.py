"""The input-preprocessing fixture tests/golden/images.npz (written by tests/golden/make_images_golden.py) and the checks
against it that the CPU and GPU tests share."""
import hashlib
import os

import numpy as np
import torch

from must3r_b200 import synthetic as syn

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "images.npz"))
DEMO = sorted({k.split(".")[1] for k in G.files if k.startswith("demo.")})
SLAM = sorted({k.split(".")[1] for k in G.files if k.startswith("slam.")})


def case(kind, name):
    p = f"{kind}.{name}."
    return {k[len(p):]: G[k] for k in G.files if k.startswith(p)}


def frame(c):
    """The case's input frame, regenerated and checked against the stored digest."""
    H, W = (int(v) for v in c["input"][:2])
    f = syn.synthetic_frame(H, W, seed=int(c["seed"]))
    assert hashlib.sha256(f.tobytes()).hexdigest() == str(c["input_sha256"])
    return f


def sha(a) -> str:
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu().contiguous().numpy()
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def img_norm(u8_hwc):
    """ToTensor + Normalize(0.5, 0.5) in fp32, in torchvision's order: [3,H,W]."""
    t = torch.from_numpy(np.ascontiguousarray(u8_hwc)).permute(2, 0, 1).float()
    return ((t / 255) - 0.5) / 0.5


def assert_resized_is_pils(u8, c):
    """u8 [H,W,3] is PIL's resized image of the SLAM case: same sampled pixels, same image where it is stored whole, and
    the same SHA-256."""
    assert list(u8.shape) == list(c["resized_shape"])
    assert np.array_equal(u8.reshape(-1)[c["resized_sample_idx"]], c["resized_sample"])
    if "resized" in c:
        assert np.array_equal(u8, c["resized"])
    assert sha(u8) == str(c["resized_sha256"])


def assert_close_to_demo(img, c):
    """img [3,h,w] fp32 agrees with the reference's demo image within 1e-5: the sampled pixels, and the per-channel,
    per-row and per-column sums (as means over the summed pixels)."""
    oh, ow = (int(v) for v in c["true_shape"])
    assert img.shape == (3, oh, ow)
    assert np.abs(img.reshape(-1)[c["sample_idx"]] - c["sample"]).max() <= 1e-5
    x = img.astype(np.float64)
    assert np.abs(x.sum(axis=(1, 2)) - c["sums"]).max() <= 1e-5 * oh * ow
    assert np.abs(x.sum(axis=2) - c["row_sums"]).max() <= 1e-5 * ow
    assert np.abs(x.sum(axis=1) - c["col_sums"]).max() <= 1e-5 * oh
