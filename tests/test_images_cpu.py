"""Input preprocessing (must3r_b200/engine/images.py) against the reference's outputs in tests/golden/images.npz, without
a GPU: the geometry of every case, and the host coefficient tables the kernels consume, applied here by a NumPy model of
the kernels' passes: the fixed-point one must reproduce PIL's uint8 images bit for bit."""
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

from must3r_b200 import ops, synthetic as syn
from must3r_b200.engine import images

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from images_golden import (DEMO, SLAM, assert_close_to_demo, assert_resized_is_pils, case, frame,  # noqa: E402
                           img_norm)


def pil_pass(src, bounds, weights, axis):
    """One pass of Pillow's 8-bit resampler: 0.5 + sum src * w (22 fractional bits), >> 22, clamped to 0..255."""
    s = np.moveaxis(src, axis, 0).astype(np.int64)
    out = np.empty((bounds.shape[0],) + s.shape[1:], np.int64)
    for i, (b0, n) in enumerate(bounds):
        acc = np.full(s.shape[1:], 1 << 21, np.int64)
        for k in range(n):
            acc += s[b0 + k] * int(weights[i, k])
        out[i] = np.clip(acc >> 22, 0, 255)
    return np.moveaxis(out, 0, axis).astype(np.uint8)


def float_pass(src, bounds, weights, axis):
    s = np.moveaxis(src, axis, 0)
    out = np.zeros((bounds.shape[0],) + s.shape[1:], np.float32)
    for i, (b0, n) in enumerate(bounds):
        acc = np.zeros(s.shape[1:], np.float32)
        for k in range(n):
            acc = acc + s[b0 + k] * weights[i, k]
        out[i] = acc
    return np.moveaxis(out, 0, axis)


@pytest.mark.parametrize("name", DEMO)
def test_demo_geometry_matches_the_reference(name):
    c = case("demo", name)
    H, W, size = (int(v) for v in c["input"])
    geo = images._demo_geometry(size, H, W)
    assert list(geo.crop) == list(c["crop"])
    assert list(geo.out_hw) == list(c["true_shape"])
    _, to_rescaled, to_orig = images.get_resize_function(size, 16, H, W)
    assert np.array_equal(to_rescaled, c["to_rescaled"]) and np.array_equal(to_orig, c["to_orig"])
    if [max(H, W), min(H, W)] not in images.ratios_resolutions[size].values():      # else: passed through unchanged
        assert list(images.get_HW_resolution(H, W, size)) == list(c["true_shape"])


@pytest.mark.parametrize("name", SLAM)
def test_slam_geometry_matches_the_reference(name):
    c = case("slam", name)
    H1, W1, res = (int(v) for v in c["input"])
    (H, W), filt, crop, focal = images._slam_geometry(H1, W1, res)
    assert [H, W, 3] == list(c["resized_shape"])
    assert filt == str(c["filter"])
    assert list(crop) == list(c["crop"])
    assert [crop[3], crop[2]] == list(c["true_shape"][0]) and [crop[0], crop[1]] == list(c["offset"][0])
    assert focal == float(c["focal"])
    assert list(c["img_shape"]) == [1, 3, crop[3], crop[2]]


@pytest.mark.parametrize("name", SLAM)
def test_pil_tables_reproduce_pil_bit_for_bit(name):
    """The int32 tables the kernel consumes, applied in the kernel's order, give PIL's resized image exactly; ImgNorm of
    its crop box is the reference's fp32 image exactly."""
    c = case("slam", name)
    f = frame(c)
    H, W = (int(v) for v in c["resized_shape"][:2])
    xb, xw, yb, yw, row0, rows = images._pil_plan(f.shape[0], f.shape[1], H, W, str(c["filter"]))
    assert xb[:, 1].max() <= xw.shape[1] and yb[:, 1].max() <= yw.shape[1]
    assert (xb[:, 0] + xb[:, 1]).max() <= f.shape[1] and (yb[:, 0] + yb[:, 1]).max() <= rows
    got = pil_pass(pil_pass(f[row0:row0 + rows], xb, xw, 1), yb, yw, 0)
    assert_resized_is_pils(got, c)
    x0, y0, w, h = (int(v) for v in c["crop"])
    img = img_norm(got[y0:y0 + h, x0:x0 + w])[None].numpy()
    assert hashlib.sha256(img.tobytes()).hexdigest() == str(c["img_sha256"])


@pytest.mark.parametrize("name", ["d1080p", "d224", "dportrait"])
def test_aa_tables_match_torchvision(name):
    """The fp32 antialiased-bilinear tables, applied in the kernel's order to the normalised crop, agree with the
    reference's images within 1e-5."""
    c = case("demo", name)
    f = frame(c)
    top, left, ch, cw = (int(v) for v in c["crop"])
    oh, ow = (int(v) for v in c["true_shape"])
    xb, xw = images.aa_bilinear_coeffs(cw, ow)
    yb, yw = images.aa_bilinear_coeffs(ch, oh)
    x = img_norm(f[top:top + ch, left:left + cw]).numpy()
    got = float_pass(float_pass(x, xb, xw, 2), yb, yw, 1)
    assert_close_to_demo(got, c)


def test_identity_tables_are_exact_copies():
    """A pass whose size does not change is skipped by Pillow and aten: its table is one unit weight per output."""
    b, w = images.pil_coeffs(384, 384, "lanczos")
    assert (b[:, 0] == np.arange(384)).all() and (b[:, 1] == 1).all() and (w == 1 << 22).all()
    b, w = images.aa_bilinear_coeffs(224, 224)
    assert (b[:, 1] == 1).all() and (w == 1.0).all()


def test_entry_points_fail_loudly_without_cuda():
    f = syn.synthetic_frame(48, 64, seed=1)
    with pytest.raises(RuntimeError, match="CUDA"):
        images.preproc_frame(f, 0, res=512, device="cpu")
    with pytest.raises(RuntimeError, match="CUDA"):
        images.load_images([f], 224, verbose=False, device="cpu")
    op, _, _ = images.get_resize_function(512, 16, 48, 64)
    with pytest.raises(RuntimeError, match="CUDA"):
        op(f, device="cpu")
    src = torch.from_numpy(f)[None]
    tabs = [torch.zeros(8, dtype=torch.int32)] * 4
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.resample_pil_u8(src, tabs, 1, 1, (48, 64), 0, 48, torch.zeros(10, dtype=torch.uint8), (0, 0, 64, 48),
                            out=torch.zeros(1, 3, 48, 64))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.resize_aa_bilinear_u8(src, tabs, 1, 1, (48, 64), torch.zeros(10), torch.zeros(1, 3, 48, 64))
