"""Input preprocessing on the GPU: the reference's image loaders with the resampling done by CUDA kernels.

Replaces
  * must3r/tools/image.py:17-93 (ratios_resolutions, get_HW_resolution, get_resize_function) and the demo's
    load_images (must3r/demo/inference.py:63-76): ImgNorm, torchvision CenterCrop, then an antialiased bilinear
    Resize of the float image (m3r_resize_aa_bilinear_u8; agrees with torchvision to ~1e-6, not bitwise);
  * the SLAM front end's preproc_frame (must3r/slam/model.py:99-120 with _resize_pil_image,
    dust3r/dust3r/utils/image.py:64-71): PIL resize (LANCZOS when shrinking, BICUBIC otherwise), crop, ImgNorm
    (m3r_resample_pil_u8; bitwise equal to PIL + torchvision).

Frames are RGB uint8 HWC.  Host frames (paths decoded by PIL, numpy arrays, CPU tensors) are copied into pinned memory
and uploaded with an asynchronous copy on the current stream; CUDA tensors are read in place (any row pitch).  The
coefficient tables are computed here, on the host, in double precision like Pillow (float like aten), and cached per
geometry; the kernels only do the multiply-adds.  Scratch memory comes from model.common.workspace, so two host threads
on their own streams (the SLAM worker) do not share it.  Nothing synchronises the device.
"""
from __future__ import annotations

import functools
import math
import os
from typing import Optional, Tuple

import numpy as np
import torch

from .. import ops
from ..model import common as cm

# output (long side, short side) per aspect ratio, keyed by the long side
ratios_resolutions = {
    224: {1.0: [224, 224]},
    336: {1.0: [336, 336]},
    384: {4 / 3: [384, 288], 3 / 2: [384, 256], 2 / 1: [384, 192], 3 / 1: [384, 128]},
    448: {1.0: [448, 448]},
    512: {4 / 3: [512, 384], 32 / 21: [512, 336], 16 / 9: [512, 288], 2 / 1: [512, 256], 16 / 5: [512, 160]},
    768: {4 / 3: [768, 576], 3 / 2: [768, 512], 16 / 9: [768, 432], 2 / 1: [768, 384], 16 / 5: [768, 240]},
}


def get_HW_resolution(H, W, maxdim, patchsize=16):
    """(h, w) of the tabulated resolution whose aspect ratio is nearest to W / H (orientation preserved)."""
    if isinstance(maxdim, int) and maxdim not in ratios_resolutions:
        raise AssertionError(f"Error, maxdim={maxdim} not implemented yet.")
    table = maxdim if isinstance(maxdim, dict) else ratios_resolutions[maxdim]
    if isinstance(patchsize, tuple):
        assert len(patchsize) == 2 and patchsize[0] == patchsize[1], "Error, non square patches not managed"
    ratios = np.array(list(table.keys()))
    landscape = W >= H
    diff = np.abs(W / H - ratios) if landscape else np.abs(W / H - 1 / ratios)
    long_short = table[ratios[np.argmin(diff)]]
    if isinstance(maxdim, int):
        assert max(long_short) == maxdim
    return long_short[::-1] if landscape else long_short


class _Geometry:
    """One input size's resize: crop box (top, left, h, w) of the source, output (h, w) and the reference's matrices."""

    def __init__(self, crop, out_hw, to_rescaled, to_orig):
        self.crop, self.out_hw, self.to_rescaled, self.to_orig = crop, tuple(out_hw), to_rescaled, to_orig


def _demo_geometry(maxdim, H, W) -> _Geometry:
    table = maxdim if isinstance(maxdim, dict) else ratios_resolutions[maxdim]
    if [max(H, W), min(H, W)] in table.values():
        return _Geometry((0, 0, H, W), (H, W), np.eye(3), np.eye(3))
    th, tw = get_HW_resolution(H, W, maxdim)
    ratio, target = W / H, tw / th
    to_orig_crop, to_rescaled_crop = np.eye(3), np.eye(3)
    if abs(ratio - target) < np.finfo(np.float32).eps:
        ch, cw = H, W
    elif ratio < target:                      # too tall: crop rows
        ch, cw = int(W / target), W
        to_orig_crop[1, 2], to_rescaled_crop[1, 2] = (H - ch) / 2.0, -(H - ch) / 2.0
    else:                                     # too wide: crop columns
        ch, cw = H, int(H * target)
        to_orig_crop[0, 2], to_rescaled_crop[0, 2] = (W - cw) / 2.0, -(W - cw) / 2.0
    to_orig_resize = np.array([[cw / tw, 0, 0], [0, ch / th, 0], [0, 0, 1]])
    to_rescaled_resize = np.array([[tw / cw, 0, 0], [0, th / ch, 0], [0, 0, 1]])
    # torchvision.transforms.functional.center_crop's offsets (Python round: half to even)
    top, left = int(round((H - ch) / 2.0)), int(round((W - cw) / 2.0))
    return _Geometry((top, left, ch, cw), (th, tw), to_rescaled_resize @ to_rescaled_crop, to_orig_crop @ to_orig_resize)


# ------------------------------------------------------------------------------------------- coefficient tables
PIL_PRECISION_BITS = 22        # Pillow's 8-bit resampler: 32 - 8 - 2 fractional bits


def _sinc(x):
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x


def _lanczos(x):
    return _sinc(x) * _sinc(x / 3) if -3.0 <= x < 3.0 else 0.0


def _bicubic(x):                # Keys cubic, a = -0.5
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


PIL_FILTERS = {"lanczos": (_lanczos, 3.0), "bicubic": (_bicubic, 2.0)}


def _identity_tables(n, dtype, one):
    bounds = np.stack([np.arange(n, dtype=np.int32), np.ones(n, dtype=np.int32)], 1)
    return bounds, np.full((n, 1), one, dtype=dtype)


@functools.lru_cache(maxsize=256)
def pil_coeffs(in_size: int, out_size: int, filt: str) -> Tuple[np.ndarray, np.ndarray]:
    """Pillow's resampling coefficients for one axis: bounds [out, 2] int32 (first input index, taps) and weights
    [out, k] int32 with 22 fractional bits.  Double precision, per-output normalisation, then rounding half away from
    zero to integers, as Pillow's precompute_coeffs / normalize_coeffs_8bpc.  An axis whose size does not change is a
    pass Pillow skips: its table is the identity (weight 1.0)."""
    if in_size == out_size:
        return _identity_tables(out_size, np.int32, 1 << PIL_PRECISION_BITS)
    fn, support = PIL_FILTERS[filt]
    scale = filterscale = float(in_size) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = support * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    weights = np.zeros((out_size, ksize), np.int32)
    inv = 1.0 / filterscale
    one = float(1 << PIL_PRECISION_BITS)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [fn((x + xmin - center + 0.5) * inv) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        if ww != 0.0:
            k = [w / ww for w in k]
        weights[xx, :xmax] = [int(-0.5 + w * one) if w < 0 else int(0.5 + w * one) for w in k]
        bounds[xx] = (xmin, xmax)
    return bounds, weights


@functools.lru_cache(maxsize=256)
def aa_bilinear_coeffs(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray]:
    """aten's antialiased bilinear weights for one axis (align_corners=False, no explicit scale): bounds [out, 2]
    int32 and fp32 weights [out, k], triangle filter widened by the downscale factor, normalised per output."""
    if in_size == out_size:
        return _identity_tables(out_size, np.float32, 1.0)
    f32 = np.float32
    scale = f32(in_size) / f32(out_size)
    support = f32(scale) if scale >= 1.0 else f32(1.0)
    invscale = f32(1.0) / scale if scale >= 1.0 else f32(1.0)
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int32)
    weights = np.zeros((out_size, ksize), np.float32)
    for i in range(out_size):
        center = f32(float(scale) * (i + 0.5))
        xmin = max(int(float(center - support) + 0.5), 0)
        xsize = min(max(min(int(float(center + support) + 0.5), in_size) - xmin, 0), ksize)
        w = np.zeros(xsize, np.float32)
        for j in range(xsize):
            x = abs(f32(float(f32(j + xmin) - center) + 0.5) * float(invscale))
            w[j] = f32(1.0 - x) if x < 1.0 else f32(0.0)
        total = f32(0.0)
        for v in w:
            total = f32(total + v)
        if total != 0.0:
            w = (w / total).astype(np.float32)
        weights[i, :xsize] = w
        bounds[i] = (xmin, xsize)
    return bounds, weights


def _pil_plan(in_h, in_w, out_h, out_w, filt):
    """Tables of one PIL resize, with the vertical bounds relative to the first source row the horizontal pass reads
    (Pillow resamples only rows [ybox_first, ybox_last) horizontally)."""
    xb, xw = pil_coeffs(in_w, out_w, filt)
    yb, yw = pil_coeffs(in_h, out_h, filt)
    row0 = int(yb[0, 0])
    rows = int(yb[-1, 0] + yb[-1, 1]) - row0
    yb = yb.copy()
    yb[:, 0] -= row0
    return xb, xw, yb, yw, row0, rows


# ------------------------------------------------------------------------------------------- device plumbing
def _device(device) -> torch.device:
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"must3r_b200 image preprocessing runs on CUDA devices only (got device {dev})")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


def _align(n: int) -> int:
    return (n + 255) // 256 * 256


@functools.lru_cache(maxsize=128)
def _packed_tables(key):
    """All tables of one geometry in one pinned host buffer (read-only once built, so it can be the source of any
    number of asynchronous uploads) and the byte offset of each."""
    kind, in_h, in_w, out_h, out_w, filt = key
    if kind == "pil":
        xb, xw, yb, yw, row0, rows = _pil_plan(in_h, in_w, out_h, out_w, filt)
        extra = (row0, rows)
    else:
        xb, xw = aa_bilinear_coeffs(in_w, out_w)
        yb, yw = aa_bilinear_coeffs(in_h, out_h)
        extra = ()
    parts = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in (xb, xw, yb, yw)]
    offs, n = [], 0
    for p in parts:
        offs.append(n)
        n += _align(p.size)
    host = torch.zeros(n, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    for o, p in zip(offs, parts):
        host[o:o + p.size] = torch.from_numpy(p)
    return host, offs, xw.shape[1], yw.shape[1], extra


def _as_frames(frames, dev) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """uint8 [V,H,W,3]: (device tensor read in place, None) or (None, pinned host copy to upload)."""
    if isinstance(frames, torch.Tensor) and frames.is_cuda:
        t = frames if frames.dim() == 4 else frames[None]
        if t.dtype != torch.uint8 or t.shape[-1] != 3:
            raise ValueError(f"expected RGB uint8 frames [V,H,W,3], got {tuple(t.shape)} {t.dtype}")
        if t.device != dev:
            raise ValueError(f"frames are on {t.device}, not on {dev}")
        if t.stride(3) != 1 or t.stride(2) != 3:
            t = t.contiguous()
        return t, None
    arrs = [frames] if not isinstance(frames, (list, tuple)) else list(frames)
    arrs = [a.numpy() if isinstance(a, torch.Tensor) else np.asarray(a) for a in arrs]
    if len(arrs) == 1 and arrs[0].ndim == 4:
        arrs = list(arrs[0])
    for a in arrs:
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape != arrs[0].shape:
            raise ValueError(f"expected RGB uint8 frames [H,W,3] of one size, got {a.shape} {a.dtype}")
    pinned = torch.empty((len(arrs),) + arrs[0].shape, dtype=torch.uint8, pin_memory=True)
    dst = pinned.numpy()
    for i, a in enumerate(arrs):
        dst[i] = a
    return None, pinned


def _run(kind, frames, in_hw, out_hw, dev, *, filt="", crop=None, src_box=None, want_u8=False):
    """Enqueue one launch over V frames of one size on the current stream; returns (fp32 [V,3,h,w] or None, uint8
    [V,out_h,out_w,3] or None).  PIL: `crop` = (x, y, w, h) box of the resized image.  AA: `src_box` = (top, left, h, w)
    region of the source that is resized."""
    with torch.cuda.device(dev):
        dsrc, pinned = _as_frames(frames, dev)
        V = (dsrc if dsrc is not None else pinned).shape[0]
        H, W = in_hw
        if (dsrc if dsrc is not None else pinned).shape[1:3] != (H, W):
            raise ValueError("frames do not have the size this resize was planned for")
        oh, ow = out_hw
        if kind == "aa":
            top, left, sh, sw = src_box
            key = ("aa", sh, sw, oh, ow, "")
        else:
            key = ("pil", H, W, oh, ow, filt)
        tabs, offs, xk, yk, extra = _packed_tables(key)
        if kind == "pil":
            row0, rows = extra
            tmp_bytes = V * rows * ow * 3
        else:
            tmp_bytes = V * 3 * sh * ow * 4
        up_bytes = 0 if pinned is None else pinned.numel()
        n_tab = tabs.numel()
        ws = cm.workspace(dev, n_tab + _align(up_bytes) + _align(tmp_bytes), "img")
        ws[:n_tab].copy_(tabs, non_blocking=True)
        if pinned is not None:
            up = ws[n_tab:n_tab + up_bytes]
            up.copy_(pinned.view(-1), non_blocking=True)
            dsrc = up.view(pinned.shape)
        tmp = ws[n_tab + _align(up_bytes):]
        tab = [ws[o:] for o in offs]
        if kind == "pil":
            cx, cy, cw, ch = crop if crop is not None else (0, 0, ow, oh)
            out = torch.empty((V, 3, ch, cw), device=dev, dtype=torch.float32) if crop is not None else None
            u8 = torch.empty((V, oh, ow, 3), device=dev, dtype=torch.uint8) if want_u8 else None
            ops.resample_pil_u8(dsrc, tab, xk, yk, (oh, ow), row0, rows, tmp, (cx, cy, cw, ch), out=out, out_u8=u8)
            return out, u8
        src = dsrc[:, top:top + sh, left:left + sw]
        out = torch.empty((V, 3, oh, ow), device=dev, dtype=torch.float32)
        ops.resize_aa_bilinear_u8(src, tab, xk, yk, (oh, ow), tmp, out)
        return out, None


# ------------------------------------------------------------------------------------------- the demo path
def get_resize_function(maxdim, patch_size, H, W):
    """(op, to_rescaled, to_orig) as the reference's get_resize_function (must3r/tools/image.py:53-93).  `op` takes
    RGB uint8 frames [H,W,3] or [V,H,W,3] (numpy, CPU or CUDA tensor) instead of an ImgNorm'ed tensor and returns the
    ImgNorm'ed, center-cropped, resized fp32 images [3,h,w] / [V,3,h,w] on the GPU (the current CUDA device, or the
    frames' device); the normalisation is fused into the kernel."""
    geo = _demo_geometry(maxdim, H, W)

    def op(frames, device=None):
        single = getattr(frames, "ndim", 0) == 3
        dev = _device(device if device is not None else
                      (frames.device if isinstance(frames, torch.Tensor) and frames.is_cuda else "cuda"))
        out, _ = _run("aa", frames, (H, W), geo.out_hw, dev, src_box=geo.crop)
        return out[0] if single else out

    return op, geo.to_rescaled, geo.to_orig


def _load_rgb(item):
    if isinstance(item, (str, os.PathLike)):
        import PIL.Image
        with PIL.Image.open(item) as im:
            return np.asarray(im.convert("RGB")), str(item)
    if isinstance(item, torch.Tensor):
        return item, None
    return np.asarray(item), None


def load_images(folder_content, size, patch_size=16, verbose=True, device="cuda"):
    """The demo's load_images (must3r/demo/inference.py:63-76): a list of dict(img=[3,h,w] fp32 on `device`,
    true_shape=np.int32([h, w])) in input order.  Items are image paths or RGB uint8 [H,W,3] numpy arrays / tensors.
    Paths are decoded as PIL's .convert('RGB') (no EXIF transpose, as the reference) by engine/imagefiles.py: the
    files a GPU decoder takes on the GPU in batches (waiting for each batch's status words is the one host wait), other
    files by PIL on the host.  Frames of one size are resized in one launch."""
    from . import imagefiles
    dev = _device(device)
    items = list(folder_content)
    paths = [k for k, item in enumerate(items) if isinstance(item, (str, os.PathLike))]
    with torch.cuda.device(dev):
        decoded = dict(zip(paths, imagefiles.decode_parsed_all([imagefiles.parse(items[k], False) for k in paths],
                                                               dev))) if paths else {}
    frames, names, groups = [], [], {}
    for i, item in enumerate(items):
        f, name = (decoded[i], str(item)) if i in decoded else _load_rgb(item)
        if f.ndim != 3 or f.shape[2] != 3:
            raise ValueError(f"item {i}: expected an RGB image [H,W,3], got shape {tuple(f.shape)}")
        frames.append(f)
        names.append(name if name is not None else f"image {i}")
        groups.setdefault(tuple(f.shape[:2]), []).append(i)
    imgs = [None] * len(frames)
    for (H, W), idx in groups.items():
        geo = _demo_geometry(size, H, W)
        group = [frames[i] for i in idx]
        if any(isinstance(f, torch.Tensor) and f.is_cuda for f in group):
            group = torch.stack([f.to(dev) if isinstance(f, torch.Tensor) else torch.from_numpy(np.asarray(f)).to(dev)
                                 for f in group])
        out, _ = _run("aa", group, (H, W), geo.out_hw, dev, src_box=geo.crop)
        for j, i in enumerate(idx):
            imgs[i] = dict(img=out[j], true_shape=np.int32([geo.out_hw[0], geo.out_hw[1]]))
    if verbose:
        for name, f, d in zip(names, frames, imgs):
            print(f' - adding {name} with resolution {f.shape[1]}x{f.shape[0]} --> {d["true_shape"][1]}x{d["true_shape"][0]}')
    return imgs


# ------------------------------------------------------------------------------------------- the SLAM path
def _slam_geometry(H1, W1, res):
    """What preproc_frame computes from the frame size: resized (W, H), filter, crop box (x, y, w, h), focal ratio."""
    longsize = res
    if res in (224, 336, 448):
        longsize = max(W1, H1) / min(W1, H1) * res       # the short side becomes res
    S = max(W1, H1)
    filt = "lanczos" if S > longsize else "bicubic"
    W, H = (int(round(x * longsize / S)) for x in (W1, H1))
    cx, cy = W // 2, H // 2
    if res in (224, 336, 448):
        halfw = halfh = res // 2
    else:
        halfw, halfh = ((2 * cx) // 16) * 8, ((2 * cy) // 16) * 8
    return (H, W), filt, (cx - halfw, cy - halfh, 2 * halfw, 2 * halfh), W1 / W


def preproc_frame(img, idx, res=512, device="cuda"):
    """The SLAM front end's preproc_frame (must3r/slam/model.py:99-120): returns (dict(img=[1,3,h,w] fp32 on
    `device`, true_shape=np.int32([[h, w]]), idx, instance=str(idx), offset=np.int32([[x0, y0]])), to_orig_focal).
    img: RGB uint8 [H,W,3] (numpy, CPU or CUDA tensor).  Bitwise equal to the reference."""
    dev = _device(device)
    H1, W1 = int(img.shape[0]), int(img.shape[1])
    (H, W), filt, (x0, y0, cw, ch), focal = _slam_geometry(H1, W1, res)
    out, _ = _run("pil", img, (H1, W1), (H, W), dev, filt=filt, crop=(x0, y0, cw, ch))
    return dict(img=out, true_shape=np.int32([[ch, cw]]), idx=idx, instance=str(idx), offset=np.int32([[x0, y0]])), focal


def resize_pil(frames, out_hw, filt, device="cuda", crop=None):
    """PIL-exact resize of RGB uint8 frames [V,H,W,3] (or one [H,W,3]) to out_hw = (h, w) with `filt` 'lanczos' or
    'bicubic' (the same size is a copy): returns (uint8 [V,h,w,3], fp32 ImgNorm of the crop box (x, y, w, h) or None)."""
    dev = _device(device)
    H, W = int(frames.shape[-3]), int(frames.shape[-2])
    out, u8 = _run("pil", frames, (H, W), tuple(out_hw), dev, filt=filt, crop=crop, want_u8=True)
    return u8, out
