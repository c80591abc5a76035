"""Baseline JPEGs decoded on the GPU by the CUDA decoder (csrc/jpeg.cu), bitwise what
np.asarray(PIL.Image.open(p).convert('RGB')) gives (after PIL.ImageOps.exif_transpose when asked).  engine/imagefiles.py
decides which decoder takes a file.

The host reads each file, parses its headers and makes one pass over its entropy-coded data into a pinned buffer
(m3r_jpeg_prepare, through ctypes, so the GIL is released); only those compressed bytes cross PCIe.  One launch sequence
decodes a batch of images of any sizes and samplings on the current stream.  Reading the images' status words back is
the one host wait per batch: an image whose stream the decoder found malformed is decoded again by Pillow, so the caller
gets Pillow's exact outcome, pixels or exception.  Scratch memory comes from model.common.workspace (per stream).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import torch

from .. import _lib, ops
from ..model import common as cm

# a batch's coefficient and plane workspace stays below this (about 40 1080p frames)
WORK_BUDGET = 512 << 20


def _align(n: int) -> int:
    return (n + 255) // 256 * 256


class Parsed:
    """One file read into memory and parsed: `info.eligible` and the orientation decide whether the GPU takes it."""

    def __init__(self, path, exif_transpose: bool, data: Optional[bytes] = None):
        self.path, self.exif_transpose = path, exif_transpose
        if data is None:
            with open(path, "rb") as f:
                data = f.read()
        self.data = data
        self.info = ops.jpeg_parse(self.data)
        self.orientation = self.info.orientation if exif_transpose else 1
        self.gpu = bool(self.info.eligible) and (not exif_transpose or bool(self.info.orientation_exact))

    @property
    def out_hw(self):
        H, W = self.info.height, self.info.width
        return (W, H) if self.orientation in (5, 6, 7, 8) else (H, W)

    @property
    def work_bytes(self) -> int:
        i = self.info
        blocks = ((i.width + 8 * i.hs[0] - 1) // (8 * i.hs[0])) * ((i.height + 8 * i.vs[0] - 1) // (8 * i.vs[0]))
        return blocks * (i.hs[0] * i.vs[0] + 2) * 64 * 3 + i.prep_bytes


def decode_parsed(items: Sequence[Parsed], dev: torch.device) -> List[Optional[torch.Tensor]]:
    """Decode eligible parsed files as one batch on the current stream of `dev`; returns uint8 [H,W,3] CUDA tensors,
    None where the decoder reported the stream malformed or the data turned out ineligible (the caller uses Pillow).
    Waits for the batch's status words (one event wait, no device synchronisation)."""
    outs: List[Optional[torch.Tensor]] = [None] * len(items)
    if not items:
        return outs
    with torch.cuda.device(dev):
        offs, n = [], 0
        for it in items:
            offs.append(n)
            n += _align(it.info.prep_bytes)
        host = torch.empty(n + _align(C.sizeof(_lib.JpegDesc) * len(items)), dtype=torch.uint8, pin_memory=True)
        base = host.data_ptr()
        descs, idx = [], []
        for k, (it, o) in enumerate(zip(items, offs)):
            d = ops.jpeg_prepare(it.data, it.info, it.orientation, base + o, o)
            if d is not None:
                descs.append(d)
                idx.append(k)
        if not descs:
            return outs
        arr = (_lib.JpegDesc * len(descs))(*descs)
        work_bytes = ops.jpeg_plan(arr)
        for d, k in zip(arr, idx):
            oh, ow = items[k].out_hw
            outs[k] = torch.empty((oh, ow, 3), dtype=torch.uint8, device=dev)
            d.out = outs[k].data_ptr()
        C.memmove(base + n, C.addressof(arr), C.sizeof(arr))
        blob_bytes = n + C.sizeof(arr)
        ws = cm.workspace(dev, _align(blob_bytes) + work_bytes + 256, "jpeg")
        blob, work = ws[:blob_bytes], ws[_align(blob_bytes):]
        blob.copy_(host[:blob_bytes], non_blocking=True)
        status = torch.empty(len(descs), dtype=torch.int32, device=dev)
        ops.jpeg_decode(arr, blob, n, work, status)
        st_host = torch.empty(len(descs), dtype=torch.int32, pin_memory=True)
        st_host.copy_(status, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()                  # the one host wait: the status words (the staging buffer is free after it)
        for s, k in zip(st_host.tolist(), idx):
            if s:
                outs[k] = None
        return outs


def batches(items: Sequence[Parsed]):
    batch, work = [], 0
    for it in items:
        if batch and (len(batch) >= 64 or work + it.work_bytes > WORK_BUDGET):
            yield batch
            batch, work = [], 0
        batch.append(it)
        work += it.work_bytes
    if batch:
        yield batch


def decode_files(paths: Sequence, device="cuda", exif_transpose: bool = False) -> List[torch.Tensor]:
    """engine.imagefiles.decode_files: one CUDA uint8 [H,W,3] tensor per path, bitwise equal to
    np.asarray(PIL.Image.open(p).convert('RGB')) (after PIL.ImageOps.exif_transpose when `exif_transpose`), eligible
    JPEGs and PNGs decoded on the GPU, anything else by Pillow, whose exceptions propagate."""
    from . import imagefiles
    return imagefiles.decode_files(paths, device, exif_transpose)
