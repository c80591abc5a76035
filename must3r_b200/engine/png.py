"""PNG files decoded on the GPU by the CUDA decoder (csrc/png.cu), bitwise what np.asarray(PIL.Image.open(p).convert('RGB'))
gives (after PIL.ImageOps.exif_transpose when asked).

The host reads each file and walks its chunks (m3r_png_parse / m3r_png_prepare, through ctypes, so the GIL is released):
only the palette and the concatenated IDAT payloads are staged in pinned memory and cross PCIe.  One launch sequence
inflates and unfilters a batch of images of any sizes and colour types on the current stream.  Reading the images'
status words back is the one host wait per batch: an image whose stream the decoder found malformed is decoded again by
Pillow, so the caller gets Pillow's exact outcome, pixels or exception.  Scratch memory comes from
model.common.workspace (per stream).

A file goes to the GPU when it is an 8-bit, non-interlaced L, RGB, P, LA or RGBA PNG whose chunks the parser accepts,
when it has at most PIL.Image.MAX_IMAGE_PIXELS pixels (so Pillow's decompression-bomb warning and error still come from
Pillow), when Pillow opens it as that mode and size (so whatever Pillow's chunk handlers reject before the image data is
still rejected by Pillow), and, with the EXIF transpose, when it has no eXIf and no text chunk (Pillow's getexif reads
EXIF from both): such a file is never transposed.  Everything else, 16-bit and interlaced PNGs included, goes to Pillow.
"""
from __future__ import annotations

import ctypes as C
import io
from typing import List, Optional, Sequence

import torch

from .. import _lib, ops
from ..model import common as cm

# a batch's scanline workspace stays below this (about 80 1080p RGB frames)
WORK_BUDGET = 512 << 20

SIGNATURE = b"\x89PNG\r\n\x1a\n"
MODES = {0: "L", 2: "RGB", 3: "P", 4: "LA", 6: "RGBA"}


def _align(n: int) -> int:
    return (n + 255) // 256 * 256


def _pillow_opens(data: bytes, info) -> bool:
    """Pillow reads the chunks before the image data (CRCs, its chunk handlers) and sees this mode and size."""
    import PIL.Image
    try:
        with PIL.Image.open(io.BytesIO(data), formats=["PNG"]) as im:
            return im.mode == MODES[info.color_type] and im.size == (info.width, info.height)
    except Exception:
        return False


class Parsed:
    """One file read into memory and its chunks walked: `gpu` says whether the GPU decoder takes it."""

    def __init__(self, path, exif_transpose: bool, data: Optional[bytes] = None):
        import PIL.Image
        import PIL.PngImagePlugin
        self.path, self.exif_transpose = path, exif_transpose
        if data is None:
            with open(path, "rb") as f:
                data = f.read()
        self.data = data
        self.info = i = ops.png_parse(self.data)
        limit = PIL.Image.MAX_IMAGE_PIXELS
        self.gpu = (bool(i.eligible) and (limit is None or i.width * i.height <= limit)
                    and not (exif_transpose and (i.has_exif or i.has_text))
                    and i.text_bytes <= PIL.PngImagePlugin.MAX_TEXT_MEMORY and _pillow_opens(self.data, i))

    @property
    def out_hw(self):
        return self.info.height, self.info.width

    @property
    def work_bytes(self) -> int:
        i = self.info
        return i.height * (1 + i.width * i.channels) + i.prep_bytes


def decode_parsed(items: Sequence[Parsed], dev: torch.device) -> List[Optional[torch.Tensor]]:
    """Decode eligible parsed files as one batch on the current stream of `dev`; returns uint8 [H,W,3] CUDA tensors,
    None where the decoder reported the stream malformed (the caller uses Pillow).  Waits for the batch's status words
    (one event wait, no device synchronisation)."""
    outs: List[Optional[torch.Tensor]] = [None] * len(items)
    if not items:
        return outs
    with torch.cuda.device(dev):
        offs, n = [], 0
        for it in items:
            offs.append(n)
            n += _align(it.info.prep_bytes)
        host = torch.empty(n + _align(C.sizeof(_lib.PngDesc) * len(items)), dtype=torch.uint8, pin_memory=True)
        base = host.data_ptr()
        arr = (_lib.PngDesc * len(items))(*[ops.png_prepare(it.data, it.info, 1, base + o, o)
                                            for it, o in zip(items, offs)])
        work_bytes = ops.png_plan(arr)
        for d, k in zip(arr, range(len(items))):
            oh, ow = items[k].out_hw
            outs[k] = torch.empty((oh, ow, 3), dtype=torch.uint8, device=dev)
            d.out = outs[k].data_ptr()
        C.memmove(base + n, C.addressof(arr), C.sizeof(arr))
        blob_bytes = n + C.sizeof(arr)
        ws = cm.workspace(dev, _align(blob_bytes) + work_bytes + 256, "png")
        blob, work = ws[:blob_bytes], ws[_align(blob_bytes):]
        blob.copy_(host[:blob_bytes], non_blocking=True)
        status = torch.empty(len(items), dtype=torch.int32, device=dev)
        ops.png_decode(arr, blob, n, work, status)
        st_host = torch.empty(len(items), dtype=torch.int32, pin_memory=True)
        st_host.copy_(status, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()                  # the one host wait: the status words (the staging buffer is free after it)
        for k, s in enumerate(st_host.tolist()):
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
