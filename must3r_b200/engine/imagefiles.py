"""Image files as CUDA uint8 [H,W,3] tensors, bitwise what np.asarray(PIL.Image.open(p).convert('RGB')) gives (after
PIL.ImageOps.exif_transpose when asked): the one place that decides which decoder takes a file.

Baseline JPEGs go to the CUDA JPEG decoder (engine/jpeg.py) and 8-bit non-interlaced PNGs to the CUDA PNG decoder
(engine/png.py), in batches under each decoder's workspace budget; every other file, and any file whose stream a GPU
decoder reports malformed, is decoded by Pillow on the host and uploaded from pinned memory on the current stream, so
Pillow's exceptions propagate unchanged.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np
import torch

from . import jpeg, png


def pillow_decode(path, exif_transpose: bool) -> np.ndarray:
    """RGB uint8 [H,W,3] as Pillow decodes it (the reference's loaders)."""
    import PIL.Image
    import PIL.ImageOps
    with PIL.Image.open(path) as im:
        if exif_transpose:
            im = PIL.ImageOps.exif_transpose(im)
        return np.asarray(im.convert('RGB'))


def _decoder(data: bytes):
    """The Parsed class of the decoder a file's first bytes name (jpeg.Parsed for anything that is not a PNG; its `gpu`
    is False for what is not a JPEG either)."""
    return png.Parsed if data[:8] == png.SIGNATURE else jpeg.Parsed


def parse(path, exif_transpose: bool):
    """The file read into memory and parsed by the decoder its signature names."""
    with open(path, "rb") as f:
        data = f.read()
    return _decoder(data)(path, exif_transpose, data)


def upload(a: np.ndarray, dev: torch.device) -> torch.Tensor:
    """A host frame copied to `dev` through pinned memory on the current stream (no host wait)."""
    buf = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
    buf.numpy()[...] = a
    out = torch.empty(a.shape, dtype=torch.uint8, device=dev)
    out.copy_(buf, non_blocking=True)
    return out


def decode_parsed_all(items: Sequence, dev: torch.device) -> List[torch.Tensor]:
    """Every parsed file as a CUDA uint8 [H,W,3] tensor on the current stream: the ones a GPU decoder takes decoded in
    batches per decoder, the rest (and any a decoder handed back) by Pillow and uploaded."""
    out: List[Optional[torch.Tensor]] = [None] * len(items)
    for mod in (jpeg, png):
        idx = [k for k, it in enumerate(items) if it.gpu and isinstance(it, mod.Parsed)]
        pos = 0
        for batch in mod.batches([items[k] for k in idx]):
            for k, t in zip(idx[pos:pos + len(batch)], mod.decode_parsed(batch, dev)):
                out[k] = t
            pos += len(batch)
    for k, it in enumerate(items):
        if out[k] is None:
            out[k] = upload(pillow_decode(it.path, it.exif_transpose), dev)
    return out


# The formats the SLAM read-ahead decodes on the GPU.  It decodes one frame at a time, and one PNG inflates on a single
# warp (deflate is serial within a stream), which takes longer than Pillow on a host thread (README, input pipeline),
# so its PNG frames stay with Pillow.
READ_AHEAD_ON_GPU = (jpeg.Parsed,)


def decode_frame(path, dev: torch.device) -> torch.Tensor:
    """One frame of the SLAM read-ahead (EXIF orientation applied) on the current stream, decoded by itself.  A format
    the read-ahead keeps on the host is decoded by Pillow straight away, without being parsed for the GPU."""
    with open(path, "rb") as f:
        head = f.read(8)
    if _decoder(head) not in READ_AHEAD_ON_GPU:
        return upload(pillow_decode(path, True), dev)
    return decode_parsed_all([parse(path, True)], dev)[0]


def decode_files(paths: Sequence, device="cuda", exif_transpose: bool = False) -> List[torch.Tensor]:
    """One CUDA uint8 [H,W,3] tensor per path, bitwise equal to np.asarray(PIL.Image.open(p).convert('RGB')) (after
    PIL.ImageOps.exif_transpose when `exif_transpose`).  Eligible JPEGs and PNGs are decoded on the GPU; anything else,
    and any file whose stream a GPU decoder reports malformed, by Pillow, whose exceptions propagate."""
    dev = torch.device(device)
    if dev.type != "cuda":
        raise RuntimeError(f"must3r_b200 image decoding runs on CUDA devices only (got device {dev})")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        return decode_parsed_all([parse(p, exif_transpose) for p in paths], dev)
