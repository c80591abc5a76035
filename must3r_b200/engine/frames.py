"""Frame sources of the online SLAM command line: the reference's image-folder loaders (must3r/slam/data.py:
ImageCollection, AutoMultiLoader) and its grab_frame (must3r/slam/slam.py:38-46), plus a bounded read-ahead that
decodes the frames on a host thread and hands them to the GPU.

The loaders only sequence file paths; nothing is decoded while the schedule of a run is built.  The sequencing is the
reference's: with several folders the frames alternate between them, a folder that has run out is skipped (its turn
goes to the next one), and `grab()` moves every folder on by one frame.  Video files and camera streams (cv2) are not
supported.

Frames are RGB uint8 with the EXIF orientation applied (as cv2.imread does), bitwise what PIL decodes: `decode` runs
PIL on the host; the read-ahead hands each file to engine/imagefiles.py, which decodes it on the GPU or with PIL.  The
reference decodes with cv2.imread and converts BGR to RGB, so the arrays are the same for lossless formats such as PNG;
for JPEG the two decoders may differ in the last bits.
"""
from __future__ import annotations

import os
import queue
import threading
import time
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

# must3r/slam/data.py:7-8: the extensions cv2.imread reads
IM_FORMATS = ['jpg', 'jpeg', 'jpe', 'png', 'tiff', 'tif', 'bmp', 'dib', 'jp2',
              'webp', 'pbm', 'pgm', 'ppm', 'pxm', 'pnm', 'pfm', 'sr', 'ras', 'exr', 'hdr', 'pic']


def list_frames(rootdir: str, image_string: Optional[str] = None) -> List[str]:
    """The files of `rootdir`, sorted by name, whose extension is one of IM_FORMATS (any case) and whose name contains
    `image_string` (if given)."""
    def sel(name):
        return name.split('.')[-1].lower() in IM_FORMATS and (image_string is None or image_string in name)
    return [n for n in sorted(os.listdir(rootdir)) if sel(n)]


class ImageCollection:
    """One folder of frames (must3r/slam/data.py:83-125); `read()` returns (None, path) or (None, None) past the end."""

    def __init__(self, rootdir: str, image_string: Optional[str] = None):
        self.rootdir = rootdir
        self.frames = list_frames(rootdir, image_string)
        if not self.frames:
            raise ValueError(f"no image files in {rootdir}" + (f" containing '{image_string}'" if image_string else ""))
        self.current_frame = 0

    def __len__(self):
        return len(self.frames)

    def grab(self):
        self.current_frame += 1

    def read(self):
        path = None
        if self.current_frame < len(self):
            path = os.path.join(self.rootdir, self.frames[self.current_frame])
            self.current_frame += 1
        return None, path


class AutoMultiLoader:
    """Frames taken in turn from several folders (must3r/slam/data.py:44-77); `read()` returns (None, path, cam_id)."""

    def __init__(self, inp: Sequence[str], image_string: Optional[str] = None):
        self.CAMERAS = [ImageCollection(d, image_string) for d in inp]
        self.whos_turn = 0

    def __len__(self):
        return int(sum(len(cam) for cam in self.CAMERAS))

    def next_agent(self):
        self.whos_turn = (self.whos_turn + 1) % len(self.CAMERAS)

    def grab(self):
        for _ in range(len(self.CAMERAS)):
            self.CAMERAS[self.whos_turn].grab()
            self.next_agent()

    def read(self):
        path, loop_c = None, 0
        while path is None and loop_c < len(self.CAMERAS):
            ret, path = self.CAMERAS[self.whos_turn].read()
            camid = self.whos_turn
            self.next_agent()
            loop_c += 1
        return ret, path, camid


def grab_frame(camera, skip_every: int = 1) -> Tuple[Optional[str], int]:
    """must3r/slam/slam.py:38-46: read one frame, then grab (skip) skip_every - 1 more -> (path or None, cam_id)."""
    read = camera.read()
    camid = 0 if len(read) != 3 else read[2]
    for _ in range(skip_every - 1):
        camera.grab()
    return read[1], camid


def schedule(camera, skip_every: int = 1, grab_every: int = 1):
    """The frames the reference's headless main (must3r/slam/slam.py:648-656) feeds to the model: `len(camera) //
    skip_every` items (path, cam_id, timestamp = frame_id * skip_every), and the path of the frame read after the last
    one (None past the end), whose size the reference also records.  `grab_every` is grab_frame's skip: the reference's
    main assigns SKIP_EVERY to a local name, so its grab_frame keeps skipping nothing (grab_every = 1)."""
    path, cam_id = grab_frame(camera, grab_every)
    items = []
    for frame_id in range(len(camera) // skip_every):
        if path is None:
            raise ValueError(f"frame {frame_id}: the sources ran out before len(sources) // skip_every frames")
        items.append((path, cam_id, frame_id * skip_every))
        path, cam_id = grab_frame(camera, grab_every)
    return items, path


def decode(path: str) -> np.ndarray:
    """RGB uint8 [H,W,3] of an image file (PIL, EXIF orientation applied)."""
    import PIL.Image
    import PIL.ImageOps
    with PIL.Image.open(path) as im:
        im = PIL.ImageOps.exif_transpose(im)
        return np.asarray(im.convert('RGB'))


def image_size(path: str) -> Tuple[int, int]:
    """(H, W) of decode(path), from the file's header and EXIF orientation, without decoding the pixels."""
    import PIL.Image
    with PIL.Image.open(path) as im:
        W, H = im.size
        if im.getexif().get(0x0112) in (5, 6, 7, 8):        # transposed orientations swap the axes
            W, H = H, W
    return H, W


class ReadAhead:
    """Decodes `paths` in order on one host thread, up to `depth` frames ahead of the consumer.  The reader reads each
    file and parses it (engine/imagefiles.py, EXIF orientation applied); a file a GPU decoder takes has its compressed
    bytes staged in pinned memory and decoded on the reader's own stream, and the reader waits for its status word;
    any other file (or one the GPU decoder hands back) is decoded by PIL and uploaded on the same stream.  `get()` makes the
    device's current stream wait on the event recorded after the frame and returns the CUDA tensor [H,W,3]; it waits
    on the host only when the reader is behind and never synchronises the device.  Memory stays bounded by depth + 2
    frames whatever the length of the sequence.  `wait_s` is the time `get()` has spent waiting for the reader."""

    def __init__(self, paths: Sequence[str], device, depth: int = 4):
        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.paths = list(paths)
        nslots = depth + 2
        self._events = [torch.cuda.Event() for _ in range(nslots)]
        self._free: queue.Queue = queue.Queue()
        for s in range(nslots):
            self._free.put(s)
        self._ready: queue.Queue = queue.Queue()
        self._next = 0
        self.wait_s = 0.0
        self._stop = threading.Event()
        self._thread = threading.Thread(target=self._reader, name="m3r-frame-reader", daemon=True)
        self._thread.start()

    def _reader(self):
        from . import imagefiles
        try:
            torch.cuda.set_device(self.device)
            stream = torch.cuda.Stream(self.device)
            for path in self.paths:
                slot = self._free.get()
                if slot is None or self._stop.is_set():
                    return
                with torch.cuda.stream(stream):
                    out = imagefiles.decode_frame(path, self.device)
                    self._events[slot].record(stream)
                self._ready.put((slot, out))
        except BaseException as e:      # handed to the consumer, which raises it
            self._ready.put((None, e))

    def __len__(self):
        return len(self.paths)

    def get(self) -> torch.Tensor:
        if self._next >= len(self.paths):
            raise IndexError("no frame left")
        t = time.perf_counter()
        slot, out = self._ready.get()
        self.wait_s += time.perf_counter() - t
        if slot is None:
            raise RuntimeError(f"decoding {self.paths[self._next]} failed") from out
        self._next += 1
        consumer = torch.cuda.current_stream(self.device)
        consumer.wait_event(self._events[slot])
        out.record_stream(consumer)
        self._free.put(slot)
        return out

    def close(self):
        self._stop.set()
        self._free.put(None)
        self._thread.join()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
