"""A corpus of JPEG (and other) files generated at test time with Pillow, for the JPEG decoder's tests.

Each entry is (name, bytes, eligible): `eligible` says whether the GPU decoder is meant to take the file.  The corpus
covers the sizes, samplings, qualities, restart intervals, orientations and ineligible kinds the decoder must handle.
"""
from __future__ import annotations

import io
import struct

import numpy as np

SIZES = [(1, 1), (1, 17), (8, 8), (9, 15), (16, 16), (17, 31), (33, 65), (480, 640), (640, 480)]   # (H, W)
SUBSAMPLING = {"444": 0, "422": 1, "420": 2}


def content(H, W, kind, seed=0):
    """smooth: gradients and a disc; noisy: uniform noise (reaches the IDCT's range limit at quality 100)."""
    rng = np.random.default_rng(seed + H * 1000 + W)
    if kind == "noisy":
        return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    r = 127 + 120 * np.sin(x / max(W, 1) * 6.0) * np.cos(y / max(H, 1) * 4.0)
    g = 255 * x / max(W - 1, 1)
    b = np.where((x - W / 2) ** 2 + (y - H / 2) ** 2 < (min(H, W) / 3) ** 2, 230.0, 20.0)
    return np.clip(np.stack([r, g, b], -1) + rng.normal(0, 3, (H, W, 3)), 0, 255).astype(np.uint8)


def exif_orientation(o: int, little: bool) -> bytes:
    """A minimal EXIF block (TIFF header, IFD0 with one SHORT Orientation entry) in either byte order."""
    e = "<" if little else ">"
    tiff = (b"II" if little else b"MM") + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1)
    tiff += struct.pack(e + "HHI", 0x0112, 3, 1) + struct.pack(e + "HH", o, 0) + struct.pack(e + "I", 0)
    return b"Exif\x00\x00" + tiff


def save(arr, **kw) -> bytes:
    import PIL.Image
    buf = io.BytesIO()
    mode = "L" if arr.ndim == 2 else "RGB"
    PIL.Image.fromarray(arr, mode).save(buf, **kw)
    return buf.getvalue()


def corpus(big: bool = False):
    """[(name, bytes, eligible)]; `big` adds a 1080x1920 frame."""
    out = []
    sizes = SIZES + ([(1080, 1920)] if big else [])
    for H, W in sizes:
        for kind in ("smooth", "noisy"):
            img = content(H, W, kind)
            for ss, sv in SUBSAMPLING.items():
                for q in (1, 50, 90, 100):
                    if H * W > 20000 and q in (1, 50):
                        continue
                    out.append((f"{H}x{W}_{kind}_{ss}_q{q}", save(img, format="JPEG", quality=q, subsampling=sv), True))
            out.append((f"{H}x{W}_{kind}_gray_q90", save(img[..., 1], format="JPEG", quality=90), True))
    img = content(33, 65, "smooth")
    out.append(("opt_420", save(img, format="JPEG", quality=85, optimize=True), True))
    out.append(("opt_444", save(img, format="JPEG", quality=85, subsampling=0, optimize=True), True))
    for ss, sv in SUBSAMPLING.items():
        out.append((f"rst_blocks1_{ss}", save(img, format="JPEG", quality=90, subsampling=sv, restart_marker_blocks=1), True))
        out.append((f"rst_blocks4_{ss}", save(img, format="JPEG", quality=90, subsampling=sv, restart_marker_blocks=4), True))
        out.append((f"rst_rows1_{ss}", save(img, format="JPEG", quality=90, subsampling=sv, restart_marker_rows=1), True))
    out.append(("rst_rows1_gray", save(img[..., 0], format="JPEG", quality=90, restart_marker_rows=1), True))
    big_rst = content(480, 640, "smooth")
    out.append(("rst_rows1_480x640", save(big_rst, format="JPEG", quality=95, restart_marker_rows=1), True))
    img = content(17, 31, "smooth")
    for o in range(1, 9):
        for little in (True, False):
            out.append((f"exif{o}_{'le' if little else 'be'}",
                        save(img, format="JPEG", quality=90, exif=exif_orientation(o, little)), True))
    out.append(("exif9", save(img, format="JPEG", quality=90, exif=exif_orientation(9, True)), True))
    xmp = b'<x:xmpmeta xmlns:x="adobe:ns:meta/"><rdf:Description tiff:Orientation="6"/></x:xmpmeta>'
    out.append(("xmp6", save(img, format="JPEG", quality=90, xmp=xmp), True))
    out.append(("progressive", save(img, format="JPEG", quality=90, progressive=True), False))
    import PIL.Image
    buf = io.BytesIO()
    PIL.Image.fromarray(img, "RGB").convert("CMYK").save(buf, format="JPEG", quality=90)
    out.append(("cmyk", buf.getvalue(), False))
    out.append(("keep_rgb", save(img, format="JPEG", quality=90, keep_rgb=True, subsampling=0), False))
    out.append(("png", save(img, format="PNG"), False))
    return out


def write(tmpdir, entries):
    """Write the entries as files (.jpg, or .png for the PNG); returns [(path, eligible)]."""
    import os
    paths = []
    for name, data, eligible in entries:
        p = os.path.join(str(tmpdir), name + (".png" if name == "png" else ".jpg"))
        with open(p, "wb") as f:
            f.write(data)
        paths.append((p, eligible))
    return paths


def pillow(path, exif_transpose: bool) -> np.ndarray:
    import PIL.Image
    import PIL.ImageOps
    with PIL.Image.open(path) as im:
        if exif_transpose:
            im = PIL.ImageOps.exif_transpose(im)
        return np.asarray(im.convert("RGB"))


# ============================================================================ plain-numpy sequential decoder
# The CPU statement of what csrc/jpeg.cu computes: libjpeg-turbo's baseline Huffman decoding, DC prediction,
# jidctint.c's ISLOW IDCT, jdsample.c's fancy upsampling, jdcolor.c's YCbCr->RGB and Pillow's exif_transpose.  The
# decoder state (bit offset, block within the MCU, zig-zag index) and its error bits are the kernels'.
EHUFF, ESHORT = 1, 2
NATURAL = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
           21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
           60, 61, 54, 47, 55, 62, 63]


def _huff(bits, vals):
    """{(length, code): symbol} of a canonical table."""
    t, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            t[(length, code)] = vals[k]
            code, k = code + 1, k + 1
        code <<= 1
    return t


def unstuff(data: bytes, start: int):
    """Entropy-coded bytes with FF 00 -> FF and the restart markers dropped, and each segment's first bit."""
    out, segs, i = bytearray(), [0], start
    while i < len(data):
        b = data[i]
        if b != 0xFF:
            out.append(b)
            i += 1
            continue
        j = i + 1
        while data[j] == 0xFF:
            j += 1
        m, i = data[j], j + 1
        if m == 0:
            out.append(0xFF)
        elif 0xD0 <= m <= 0xD7:
            segs.append(8 * len(out))
        else:
            break
    return bytes(out), segs


class Jpeg:
    """Headers of an eligible baseline JPEG (one interleaved scan in frame order), its entropy-coded stream as bits and
    the restart segments [start, end) in bits."""

    def __init__(self, data: bytes):
        qt, dc, ac, self.ri, i = {}, {}, {}, 0, 2
        while True:
            while data[i] == 0xFF:
                i += 1
            m = data[i]
            n = int.from_bytes(data[i + 1:i + 3], "big")
            p = data[i + 3:i + 1 + n]
            i += 1 + n
            if m == 0xDB:
                o = 0
                while o < len(p):
                    pq, tq = p[o] >> 4, p[o] & 15
                    w = 2 if pq else 1
                    v = [int.from_bytes(p[o + 1 + w * k:o + 1 + w * k + w], "big") for k in range(64)]
                    q = np.zeros(64, np.int64)
                    q[NATURAL] = v
                    qt[tq] = q
                    o += 1 + 64 * w
            elif m == 0xC4:
                o = 0
                while o < len(p):
                    tc, th = p[o] >> 4, p[o] & 15
                    bits = list(p[o + 1:o + 17])
                    vals = list(p[o + 17:o + 17 + sum(bits)])
                    (ac if tc else dc)[th] = _huff(bits, vals)
                    o += 17 + sum(bits)
            elif m == 0xDD:
                self.ri = int.from_bytes(p[:2], "big")
            elif m in (0xC0, 0xC1):
                self.H, self.W, nc = int.from_bytes(p[1:3], "big"), int.from_bytes(p[3:5], "big"), p[5]
                self.comps = [(p[7 + 3 * c] >> 4, p[7 + 3 * c] & 15, p[8 + 3 * c]) for c in range(nc)]
            elif m == 0xDA:
                ns = p[0]
                self.tabs = [(dc[p[2 + 2 * c] >> 4], ac[p[2 + 2 * c] & 15]) for c in range(ns)]
                break
        nc = len(self.comps)
        if nc == 1:
            self.comps = [(1, 1, self.comps[0][2])]
        self.hs = [c[0] for c in self.comps]
        self.vs = [c[1] for c in self.comps]
        self.qt = [qt[c[2]] for c in self.comps]
        self.blk_comp = [c for c in range(nc) for _ in range(self.hs[c] * self.vs[c])]
        self.bpm = len(self.blk_comp)
        self.mcux = -(-self.W // (8 * self.hs[0]))
        self.mcuy = -(-self.H // (8 * self.vs[0]))
        stream, starts = unstuff(data, i)
        self.bits = np.concatenate([np.unpackbits(np.frombuffer(stream, np.uint8)), np.zeros(64, np.uint8)])
        self.segs = list(zip(starts, starts[1:] + [8 * len(stream)]))
        self.seg_blocks = (self.ri if self.ri else self.mcux * self.mcuy) * self.bpm

    def _get(self, p, n):
        v = 0
        for b in self.bits[p:p + n]:
            v = (v << 1) | int(b)
        return v

    def _symbol(self, table, p):
        for length in range(1, 17):
            s = table.get((length, self._get(p, length)))
            if s is not None:
                return length, s
        return 0, -1

    def step(self, st):
        """One symbol from state (p, c, z): (new state, (zig-zag index, value) or None, error bit, block completed)."""
        p, c, z = st
        comp = self.blk_comp[c]
        dct, act = self.tabs[comp]
        write, bad = None, 0
        if z == 0:
            length, s = self._symbol(dct, p)
            if length == 0 or s > 11:
                bad, p, z = 1, p + (length or 1), 64
            else:
                v = self._get(p + length, s)
                write = (0, _extend(v, s))
                p, z = p + length + s, 1
        else:
            length, s = self._symbol(act, p)
            if length == 0:
                bad, p, z = 1, p + 1, 64
            else:
                r, sz = s >> 4, s & 15
                if sz == 0:
                    z = min(z + 16, 64) if r == 15 else 64
                    p += length
                elif sz > 10 or z + r > 63:
                    bad, p, z = 1, p + length + sz, 64
                else:
                    z += r
                    write = (z, _extend(self._get(p + length, sz), sz))
                    p, z = p + length + sz, z + 1
        done = z >= 64
        if done:
            z, c = 0, (c + 1) % self.bpm
        return (p, c, z), write, bad, done

    def run(self, st, end):
        """Decode symbols while the bit offset is below `end` (a subsequence): (exit state, blocks completed)."""
        n = 0
        while st[0] < end:
            st, _, _, done = self.step(st)
            n += done
        return st, n

    def trace(self, seg):
        """Every symbol-boundary state of a segment decoded from its start until the offset reaches its end, and the
        blocks completed before each."""
        a, b = self.segs[seg]
        st, n, out = (a, 0, 0), 0, [((a, 0, 0), 0)]
        while st[0] < b:
            st, _, _, done = self.step(st)
            n += done
            out.append((st, n))
        return out

    def coefficients(self):
        """int16 [blocks, 64] in natural order with DC values, and the error bits of the kernels' status word."""
        total = self.mcux * self.mcuy * self.bpm
        coef = np.zeros((total, 64), np.int64)
        err = 0
        for s, (a, b) in enumerate(self.segs):
            blk, end = s * self.seg_blocks, min(total, (s + 1) * self.seg_blocks)
            st = (a, 0, 0)
            while blk < end:
                if st[0] >= b:
                    err |= ESHORT
                    break
                st, write, bad, done = self.step(st)
                if write is not None:
                    coef[blk, NATURAL[write[0]]] = write[1]
                err |= bad * EHUFF | (ESHORT if st[0] > b else 0)
                blk += done
        for comp in range(len(self.comps)):           # DC prediction, restarting at every segment
            pred, seg = 0, 0
            for k in range(total):
                if self.blk_comp[k % self.bpm] != comp:
                    continue
                if k // self.seg_blocks != seg:
                    pred, seg = 0, k // self.seg_blocks
                pred += int(coef[k, 0])
                coef[k, 0] = pred
        return coef.astype(np.int16), err


def _extend(v, s):
    return 0 if s == 0 else (v - (1 << s) + 1 if v < (1 << (s - 1)) else v)


def _idct_pass(x, shift):
    """One 8-point jpeg_idct_islow pass along the last axis (int64 = JLONG), DESCALE by `shift`."""
    f = {k: v for k, v in dict(a=2446, b=3196, c=4433, d=6270, e=7373, f=9633, g=12299, h=15137, i=16069, j=16819,
                                k=20995, l=25172).items()}
    z2, z3 = x[..., 2], x[..., 6]
    z1 = (z2 + z3) * f["c"]
    tmp2, tmp3 = z1 - z3 * f["h"], z1 + z2 * f["d"]
    tmp0, tmp1 = (x[..., 0] + x[..., 4]) * 8192, (x[..., 0] - x[..., 4]) * 8192
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * f["f"]
    t0, t1, t2, t3 = t0 * f["a"], t1 * f["j"], t2 * f["l"], t3 * f["g"]
    z1, z2, z3, z4 = -z1 * f["e"], -z2 * f["k"], -z3 * f["i"] + z5, -z4 * f["b"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    r = 1 << (shift - 1)
    out = [t10 + t3, t11 + t2, t12 + t1, t13 + t0, t13 - t0, t12 - t1, t11 - t2, t10 - t3]
    return np.stack([(o + r) >> shift for o in out], -1)


def idct_islow(coef, q):
    """[N, 64] int16 coefficients, natural order, and the [64] table -> [N, 8, 8] uint8 (range_limit & RANGE_MASK)."""
    x = (coef.astype(np.int64) * q).reshape(-1, 8, 8)
    ws = _idct_pass(x.transpose(0, 2, 1), 11).transpose(0, 2, 1).astype(np.int32).astype(np.int64)   # columns
    o = _idct_pass(ws, 18)                                                                            # rows
    v = ((o & 1023) ^ 512) - 512
    return np.clip(v + 128, 0, 255).astype(np.uint8)


def _upsample(plane, dw, dh, h2, v2, H, W):
    """jdsample.c for one chroma plane [rows, cols] at the downsampled size (dh, dw) -> [H, W] int."""
    c = plane[:dh, :dw].astype(np.int64)
    if not h2 and not v2:
        return c[:H, :W]
    if h2 and dw <= 2:                                  # box
        c = np.repeat(c, 2, 1)
        if v2:
            c = np.repeat(c, 2, 0)
        return c[:H, :W]
    if v2:                                              # rows: 3 * nearest + next nearest
        up, dn = c[np.maximum(np.arange(dh) - 1, 0)], c[np.minimum(np.arange(dh) + 1, dh - 1)]
        rows = np.empty((2 * dh, dw), np.int64)
        rows[0::2], rows[1::2] = 3 * c + up, 3 * c + dn
        if not h2:                                      # h1v2
            rows[0::2] += 1
            rows[1::2] += 2
            return (rows >> 2)[:H, :W]
        c = rows
    left, right = c[:, np.maximum(np.arange(dw) - 1, 0)], c[:, np.minimum(np.arange(dw) + 1, dw - 1)]
    out = np.empty((c.shape[0], 2 * dw), np.int64)
    if v2:                                              # h2v2 on the column sums
        out[:, 0::2], out[:, 1::2] = (3 * c + left + 8) >> 4, (3 * c + right + 7) >> 4
    else:                                               # h2v1
        out[:, 0::2], out[:, 1::2] = (3 * c + left + 1) >> 2, (3 * c + right + 2) >> 2
    return out[:H, :W]


def transpose(img, orientation):
    """Pillow's exif_transpose methods for orientations 2..8."""
    return {2: lambda a: a[:, ::-1], 3: lambda a: a[::-1, ::-1], 4: lambda a: a[::-1], 5: lambda a: a.transpose(1, 0, 2),
            6: lambda a: np.rot90(a, -1), 7: lambda a: a.transpose(1, 0, 2)[::-1, ::-1], 8: lambda a: np.rot90(a, 1)}.get(
        orientation, lambda a: a)(img)


def decode(data: bytes, orientation: int = 1):
    """RGB uint8 [H, W, 3] of an eligible baseline JPEG, and the kernels' error bits."""
    j = Jpeg(data)
    coef, err = j.coefficients()
    planes = []
    for comp in range(len(j.comps)):
        h, v = j.hs[comp], j.vs[comp]
        k = [b for b in range(coef.shape[0]) if j.blk_comp[b % j.bpm] == comp]
        px = idct_islow(coef[k], j.qt[comp]).reshape(j.mcuy, j.mcux, v, h, 8, 8)
        planes.append(px.transpose(0, 2, 4, 1, 3, 5).reshape(j.mcuy * v * 8, j.mcux * h * 8))
    Y = planes[0][:j.H, :j.W].astype(np.int64)
    if len(planes) == 1:
        rgb = np.stack([Y, Y, Y], -1)
    else:
        h2, v2 = j.hs[0] == 2, j.vs[0] == 2
        dw, dh = -(-j.W // j.hs[0]), -(-j.H // j.vs[0])
        cb = _upsample(planes[1], dw, dh, h2, v2, j.H, j.W) - 128
        cr = _upsample(planes[2], dw, dh, h2, v2, j.H, j.W) - 128
        r = Y + ((91881 * cr + 32768) >> 16)
        g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16)
        b = Y + ((116130 * cb + 32768) >> 16)
        rgb = np.stack([r, g, b], -1)
    return np.ascontiguousarray(transpose(np.clip(rgb, 0, 255).astype(np.uint8), orientation)), err


def partition(j: Jpeg, seg: int, sub_bits: int, max_rounds: int = 100000):
    """Model of the self-synchronising partition of one segment: subsequences of `sub_bits`, a speculative pass from
    assumed states (the first one's is known), then rounds in which each subsequence whose entry differs from its
    predecessor's exit is decoded again from that exit, until no entry changes.  Returns ([entry states], [blocks
    completed per subsequence], rounds)."""
    a, b = j.segs[seg]
    subs = [(s, min(s + sub_bits, b)) for s in range(a, b, sub_bits)]
    entry = [(s, 0, 0) for s, _ in subs]
    res = [j.run(e, end) for e, (_, end) in zip(entry, subs)]
    rounds = 0
    while rounds < max_rounds:
        new = [entry[0]] + [res[g - 1][0] for g in range(1, len(subs))]
        changed = [g for g in range(len(subs)) if new[g] != entry[g]]
        if not changed:
            break
        rounds += 1
        for g in changed:
            entry[g] = new[g]
            res[g] = j.run(entry[g], subs[g][1])
    return entry, [n for _, n in res], rounds


def all_ones_dc_code(data: bytes) -> bytes:
    """`data` with one more length-9 symbol in its first DC table: the last length-9 code becomes all ones, which libjpeg
    rejects (JERR_BAD_HUFF_TABLE) although no code the stream uses changes."""
    i = 2
    while True:
        m, n = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        if m == 0xC4 and data[i + 4] == 0x00:
            bits = bytearray(data[i + 5:i + 21])
            assert bits[8] >= 1 and not any(bits[9:])
            nv = sum(bits)
            bits[8] += 1
            seg = b"\x00" + bytes(bits) + data[i + 21:i + 21 + nv] + bytes([0x0B]) + data[i + 21 + nv:i + 2 + n]
            return data[:i] + b"\xff\xc4" + (len(seg) + 2).to_bytes(2, "big") + seg + data[i + 2 + n:]
        i += 2 + n
