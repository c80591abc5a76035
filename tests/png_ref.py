"""PNG test material: a small PNG writer that picks each row's filter, the zlib strategy and how IDAT is split, a
corpus built with it, hand-made malformed deflate streams, and a plain-Python statement of the CUDA decoder's
arithmetic (csrc/png.cu): inflate with zlib's checks in the kernel's order, Adler-32, unfilter and the RGB conversion,
with the same M3R_PNG_E* status bits."""
import io
import struct
import zlib

import numpy as np

# status bits (include/must3r_b200.h)
EBTYPE, ESTORED, ECODES, EREPEAT, ENOEOB, ESYMBOL, EDIST, ELENGTH, EFILTER, EPALETTE, EADLER = (1 << k for k in range(11))
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
SIG = b"\x89PNG\r\n\x1a\n"


def pillow(path, exif_transpose=False):
    import PIL.Image
    import PIL.ImageOps
    with PIL.Image.open(path) as im:
        if exif_transpose:
            im = PIL.ImageOps.exif_transpose(im)
        return np.asarray(im.convert("RGB"))


def content(H, W, kind, seed=0, channels=3):
    """uint8 [H,W,C]: 'smooth' gradients with a little texture, or uniform 'noisy' bytes."""
    rng = np.random.default_rng(seed)
    if kind == "noisy":
        return rng.integers(0, 256, (H, W, channels), dtype=np.uint8)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    planes = [128 + 100 * np.sin(x / (17 + 5 * c) + y / (23 + 3 * c) + seed) + rng.normal(0, 3, (H, W)) for c in range(channels)]
    return np.clip(np.stack(planes, -1), 0, 255).astype(np.uint8)


# ------------------------------------------------------------------------------------------- writer
def chunk(cid: bytes, data: bytes, crc=None) -> bytes:
    c = zlib.crc32(cid + data) if crc is None else crc
    return struct.pack(">I", len(data)) + cid + data + struct.pack(">I", c & 0xFFFFFFFF)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = abs(p - a), abs(p - b), abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(samples: np.ndarray, bpp: int, filters) -> bytes:
    """Scanlines of uint8 samples [H, W*bpp] (8-bit) with filter filters[y % len(filters)] on row y."""
    H, n = samples.shape
    out = bytearray()
    prev = np.zeros(n, np.int32)
    for y in range(H):
        row = samples[y].astype(np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), row[:-bpp]])
        ul = np.concatenate([np.zeros(bpp, np.int32), prev[:-bpp]])
        ft = filters[y % len(filters)]
        pred = [0, left, prev, (left + prev) >> 1, _paeth(left, prev, ul)][ft]
        out.append(ft)
        out += ((row - pred) & 255).astype(np.uint8).tobytes()
        prev = row
    return bytes(out)


def zstream(raw: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, stored=False) -> bytes:
    if stored:                                         # stored blocks of at most 65535 bytes
        out = bytearray(b"\x78\x01")
        for k in range(0, max(len(raw), 1), 65535):
            part = raw[k:k + 65535]
            out += bytes([1 if k + 65535 >= len(raw) else 0]) + struct.pack("<HH", len(part), 0xFFFF ^ len(part)) + part
        return bytes(out) + struct.pack(">I", zlib.adler32(raw))
    c = zlib.compressobj(level, zlib.DEFLATED, 15, 8, strategy)
    return c.compress(raw) + c.flush()


def png_bytes(samples: np.ndarray, color_type: int, *, filters=(0, 1, 2, 3, 4), level=6, strategy=zlib.Z_DEFAULT_STRATEGY,
              stored=False, palette=None, splits=(), before=(), after=(), bit_depth=8, interlace=0, stream=None) -> bytes:
    """A PNG of samples uint8 [H,W,C] (C = channels of the colour type; uint16 for bit_depth 16).  `splits`: byte
    offsets at which IDAT is cut (repeats give empty chunks); `before` / `after`: (type, data) chunks around IDAT;
    `stream`: a zlib stream used as is."""
    H, W = samples.shape[:2]
    C = CHANNELS[color_type]
    if stream is None:
        if interlace:
            raw = bytearray()
            for x0, y0, dx, dy in ((0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)):
                sub = samples[y0::dy, x0::dx]
                if sub.size:
                    raw += filter_rows(sub.reshape(sub.shape[0], -1), C, (0,))
            raw = bytes(raw)
        elif bit_depth == 16:
            be = samples.astype(">u2").view(np.uint8).reshape(H, W * C * 2)
            raw = filter_rows(be, 2 * C, filters)
        else:
            raw = filter_rows(samples.reshape(H, W * C), C, filters)
        stream = zstream(raw, level, strategy, stored)
    out = SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, bit_depth, color_type, 0, 0, interlace))
    for cid, data in before:
        out += chunk(cid, data)
    if palette is not None:
        out += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    cuts = [0] + sorted(splits) + [len(stream)]
    for a, b in zip(cuts[:-1], cuts[1:]):
        out += chunk(b"IDAT", stream[a:b])
    for cid, data in after:
        out += chunk(cid, data)
    return out + chunk(b"IEND", b"")


def exif_block(orientation=6) -> bytes:
    """A little-endian TIFF header with IFD0 holding one Orientation tag."""
    return b"II*\x00" + struct.pack("<IH", 8, 1) + struct.pack("<HHII", 0x0112, 3, 1, orientation) + b"\x00" * 4


def corpus():
    """[(name, bytes, eligible)]: every colour type, filters, zlib strategies and levels, split IDATs, ancillary chunks;
    ineligible: interlaced, 16-bit.  `eligible` is the GPU path's verdict without the EXIF transpose; the files
    with eXIf or text chunks are not eligible with it."""
    files = []
    rng = np.random.default_rng(7)
    shapes = [(1, 1), (7, 5), (33, 65), (48, 40)]
    strategies = [("z6", dict(level=6)), ("z0", dict(level=0)), ("z1", dict(level=1)), ("z9", dict(level=9)),
                  ("fixed", dict(strategy=zlib.Z_FIXED)), ("huff", dict(strategy=zlib.Z_HUFFMAN_ONLY)),
                  ("rle", dict(strategy=zlib.Z_RLE)), ("stored", dict(stored=True))]
    for ct in (0, 2, 3, 4, 6):
        for si, (H, W) in enumerate(shapes):
            for kind in ("smooth", "noisy"):
                C = CHANNELS[ct]
                if ct == 3:
                    n = [256, 17, 2, 200][si]
                    px = rng.integers(0, n, (H, W, 1), dtype=np.uint8) if kind == "noisy" else \
                        (content(H, W, "smooth", si, 1).astype(np.int32) * n // 256).astype(np.uint8)
                    extra = dict(palette=rng.integers(0, 256, (n, 3), dtype=np.uint8))
                else:
                    px, extra = content(H, W, kind, si, C), {}
                sname, sargs = strategies[(ct + 3 * si + (kind == "noisy")) % len(strategies)]
                filters = [(f,) for f in range(5)][(si + ct) % 5] if si % 2 else (0, 1, 2, 3, 4)
                files.append((f"ct{ct}_{H}x{W}_{kind}_{sname}", png_bytes(px, ct, filters=filters, **sargs, **extra), True))
    img = content(40, 56, "smooth", 3)
    files.append(("split_idat", png_bytes(img, 2, splits=(0, 0, 1, 2, 100, 100, 513)), True))
    files.append(("gama_iccp", png_bytes(img, 2, before=[(b"gAMA", struct.pack(">I", 45455)),
                                                        (b"iCCP", b"icc\x00\x00" + zlib.compress(b"\x00" * 128))]), True))
    files.append(("srgb_phys_time", png_bytes(img, 2, before=[(b"sRGB", b"\x00"), (b"pHYs", struct.pack(">IIB", 1, 1, 0))],
                                              after=[(b"tIME", b"\x07\xe8\x01\x01\x00\x00\x00")]), True))
    g = content(20, 30, "smooth", 4, 1)
    files.append(("trns_gray", png_bytes(g, 0, before=[(b"tRNS", b"\x00\x10")]), True))
    files.append(("trns_rgb", png_bytes(img, 2, before=[(b"tRNS", b"\x00\x10\x00\x20\x00\x30")]), True))
    pal = rng.integers(0, 256, (5, 3), dtype=np.uint8)
    files.append(("trns_palette", png_bytes(rng.integers(0, 5, (20, 30, 1), dtype=np.uint8), 3, palette=pal,
                                            before=[(b"tRNS", b"\x00\x80\xff")]), True))
    files.append(("exif_before", png_bytes(img, 2, before=[(b"eXIf", exif_block(6))]), True))
    files.append(("exif_after", png_bytes(img, 2, after=[(b"eXIf", exif_block(3))]), True))
    files.append(("text_before", png_bytes(img, 2, before=[(b"tEXt", b"Comment\x00hello")]), True))
    files.append(("text_after", png_bytes(img, 2, after=[(b"tEXt", b"Comment\x00after")]), True))
    files.append(("ztxt_after", png_bytes(img, 2, after=[(b"zTXt", b"Comment\x00\x00" + zlib.compress(b"x"))]), False))
    files.append(("interlaced", png_bytes(img, 2, interlace=1), False))
    files.append(("gray16", png_bytes(rng.integers(0, 65536, (12, 9, 1)).astype(np.uint16), 0, bit_depth=16), False))
    files.append(("rgb16", png_bytes(rng.integers(0, 65536, (12, 9, 3)).astype(np.uint16), 2, bit_depth=16), False))
    return files


def big_corpus():
    """Larger frames for the device tests: 1080p-class noise and smooth content, default and level 1."""
    return [("big_noise_rgb", png_bytes(content(270, 480, "noisy", 1), 2, level=1), True),
            ("big_smooth_rgba", png_bytes(content(300, 400, "smooth", 2, 4), 6), True),
            ("big_smooth_rgb_tall", png_bytes(content(517, 93, "smooth", 5), 2, filters=(4,)), True)]


def write(dirpath, files):
    out = []
    for name, data, eligible in files:
        p = dirpath / f"{name}.png"
        p.write_bytes(data)
        out.append((str(p), eligible))
    return out


# ------------------------------------------------------------------------------------------- deflate bit writer
class BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, v, n):                              # LSB first
        self.bits += [(v >> k) & 1 for k in range(n)]

    def code(self, c, n):                             # Huffman codes go MSB first
        self.bits += [(c >> (n - 1 - k)) & 1 for k in range(n)]

    def bytes(self):
        b = self.bits + [0] * (-len(self.bits) % 8)
        return bytes(sum(b[i + k] << k for k in range(8)) for i in range(0, len(b), 8))


def canonical(lens):
    """symbol -> (code, length) of the canonical code of `lens`."""
    count = [0] * 16
    for l in lens:
        if l:
            count[l] += 1
    first, code = [0] * 16, 0
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1 if l > 1 else 0
        first[l] = code
    nxt = first[:]
    out = {}
    for s, l in enumerate(lens):
        if l:
            out[s] = (nxt[l], l)
            nxt[l] += 1
    return out


FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
CLORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def zwrap(deflate: bytes, adler: int) -> bytes:
    return b"\x78\x01" + deflate + struct.pack(">I", adler)


def dynamic_header(w: BitWriter, hlit, hdist, cl_lens, seq):
    """Writes BTYPE 2's header: HLIT/HDIST/HCLEN, the code-length code and the (symbol, extra bits, extra value) seq."""
    hclen = max(k for k in range(19) if cl_lens[CLORDER[k]] or k < 4) + 1
    w.put(hlit - 257, 5)
    w.put(hdist - 1, 5)
    w.put(hclen - 4, 4)
    for k in range(hclen):
        w.put(cl_lens[CLORDER[k]], 3)
    codes = canonical(cl_lens)
    for s, nb, v in seq:
        w.code(*codes[s])
        if nb:
            w.put(v, nb)


def malformed():
    """{name: (zlib stream, raw length the image needs, predicted status bits)} for one image of 4x3 gray
    (raw = 3 * (1 + 4) = 15 bytes).  Each is an error class of the decoder."""
    H, W = 3, 4
    raw = bytes([0, 1, 2, 3, 4, 1, 5, 5, 5, 5, 2, 9, 9, 9, 9])
    n = len(raw)
    fl = canonical(FIXED_LIT)
    cases = {}

    def fixed(symbols, final=True):
        w = BitWriter()
        w.put(1 if final else 0, 1)
        w.put(1, 2)
        for s in symbols:
            if isinstance(s, tuple):                  # raw extra bits or distance code
                kind, a, b = s
                if kind == "bits":
                    w.put(a, b)
                else:
                    w.code(a, 5)
            else:
                w.code(*fl[s])
        return w

    w = BitWriter()
    w.put(1, 1)
    w.put(3, 2)
    cases["btype3"] = (zwrap(w.bytes(), zlib.adler32(raw)), n, EBTYPE)
    cases["stored_nlen"] = (b"\x78\x01" + b"\x01" + struct.pack("<HH", n, n) + raw + struct.pack(">I", zlib.adler32(raw)), n, ESTORED)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    w.put(287 - 257, 5)                                 # HLIT 287
    w.put(0, 5)
    w.put(0, 4)
    cases["too_many_lengths"] = (zwrap(w.bytes() + b"\x00" * 8, 1), n, ECODES)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    cl = [0] * 19
    cl[0] = cl[1] = cl[2] = 1                           # over-subscribed code-length code
    dynamic_header(w, 257, 1, cl, [])
    cases["oversubscribed"] = (zwrap(w.bytes() + b"\x00" * 8, 1), n, ECODES)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    cl = [0] * 19
    cl[0] = cl[16] = 1
    dynamic_header(w, 257, 1, cl, [(16, 2, 0)])         # a repeat with no previous length
    cases["repeat_first"] = (zwrap(w.bytes() + b"\x00" * 8, 1), n, EREPEAT)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    cl = [0] * 19
    cl[1], cl[17], cl[18] = 1, 2, 2
    seq = [(18, 7, 127), (18, 7, 127)]                  # 276 zeros: past HLIT + HDIST = 258
    dynamic_header(w, 257, 1, cl, seq)
    cases["repeat_past"] = (zwrap(w.bytes() + b"\x00" * 8, 1), n, EREPEAT)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    seq = [(18, 7, 65 - 11), (1, 0, 0), (1, 0, 0), (18, 7, 138 - 11), (18, 7, 257 - 67 - 138 - 11), (1, 0, 0)]
    dynamic_header(w, 257, 1, cl, seq)                  # literals 65, 66 and one distance code; no code for 256
    cases["no_eob"] = (zwrap(w.bytes() + b"\x00" * 8, 1), n, ENOEOB)
    w = BitWriter()
    w.put(1, 1)
    w.put(2, 2)
    cl = [0] * 19
    cl[1], cl[2], cl[18] = 2, 2, 1                      # incomplete literal/length code: 256 and 65 of length 2
    seq = [(18, 7, 65 - 11), (2, 0, 0), (18, 7, 138 - 11), (18, 7, 256 - 66 - 138 - 11), (2, 0, 0), (1, 0, 0)]
    dynamic_header(w, 257, 1, cl, seq)
    cases["incomplete_lit"] = (zwrap(w.bytes() + b"\x00" * 8, 1), n, ECODES)
    w = fixed([286])
    cases["lit_286"] = (zwrap(w.bytes(), 1), n, ESYMBOL)
    w = fixed([65, 257, ("dist", 30, 0)])
    cases["dist_30"] = (zwrap(w.bytes(), 1), n, ESYMBOL)
    w = fixed([257, ("dist", 0, 0)])                     # length 3, distance 1 with no output yet
    cases["dist_too_far"] = (zwrap(w.bytes(), 1), n, EDIST)
    short = zlib.compress(raw[:-3])
    cases["short"] = (short, n, ELENGTH)
    long = zlib.compress(raw + b"\x00" * 5)
    cases["long"] = (long, n, ELENGTH)
    bad = zlib.compress(raw)
    cases["adler"] = (bad[:-1] + bytes([bad[-1] ^ 1]), n, EADLER)
    bad_filter = bytearray(raw)
    bad_filter[5] = 7
    cases["filter_7"] = (zlib.compress(bytes(bad_filter)), n, EFILTER)
    cases["truncated"] = (zlib.compress(raw)[:-6], n, ELENGTH)
    return cases, (H, W)


# ------------------------------------------------------------------------------------------- statement of the kernels
class _Stop(Exception):
    pass


def _build(lens, codelen):
    """zlib's checks and a decoding map {(length, code): symbol}; raises _Stop(ECODES) as the kernel reports."""
    count = [0] * 16
    for l in lens:
        if l:
            count[l] += 1
    left, maxl = 1, 0
    for l in range(1, 16):
        left = (left << 1) - count[l]
        if left < 0:
            raise _Stop(ECODES)
        if count[l]:
            maxl = l
    if maxl == 0:
        if codelen:
            raise _Stop(ECODES)
        return {}
    if left > 0 and (codelen or maxl != 1):
        raise _Stop(ECODES)
    return {(l, c): s for s, (c, l) in canonical(lens).items()}


class _Bits:
    def __init__(self, data: bytes):
        self.d, self.n, self.p = data, len(data), 16       # bit position; the two header bytes are checked by the parser

    def get(self, k):
        v = 0
        for i in range(k):
            b = self.p + i
            bit = (self.d[b >> 3] >> (b & 7)) & 1 if (b >> 3) < self.n else 0
            v |= bit << i
        self.p += k
        return v

    def check(self):
        if self.p > 8 * self.n:
            raise _Stop(ELENGTH)

    def sym(self, table):
        code = 0
        for l in range(1, 16):
            b = self.p + l - 1
            code = (code << 1) | ((self.d[b >> 3] >> (b & 7)) & 1 if (b >> 3) < self.n else 0)
            if (l, code) in table:
                self.p += l
                return table[(l, code)]
        raise _Stop(ESYMBOL)


LBASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEXT = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DBASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
         8193, 12289, 16385, 24577]
DEXT = [0, 0, 0, 0] + [k // 2 for k in range(2, 28)]


def adler32(b: bytes) -> int:
    a, s = 1, 0
    for x in b:
        a = (a + x) % 65521
        s = (s + a) % 65521
    return (s << 16) | a


def inflate(stream: bytes, expect: int):
    """(output, status bits) as png_inflate_kernel computes them for a zlib stream whose image needs `expect` bytes.
    Symbols are written in the kernel's order: in runs of 32, the run's literals first, then its matches one after
    another, each copied from the output written so far."""
    out = bytearray(expect)
    pos = 0
    run = []

    def flush():
        for r in run:
            if r[0] == "L":
                out[r[1]] = r[2]
        for r in run:
            if r[0] == "M":
                _, p, ln, d = r
                for i in range(ln):
                    out[p + i] = out[p - d + (i if d >= ln else i % d)]
        run.clear()

    bits = _Bits(stream)
    err = 0
    try:
        last = 0
        while not last:
            last = bits.get(1)
            btype = bits.get(2)
            bits.check()
            if btype == 3:
                raise _Stop(EBTYPE)
            if btype == 0:
                bp = (bits.p + 7) >> 3
                if bp + 4 > bits.n:
                    raise _Stop(ELENGTH)
                ln, nln = struct.unpack("<HH", stream[bp:bp + 4])
                if ln != (~nln & 0xFFFF):
                    raise _Stop(ESTORED)
                if bp + 4 + ln > bits.n or pos + ln > expect:
                    raise _Stop(ELENGTH)
                out[pos:pos + ln] = stream[bp + 4:bp + 4 + ln]
                pos += ln
                bits.p = 8 * (bp + 4 + ln)
                continue
            if btype == 1:
                lit, dist = _build(FIXED_LIT, False), _build([5] * 32, False)
            else:
                hlit, hdist, hclen = bits.get(5) + 257, bits.get(5) + 1, bits.get(4) + 4
                bits.check()
                if hlit > 286 or hdist > 30:
                    raise _Stop(ECODES)
                cl = [0] * 19
                for k in range(hclen):
                    cl[CLORDER[k]] = bits.get(3)
                bits.check()
                clt = _build(cl, True)
                lens = []
                while len(lens) < hlit + hdist:
                    s = bits.sym(clt)
                    bits.check()
                    if s < 16:
                        lens.append(s)
                        continue
                    if s == 16:
                        if not lens:
                            raise _Stop(EREPEAT)
                        val, rep = lens[-1], 3 + bits.get(2)
                    elif s == 17:
                        val, rep = 0, 3 + bits.get(3)
                    else:
                        val, rep = 0, 11 + bits.get(7)
                    bits.check()
                    if len(lens) + rep > hlit + hdist:
                        raise _Stop(EREPEAT)
                    lens += [val] * rep
                if lens[256] == 0:
                    raise _Stop(ENOEOB)
                lit = _build(lens[:hlit], False)
                dist = _build(lens[hlit:], False)
            while True:
                s = bits.sym(lit)
                bits.check()
                if s < 256:
                    if pos >= expect:
                        raise _Stop(ELENGTH)
                    run.append(("L", pos, s))
                    pos += 1
                    if len(run) == 32:
                        flush()
                    continue
                if s == 256:
                    flush()
                    break
                if s > 285:
                    raise _Stop(ESYMBOL)
                ln = LBASE[s - 257] + bits.get(LEXT[s - 257])
                ds = bits.sym(dist)
                bits.check()
                if ds > 29:
                    raise _Stop(ESYMBOL)
                d = DBASE[ds] + bits.get(DEXT[ds])
                bits.check()
                if d > pos:
                    raise _Stop(EDIST)
                if pos + ln > expect:
                    raise _Stop(ELENGTH)
                run.append(("M", pos, ln, d))
                pos += ln
                if len(run) == 32:
                    flush()
        bp = (bits.p + 7) >> 3
        if bp + 4 > bits.n:
            raise _Stop(ELENGTH)
        if pos != expect:
            err |= ELENGTH
        if adler32(bytes(out[:pos])) != struct.unpack(">I", stream[bp:bp + 4])[0]:
            err |= EADLER
    except _Stop as e:
        flush()
        err |= e.args[0]
    return bytes(out[:pos]), err


def unfilter(raw: bytes, H: int, W: int, bpp: int):
    """(samples uint8 [H, W*bpp], status bits) as png_unfilter_kernel computes them."""
    stride = 1 + W * bpp
    fts = [raw[y * stride] for y in range(H)]
    if any(f > 4 for f in fts):
        return None, EFILTER
    out = np.zeros((H, W * bpp), np.int32)
    prev = np.zeros(W * bpp, np.int32)
    for y in range(H):
        f = np.frombuffer(raw, np.uint8, W * bpp, y * stride + 1).astype(np.int32)
        ft = fts[y]
        row = np.zeros(W * bpp, np.int32)
        if ft in (0, 2):
            row = (f + (prev if ft == 2 else 0)) & 255
        else:
            for i in range(W * bpp):                       # the chains along the row
                a = row[i - bpp] if i >= bpp else 0
                b = prev[i]
                c = prev[i - bpp] if i >= bpp else 0
                pred = a if ft == 1 else (a + b) >> 1 if ft == 3 else int(_paeth(a, b, c))
                row[i] = (f[i] + pred) & 255
        out[y] = row
        prev = row
    return out.astype(np.uint8), 0


def decode(data: bytes):
    """(RGB uint8 [H,W,3] or None, status bits) of an eligible PNG file, as the device path computes them."""
    pos, plte, idat = 8, None, b""
    while pos < len(data):
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        cid, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        if cid == b"IHDR":
            W, H, _, ct = struct.unpack(">IIBB", body[:10])
        elif cid == b"PLTE":
            plte = np.frombuffer(body, np.uint8).reshape(-1, 3)
        elif cid == b"IDAT":
            idat += body
        pos += 12 + n
    bpp = CHANNELS[ct]
    raw, err = inflate(idat, H * (1 + W * bpp))
    if err:
        return None, err
    s, err = unfilter(raw, H, W, bpp)
    if err:
        return None, err
    s = s.reshape(H, W, bpp)
    if ct == 3:
        idx = s[..., 0]
        if (idx >= len(plte)).any():
            return None, EPALETTE
        return plte[idx], 0
    if ct in (0, 4):
        return np.repeat(s[..., :1], 3, -1), 0
    return s[..., :3].copy(), 0


def _length_symbol(n):
    k = max(i for i in range(29) if LBASE[i] <= n)
    return 257 + k, LEXT[k], n - LBASE[k]


def far_matches():
    """{name: PNG bytes}: valid gray images whose streams copy from the far end of deflate's 32K window: stored bytes,
    then a fixed block of (length, distance) matches and literals.  In each, a literal lands 32768 bytes past a byte
    that a match before it in the same run of 32 symbols reads, or one match reads and writes 32768 - k bytes apart
    for k < 32."""
    specs = {                                   # stored bytes, symbols (int: literal, tuple: match), row stride
        "far_then_literal": (32400, [(10, 32400), (258, 1), (100, 1), 3], 331),
        "far_within_match": (32768, [(258, 32763)], 337),
        "full_window": (32768, [(258, 32768), 2], 109),
    }
    rng = np.random.default_rng(11)
    files = {}
    for name, (n, syms, stride) in specs.items():
        stored = bytearray(rng.integers(0, 256, n, dtype=np.uint8).tobytes())
        for _ in range(8):                      # make every row's filter byte 0..4, tracing copies to their source
            ops, p = [], n
            for s in syms:
                ops.append((p, s))
                p += s[0] if isinstance(s, tuple) else 1
            total = p
            out = bytearray(stored) + bytearray(total - n)
            for q, s in ops:
                if isinstance(s, tuple):
                    ln, d = s
                    for i in range(ln):
                        out[q + i] = out[q - d + (i if d >= ln else i % d)]
                else:
                    out[q] = s
            bad = [q for q in range(0, total, stride) if out[q] > 4]
            if not bad:
                break
            for q in bad:
                while q >= n:
                    qp, s = max((o for o in ops if o[0] <= q), key=lambda o: o[0])
                    ln, d = s
                    i = q - qp
                    q = qp - d + (i if d >= ln else i % d)
                stored[q] = int(rng.integers(0, 5))
        assert total % stride == 0 and not bad
        w = BitWriter()
        w.put(1, 1)
        w.put(1, 2)
        fl = canonical(FIXED_LIT)
        for s in syms:
            if isinstance(s, tuple):
                ls, nb, v = _length_symbol(s[0])
                w.code(*fl[ls])
                w.put(v, nb)
                k = max(i for i in range(30) if DBASE[i] <= s[1])
                w.code(k, 5)
                w.put(s[1] - DBASE[k], DEXT[k])
            else:
                w.code(*fl[s])
        w.code(*fl[256])
        stream = b"\x78\x01" + b"\x00" + struct.pack("<HH", n, 0xFFFF ^ n) + bytes(stored) + w.bytes() + \
            struct.pack(">I", zlib.adler32(bytes(out)))
        files[name] = with_stream(stream, total // stride, stride - 1)
    return files


def with_stream(stream: bytes, H: int, W: int, color_type=0, palette=None) -> bytes:
    """A PNG file around a given zlib stream."""
    return png_bytes(np.zeros((H, W, CHANNELS[color_type]), np.uint8), color_type, stream=stream, palette=palette)


def pillow_bytes(data: bytes) -> np.ndarray:
    import PIL.Image
    return np.asarray(PIL.Image.open(io.BytesIO(data)).convert("RGB"))
