"""PNG decoding without a GPU: the chunk parser against Pillow (size, mode, eligibility), the plain-Python statement of
the CUDA decoder (tests/png_ref.py) against Pillow bit for bit, the malformed streams against zlib and Pillow, and the
C struct layouts."""
import ctypes as C
import io
import os
import subprocess
import zlib

import numpy as np
import pytest

import png_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from must3r_b200 import _lib
    return _lib.lib()


def _open(data):
    import PIL.Image
    return PIL.Image.open(io.BytesIO(data))


def test_parser_agrees_with_pillow(lib, tmp_path):
    from must3r_b200 import ops
    from must3r_b200.engine import imagefiles, png
    for (name, data, eligible), (p, _) in zip(pr.corpus(), pr.write(tmp_path, pr.corpus())):
        info = ops.png_parse(data)
        im = _open(data)
        assert (info.width, info.height) == im.size, name
        assert bool(info.eligible) == eligible, name
        if eligible:
            assert png.MODES[info.color_type] == im.mode, name
        for t in (False, True):
            item = imagefiles.parse(p, t)
            assert isinstance(item, png.Parsed), name
            metadata = info.has_exif or info.has_text
            assert item.gpu == (eligible and not (t and metadata)), (name, t)
    assert not ops.png_parse(b"not a png at all").eligible


def test_exif_and_text_chunks_are_seen_before_and_after_the_image_data(lib):
    from must3r_b200 import ops
    files = dict((n, d) for n, d, _ in pr.corpus())
    for n in ("exif_before", "exif_after"):
        assert ops.png_parse(files[n]).has_exif, n
    for n in ("text_before", "text_after"):
        assert ops.png_parse(files[n]).has_text, n


def test_chunk_rules(lib):
    """A bad CRC before the image data, a second IDAT run, a missing IEND, a bad zlib header and Pillow's pixel limit
    keep a file off the GPU."""
    import PIL.Image
    from must3r_b200 import ops
    from must3r_b200.engine import png
    img = pr.content(9, 11, "smooth")
    good = pr.png_bytes(img, 2)
    assert ops.png_parse(good).eligible
    k = good.index(b"IHDR")
    bad_crc = bytearray(good)
    bad_crc[k + 4 + 13] ^= 1
    assert not ops.png_parse(bytes(bad_crc)).eligible
    with pytest.raises(Exception):                              # Pillow: no plugin identifies it
        _open(bytes(bad_crc))
    k = good.index(b"IDAT") - 4
    n = int.from_bytes(good[k:k + 4], "big")
    idat = good[k:k + 12 + n]
    twice = good[:k + 12 + n] + pr.chunk(b"tEXt", b"a\x00b") + idat + good[k + 12 + n:]
    assert not ops.png_parse(twice).eligible
    assert not ops.png_parse(good[:-12]).eligible                 # no IEND
    s = bytearray(pr.zstream(pr.filter_rows(img.reshape(9, -1), 3, (0,))))
    s[1] |= 0x20                                                  # FDICT
    s[1] = (s[1] & 0xE0) | (31 - ((s[0] << 8) | (s[1] & 0xE0)) % 31) % 31
    assert not ops.png_parse(pr.png_bytes(img, 2, stream=bytes(s))).eligible
    bad_idat_crc = bytearray(good)                                # Pillow ignores an IDAT CRC
    bad_idat_crc[k + 8 + n] ^= 1
    assert ops.png_parse(bytes(bad_idat_crc)).eligible
    old = PIL.Image.MAX_IMAGE_PIXELS
    try:
        PIL.Image.MAX_IMAGE_PIXELS = 9 * 11 - 1
        assert not png.Parsed("x.png", False, good).gpu
        PIL.Image.MAX_IMAGE_PIXELS = 9 * 11
        assert png.Parsed("x.png", False, good).gpu
    finally:
        PIL.Image.MAX_IMAGE_PIXELS = old


def test_statement_equals_pillow(lib):
    for name, data, eligible in pr.corpus():
        if not eligible:
            continue
        got, err = pr.decode(data)
        assert err == 0, name
        np.testing.assert_array_equal(got, pr.pillow_bytes(data), err_msg=name)


def test_malformed_classes_are_rejected(lib):
    """Every malformed stream is rejected by zlib or Pillow and by the statement with the predicted bits; the one Pillow
    accepts (output longer than the image) is only handed back to Pillow by the GPU path."""
    from must3r_b200 import ops
    cases, (H, W) = pr.malformed()
    for name, (stream, n, bits) in cases.items():
        data = pr.with_stream(stream, H, W)
        assert ops.png_parse(data).eligible, name
        _, err = pr.decode(data)
        assert err == bits, (name, err, bits)
        try:
            zlib.decompress(stream)
            zlib_ok = True
        except zlib.error:
            zlib_ok = False
        try:
            pr.pillow_bytes(data)
            pillow_ok = True
        except OSError:
            pillow_ok = False
        if name == "long":
            assert zlib_ok and pillow_ok
        else:
            assert not (zlib_ok and pillow_ok), name
    pal = np.array([[1, 2, 3], [4, 5, 6]], np.uint8)
    px = np.array([[[0], [1], [3]]], np.uint8)
    _, err = pr.decode(pr.png_bytes(px, 3, palette=pal))
    assert err == pr.EPALETTE


def test_structs_match_the_c_layout(lib, tmp_path):
    from must3r_b200 import _lib
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "must3r_b200.h"\nint main(){printf("%zu %zu\\n",'
                    'sizeof(m3r_png_info),sizeof(m3r_png_desc));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_lib.PngInfo), C.sizeof(_lib.PngDesc)]


def test_far_matches_are_valid_and_decoded(lib):
    """Streams that copy from the far end of the 32K window (a literal 32768 bytes past a byte an earlier match of its
    run reads; a match whose source and destination are 32768 - k bytes apart): zlib and Pillow accept them, and the
    statement, which writes each run of 32 symbols in the kernel's order, decodes them to Pillow's pixels."""
    from must3r_b200 import ops
    for name, data in pr.far_matches().items():
        assert ops.png_parse(data).eligible, name
        got, err = pr.decode(data)
        assert err == 0, (name, err)
        np.testing.assert_array_equal(got, pr.pillow_bytes(data), err_msg=name)
