"""The JPEG decoder's host side, without a GPU: the header parser against what Pillow reports, the entropy-segment
preparation against a Python restatement, the ABI structs' layout, and which files go to Pillow."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest

import jpeg_ref as jr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from must3r_b200 import _lib
    return _lib.lib()


@pytest.fixture(scope="module")
def corpus():
    return jr.corpus()


def test_parser_agrees_with_pillow(lib, corpus):
    import PIL.Image
    from must3r_b200 import ops
    for name, data, eligible in corpus:
        info = ops.jpeg_parse(data)
        assert bool(info.eligible) == eligible, name
        if not eligible:
            continue
        im = PIL.Image.open(io.BytesIO(data))
        assert (info.width, info.height) == im.size, name
        o = im.getexif().get(0x0112, 1)
        assert info.orientation == (o if 1 <= o <= 8 else 1) and info.orientation_exact, name
        if im.mode == "RGB":
            # Pillow's layer: (id, h, v, qtable) per component
            assert [(h, v) for _, h, v, _ in im.layer] == list(zip(info.hs, info.vs)), name
        if name.startswith("rst_blocks"):
            assert info.restart_interval == int(name.split("_")[1][len("blocks"):]), name
        elif not name.startswith("rst_"):
            assert info.restart_interval == 0, name


def _unstuff(data: bytes, start: int):
    """Python restatement of the entropy-segment pass: (bytes, [segment start bits])."""
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


def test_prepare_unstuffs_and_splits_like_python(lib, corpus):
    from must3r_b200 import ops
    for name, data, eligible in corpus:
        if not eligible:
            continue
        info = ops.jpeg_parse(data)
        buf = np.zeros(info.prep_bytes + 64, np.uint8)
        d = ops.jpeg_prepare(data, info, 1, buf.ctypes.data, 0)
        assert d is not None, name
        want, segs = _unstuff(data, info.scan_offset)
        assert d.stream_bytes == len(want), name
        assert bytes(buf[d.stream_off:d.stream_off + d.stream_bytes]) == want, name
        assert (buf[d.stream_off + d.stream_bytes:d.stream_off + d.stream_bytes + 8] == 0).all()
        got = np.frombuffer(buf[d.segs_off:d.segs_off + 8 * d.nseg].tobytes(), np.uint32).reshape(-1, 2)
        assert list(got[:, 0]) == segs, name
        assert list(got[1:, 0]) == list(got[:-1, 1]) and got[-1, 1] == 8 * len(want)
        subs = np.frombuffer(buf[d.subs_off:d.subs_off + 16 * d.nsub].tobytes(), np.uint32).reshape(-1, 4)
        for s, (a, b) in enumerate(got):            # the subsequences tile each segment
            mine = subs[subs[:, 2] == s]
            assert mine[0, 0] == a and mine[-1, 1] == b and (mine[1:, 0] == mine[:-1, 1]).all(), name


def test_structs_match_the_c_layout(lib, tmp_path):
    from must3r_b200 import _lib
    prog = tmp_path / "sz.c"
    prog.write_text('#include <stdio.h>\n#include "must3r_b200.h"\nint main(){printf("%zu %zu\\n",'
                    'sizeof(m3r_jpeg_info),sizeof(m3r_jpeg_desc));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(prog), "-o", str(exe)])
    sizes = [int(v) for v in subprocess.check_output([str(exe)]).split()]
    assert sizes == [C.sizeof(_lib.JpegInfo), C.sizeof(_lib.JpegDesc)]


def test_routing(lib, tmp_path, corpus):
    """PNGs and ineligible JPEGs take the Pillow path; unusual EXIF metadata keeps a JPEG off the transposing GPU
    path only."""
    from must3r_b200.engine import jpeg
    for p, eligible in jr.write(tmp_path, corpus):
        for t in (False, True):
            assert jpeg.Parsed(p, t).gpu == eligible, p
    img = jr.content(17, 31, "smooth")
    two = jr.save(img, format="JPEG", quality=90, exif=jr.exif_orientation(6, True))
    k = two.index(b"\xff\xe1")
    n = int.from_bytes(two[k + 2:k + 4], "big")
    two = two[:k + 2 + n] + two[k:k + 2 + n] + two[k + 2 + n:]      # a second Exif segment: Pillow concatenates them
    p = tmp_path / "two_exif.jpg"
    p.write_bytes(two)
    assert jpeg.Parsed(str(p), False).gpu and not jpeg.Parsed(str(p), True).gpu


def _small(corpus):
    import PIL.Image
    for name, data, eligible in corpus:
        if eligible and np.prod(PIL.Image.open(io.BytesIO(data)).size) <= 4000:
            yield name, data


def test_reference_decoder_bitwise_equal_to_pillow(corpus):
    """The numpy statement of the kernels' arithmetic reproduces Pillow on every small eligible file, with and without
    the EXIF transpose, and finds no error in any of them."""
    import PIL.Image
    import PIL.ImageOps
    n = 0
    for name, data in _small(corpus):
        im = PIL.Image.open(io.BytesIO(data))
        o = im.getexif().get(0x0112, 1)
        for t in (False, True):
            want = np.asarray((PIL.ImageOps.exif_transpose(im) if t else im).convert("RGB"))
            got, err = jr.decode(data, o if t and 1 <= o <= 8 else 1)
            assert err == 0, name
            np.testing.assert_array_equal(got, want, err_msg=f"{name} transpose={t}")
            n += 1
    assert n >= 200


@pytest.mark.parametrize("sub_bits", [2048, 16])
def test_partition_model_agrees_with_sequential_decoding(corpus, sub_bits):
    """The self-synchronising partition settles on the sequential decoder's state at every subsequence boundary and
    counts the blocks it completes in between, at the kernels' subsequence length (SUB_BITS in csrc/jpeg.cu) and at a
    tiny one that needs many rounds."""
    src = open(os.path.join(ROOT, "must3r_b200", "csrc", "jpeg.cu")).read()
    assert "constexpr int SUB_BITS = 2048;" in src
    names = {"33x65_noisy_420_q100", "33x65_noisy_444_q90", "33x65_smooth_422_q50", "rst_blocks4_420", "opt_420",
             "33x65_noisy_gray_q90"}
    rounds = []
    for name, data, _ in corpus:
        if name not in names:
            continue
        j = jr.Jpeg(data)
        for seg in range(len(j.segs)):
            trace = j.trace(seg)
            entry, counts, r = jr.partition(j, seg, sub_bits)
            rounds.append(r)
            a, b = j.segs[seg]
            for g, s in enumerate(range(a, b, sub_bits)):
                # the first symbol boundary at or past the subsequence's start, and past its end
                k0 = next(k for k, (st, _) in enumerate(trace) if st[0] >= s)
                k1 = next((k for k, (st, _) in enumerate(trace) if st[0] >= min(s + sub_bits, b)), len(trace) - 1)
                assert entry[g] == (trace[k0][0] if g else (a, 0, 0)), (name, seg, g)
                assert counts[g] == trace[k1][1] - trace[k0][1], (name, seg, g)
    assert len(rounds) >= len(names)
    if sub_bits == 16:
        assert max(rounds) > 1


def test_table_with_an_all_ones_code_goes_to_pillow(lib, tmp_path):
    """libjpeg rejects a Huffman table whose last code is all ones, so Pillow raises: the parser reports the file not
    eligible, and the loaders hand it to Pillow."""
    import PIL.Image
    from must3r_b200 import ops
    from must3r_b200.engine import jpeg
    good = jr.save(jr.content(33, 65, "smooth"), format="JPEG", quality=90)
    bad = jr.all_ones_dc_code(good)
    assert ops.jpeg_parse(good).eligible and not ops.jpeg_parse(bad).eligible
    p = tmp_path / "all_ones.jpg"
    p.write_bytes(bad)
    with pytest.raises(OSError):
        PIL.Image.open(str(p)).convert("RGB")
    assert not jpeg.Parsed(str(p), False).gpu
