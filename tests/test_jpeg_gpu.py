"""The CUDA JPEG decoder (csrc/jpeg.cu, engine/jpeg.py) against Pillow, bit for bit: every eligible corpus file with
and without the EXIF transpose, a mixed batch, malformed streams (status word, guard bytes, Pillow's outcome), and the
loaders that use it (load_images, ReadAhead, the SLAM command line)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import jpeg_ref as jr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    return jr.write(tmp_path_factory.mktemp("jpeg"), jr.corpus(big=True))


def _gpu_decode(paths, exif_transpose):
    """The device path alone: every file must be taken by the GPU and reported well-formed."""
    from must3r_b200.engine import jpeg
    items = [jpeg.Parsed(p, exif_transpose) for p in paths]
    assert all(it.gpu for it in items), [p for p, it in zip(paths, items) if not it.gpu]
    outs = jpeg.decode_parsed(items, torch.device("cuda", 0))
    handed_back = [os.path.basename(p) for p, o in zip(paths, outs) if o is None]
    assert not handed_back, f"{len(handed_back)} of {len(paths)} handed to Pillow: {handed_back}"
    return [o.cpu().numpy() for o in outs]


@pytest.mark.parametrize("exif_transpose", [False, True])
def test_corpus_bitwise_equal_to_pillow(files, exif_transpose):
    eligible = [p for p, e in files if e]
    mism = []
    for p in eligible:                     # one image per batch, the large uniform-noise frames at q100 included
        got = _gpu_decode([p], exif_transpose)[0]
        want = jr.pillow(p, exif_transpose)
        if got.shape != want.shape or not np.array_equal(got, want):
            mism.append(os.path.basename(p))
    assert not mism, mism


def test_mixed_batch_equals_single_images(files):
    eligible = [p for p, e in files if e]
    batch = _gpu_decode(eligible, True)
    for p, got in zip(eligible, batch):
        np.testing.assert_array_equal(got, jr.pillow(p, True), err_msg=p)


def test_public_function_routes_every_file(files):
    from must3r_b200.engine import jpeg
    paths = [p for p, _ in files]
    outs = jpeg.decode_files(paths, "cuda", exif_transpose=True)
    for p, o in zip(paths, outs):
        assert o.is_cuda and o.dtype == torch.uint8
        np.testing.assert_array_equal(o.cpu().numpy(), jr.pillow(p, True), err_msg=p)


def _malformed(tmp_path):
    img = jr.content(64, 96, "noisy")
    good = jr.save(img, format="JPEG", quality=90, subsampling=2)
    sos = good.index(b"\xff\xda")
    start = sos + 2 + int.from_bytes(good[sos + 2:sos + 4], "big")
    end = len(good) - 2
    cases = {}
    cases["truncated"] = good[:start + (end - start) // 2]
    b = bytearray(good)
    k = start + (end - start) // 3
    b[k] = (b[k] ^ 0x5A) if (b[k] ^ 0x5A) != 0xFF else 0x11
    cases["flipped"] = bytes(b)
    j = start + 40                         # 48 one bits (stuffed FF bytes): no code of a valid table is all ones
    while good[j - 1] == 0xFF:
        j += 1
    cases["absent_code"] = good[:j] + b"\xff\x00" * 6 + good[j + 12:]
    cases["early_eoi"] = good[:start + (end - start) // 2] + b"\xff\xd9"
    paths = {}
    for name, data in cases.items():
        p = tmp_path / f"{name}.jpg"
        p.write_bytes(data)
        paths[name] = str(p)
    return paths


def test_malformed_streams(tmp_path):
    """Each malformed stream that reaches the decoder sets exactly the status bits the reference decoder predicts, and
    writes nothing outside its output; the public function then gives Pillow's outcome."""
    from must3r_b200.engine import jpeg
    from must3r_b200 import ops, _lib
    import ctypes as C
    paths = _malformed(tmp_path)
    dev = torch.device("cuda", 0)
    must = {"flipped": None, "absent_code": jr.EHUFF, "early_eoi": jr.ESHORT}
    for name, p in paths.items():
        it = jpeg.Parsed(p, False)
        host = torch.empty(((it.info.prep_bytes + 255) // 256 * 256) + 256, dtype=torch.uint8, pin_memory=True)
        d = ops.jpeg_prepare(it.data, it.info, 1, host.data_ptr(), 0) if it.gpu else None
        if name == "truncated":             # no EOI: not eligible after the entropy pass
            assert d is None
            continue
        assert d is not None, name
        _, want_err = jr.decode(it.data)
        assert want_err != 0, name
        if must[name] is not None:
            assert want_err & must[name], name
        H, W = it.info.height, it.info.width
        guard = torch.full((H * W * 3 + 2 * 4096,), 0xA5, dtype=torch.uint8, device=dev)
        arr = (_lib.JpegDesc * 1)(d)
        work_bytes = ops.jpeg_plan(arr)
        arr[0].out = guard.data_ptr() + 4096
        n = (it.info.prep_bytes + 255) // 256 * 256
        C.memmove(host.data_ptr() + n, C.addressof(arr), C.sizeof(arr))
        blob = host[:n + C.sizeof(arr)].to(dev)
        work = torch.empty(work_bytes, dtype=torch.uint8, device=dev)
        status = torch.empty(1, dtype=torch.int32, device=dev)
        ops.jpeg_decode(arr, blob, n, work, status)
        torch.cuda.synchronize()
        g = guard.cpu().numpy()
        assert (g[:4096] == 0xA5).all() and (g[-4096:] == 0xA5).all(), name
        assert int(status.item()) == want_err, name
    bad = tmp_path / "all_ones.jpg"         # a table libjpeg rejects: never reaches the decoder
    bad.write_bytes(jr.all_ones_dc_code(jr.save(jr.content(33, 65, "smooth"), format="JPEG", quality=90)))
    paths["all_ones"] = str(bad)
    for name, p in paths.items():          # the public function gives Pillow's outcome
        try:
            want = jr.pillow(p, False)
        except Exception as e:
            with pytest.raises(type(e)):
                jpeg.decode_files([p], "cuda")
            continue
        got = jpeg.decode_files([p], "cuda")[0].cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg=name)


def test_load_images_jpeg_paths_equal_pillow_arrays(tmp_path):
    from must3r_b200.engine import images
    paths = []
    for k, (H, W) in enumerate([(480, 640), (480, 640), (512, 384), (300, 500)]):
        p = tmp_path / f"{k}.jpg"
        p.write_bytes(jr.save(jr.content(H, W, "smooth", seed=k), format="JPEG", quality=90, subsampling=k % 3))
        paths.append(str(p))
    png = tmp_path / "z.png"
    png.write_bytes(jr.save(jr.content(480, 640, "smooth", seed=9), format="PNG"))
    paths.append(str(png))
    a = images.load_images(paths, 512, verbose=False, device="cuda")
    b = images.load_images([jr.pillow(p, False) for p in paths], 512, verbose=False, device="cuda")
    for x, y in zip(a, b):
        assert torch.equal(x["img"], y["img"])
        assert (x["true_shape"] == y["true_shape"]).all()


def test_read_ahead_equals_pillow(files):
    from must3r_b200.engine import frames
    paths = [p for p, _ in files][::3]
    with frames.ReadAhead(paths, "cuda:0", depth=2) as src:
        for p in paths:
            got = src.get()
            np.testing.assert_array_equal(got.cpu().numpy(), frames.decode(p), err_msg=p)


def test_slam_cli_on_jpeg_folder_equals_arrays(tmp_path):
    """python -m must3r_b200.slam on a JPEG folder: the same poses and keyframes as the run fed PIL-decoded PNGs of
    the same pixels (PNG frames take the Pillow path)."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_slam_golden as mk
    chkpt = str(tmp_path / "tiny.pth")
    mk.write_checkpoint(chkpt)
    base = jr.content(240, 320, "smooth")
    outs = {}
    for kind in ("jpg", "png"):
        d = tmp_path / kind
        d.mkdir()
        for k in range(6):
            img = np.roll(base, 6 * k, axis=1)
            jp = jr.save(img, format="JPEG", quality=92)
            if kind == "jpg":
                (d / f"{k:03d}.jpg").write_bytes(jp)
            else:                           # the same pixels, as Pillow decodes the JPEG
                import io
                import PIL.Image
                (d / f"{k:03d}.png").write_bytes(jr.save(np.asarray(PIL.Image.open(io.BytesIO(jp)).convert("RGB")),
                                                          format="PNG"))
        o = tmp_path / f"out_{kind}"
        cmd = [sys.executable, "-m", "must3r_b200.slam", "--chkpt", chkpt, "--res", "224", "--input", str(d),
               "--output", str(o), "--device", "cuda:0"]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        outs[kind] = o
    names = sorted(f for f in os.listdir(outs["jpg"]) if f.endswith(".npz"))
    assert names and names == sorted(f for f in os.listdir(outs["png"]) if f.endswith(".npz"))
    for f in names:
        a, b = np.load(outs["jpg"] / f, allow_pickle=True), np.load(outs["png"] / f, allow_pickle=True)
        assert sorted(a.files) == sorted(b.files)
        for k in set(a.files) - {"fps", "gpumem"}:  # the run's wall-clock rate and memory use
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{f}:{k}")
