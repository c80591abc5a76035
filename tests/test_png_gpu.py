"""The CUDA PNG decoder (csrc/png.cu, engine/png.py) against Pillow, bit for bit: every eligible corpus file with and
without the EXIF transpose, a mixed batch, the routing of a mixed list, malformed streams (status word, guard bytes,
Pillow's outcome), and the loaders that use it (load_images, ReadAhead, the SLAM command line)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import jpeg_ref as jr
import png_ref as pr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    return pr.write(tmp_path_factory.mktemp("png"), pr.corpus() + pr.big_corpus())


def _gpu_decode(paths, exif_transpose):
    """The device path alone: every file must be taken by the GPU and reported well-formed."""
    from must3r_b200.engine import png
    items = [png.Parsed(p, exif_transpose) for p in paths]
    assert all(it.gpu for it in items), [p for p, it in zip(paths, items) if not it.gpu]
    outs = png.decode_parsed(items, torch.device("cuda", 0))
    handed_back = [os.path.basename(p) for p, o in zip(paths, outs) if o is None]
    assert not handed_back, f"{len(handed_back)} of {len(paths)} handed to Pillow: {handed_back}"
    return [o.cpu().numpy() for o in outs]


def _eligible(files, exif_transpose):
    from must3r_b200.engine import png
    return [p for p, e in files if e and png.Parsed(p, exif_transpose).gpu]


@pytest.mark.parametrize("exif_transpose", [False, True])
def test_corpus_bitwise_equal_to_pillow(files, exif_transpose):
    mism = []
    for p in _eligible(files, exif_transpose):
        got = _gpu_decode([p], exif_transpose)[0]
        want = pr.pillow(p, exif_transpose)
        if got.shape != want.shape or not np.array_equal(got, want):
            mism.append(os.path.basename(p))
    assert not mism, mism


def test_far_window_matches(tmp_path):
    """Valid streams that copy from the far end of deflate's 32K window decode on the device, alone and in one batch,
    without being handed back, to Pillow's pixels."""
    paths = []
    for name, data in pr.far_matches().items():
        p = tmp_path / f"{name}.png"
        p.write_bytes(data)
        paths.append(str(p))
    for p, got in zip(paths, _gpu_decode(paths, False)):
        np.testing.assert_array_equal(got, pr.pillow(p), err_msg=p)
    for p in paths:
        np.testing.assert_array_equal(_gpu_decode([p], False)[0], pr.pillow(p), err_msg=p)


def test_mixed_batch_equals_single_images(files):
    eligible = _eligible(files, False)
    batch = _gpu_decode(eligible, False)
    for p, got in zip(eligible, batch):
        np.testing.assert_array_equal(got, _gpu_decode([p], False)[0], err_msg=p)


def test_public_function_routes_every_file(files, tmp_path):
    from must3r_b200.engine import imagefiles
    jpegs = jr.write(tmp_path, jr.corpus())
    other = tmp_path / "x.bmp"
    import PIL.Image
    PIL.Image.fromarray(pr.content(10, 12, "smooth")).save(other)
    paths = [p for p, _ in files] + [p for p, _ in jpegs][::4] + [str(other)]
    for t in (False, True):
        outs = imagefiles.decode_files(paths, "cuda", exif_transpose=t)
        for p, o in zip(paths, outs):
            assert o.is_cuda and o.dtype == torch.uint8
            np.testing.assert_array_equal(o.cpu().numpy(), pr.pillow(p, t), err_msg=p)


def test_orientation_is_applied_on_the_store():
    from must3r_b200 import ops, _lib
    img = pr.content(13, 21, "smooth")
    data = pr.png_bytes(img, 2)
    info = ops.png_parse(data)
    dev = torch.device("cuda", 0)
    want = {1: img, 2: img[:, ::-1], 3: img[::-1, ::-1], 4: img[::-1], 5: img.transpose(1, 0, 2),
            6: np.rot90(img, -1), 7: np.rot90(img, -1)[::-1], 8: np.rot90(img, 1)}
    for o, w in want.items():
        got = _run(data, info, o, dev, (w.shape[0], w.shape[1]))[0]
        np.testing.assert_array_equal(got[4096:-4096].reshape(w.shape), w, err_msg=str(o))


def _run(data, info, orientation, dev, out_hw):
    """One image through the ops layer into an output with 4096 guard bytes on each side: (bytes, status)."""
    from must3r_b200 import ops, _lib
    n = (info.prep_bytes + 255) // 256 * 256
    host = torch.empty(n + 256, dtype=torch.uint8, pin_memory=True)
    d = ops.png_prepare(data, info, orientation, host.data_ptr(), 0)
    guard = torch.full((out_hw[0] * out_hw[1] * 3 + 2 * 4096,), 0xA5, dtype=torch.uint8, device=dev)
    arr = (_lib.PngDesc * 1)(d)
    work_bytes = ops.png_plan(arr)
    arr[0].out = guard.data_ptr() + 4096
    C.memmove(host.data_ptr() + n, C.addressof(arr), C.sizeof(arr))
    blob = host[:n + C.sizeof(arr)].to(dev)
    work = torch.zeros(work_bytes + 4096, dtype=torch.uint8, device=dev)
    status = torch.empty(1, dtype=torch.int32, device=dev)
    ops.png_decode(arr, blob, n, work, status)
    torch.cuda.synchronize()
    w = work.cpu().numpy()
    assert (w[work_bytes:] == 0).all()
    return guard.cpu().numpy(), int(status.item())


def test_malformed_streams(tmp_path):
    """Each malformed stream sets exactly the status bits the statement predicts and writes nothing outside its output;
    the public function then gives Pillow's outcome."""
    from must3r_b200 import ops
    from must3r_b200.engine import imagefiles
    cases, (H, W) = pr.malformed()
    datas = {name: pr.with_stream(s, H, W) for name, (s, _, _) in cases.items()}
    pal = np.array([[1, 2, 3], [4, 5, 6]], np.uint8)
    datas["palette_index"] = pr.png_bytes(np.array([[[0], [1], [3]]], np.uint8), 3, palette=pal)
    dev = torch.device("cuda", 0)
    for name, data in datas.items():
        info = ops.png_parse(data)
        assert info.eligible, name
        _, want_err = pr.decode(data)
        assert want_err != 0, name
        g, st = _run(data, info, 1, dev, (info.height, info.width))
        assert (g[:4096] == 0xA5).all() and (g[-4096:] == 0xA5).all(), name
        assert st == want_err, (name, st, want_err)
    for name, data in datas.items():        # the public function gives Pillow's outcome
        p = tmp_path / f"{name}.png"
        p.write_bytes(data)
        try:
            want = pr.pillow(str(p))
        except Exception as e:
            with pytest.raises(type(e)) as got:
                imagefiles.decode_files([str(p)], "cuda")
            assert str(got.value) == str(e), name
            continue
        got = imagefiles.decode_files([str(p)], "cuda")[0].cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg=name)


def test_load_images_png_paths_equal_pillow_arrays(tmp_path):
    from must3r_b200.engine import images
    paths = []
    for k, (H, W) in enumerate([(480, 640), (480, 640), (512, 384), (300, 500)]):
        p = tmp_path / f"{k}.png"
        p.write_bytes(pr.png_bytes(pr.content(H, W, "smooth", seed=k, channels=[3, 4, 3, 1][k]), [2, 6, 2, 0][k]))
        paths.append(str(p))
    a = images.load_images(paths, 512, verbose=False, device="cuda")
    b = images.load_images([pr.pillow(p) for p in paths], 512, verbose=False, device="cuda")
    for x, y in zip(a, b):
        assert torch.equal(x["img"], y["img"])
        assert (x["true_shape"] == y["true_shape"]).all()


def test_read_ahead_equals_pillow(files):
    from must3r_b200.engine import frames
    paths = [p for p, _ in files][::2]
    with frames.ReadAhead(paths, "cuda:0", depth=2) as src:
        for p in paths:
            got = src.get()
            np.testing.assert_array_equal(got.cpu().numpy(), frames.decode(p), err_msg=p)


def test_read_ahead_with_png_frames_on_the_gpu(files, monkeypatch):
    """The read-ahead with PNG frames decoded on the GPU (the mode tools/bench_png.py measures against Pillow): every
    eligible frame goes through the device decoder on the reader's stream and equals Pillow."""
    from must3r_b200.engine import frames, imagefiles, jpeg, png
    monkeypatch.setattr(imagefiles, "READ_AHEAD_ON_GPU", (jpeg.Parsed, png.Parsed))
    decoded = []
    real = png.decode_parsed

    def counted(items, dev):
        decoded.extend(it.path for it in items)
        return real(items, dev)

    monkeypatch.setattr(png, "decode_parsed", counted)
    paths = [p for p, _ in files]
    with frames.ReadAhead(paths, "cuda:0", depth=3) as src:
        for p in paths:
            np.testing.assert_array_equal(src.get().cpu().numpy(), frames.decode(p), err_msg=p)
    assert decoded == [p for p in paths if png.Parsed(p, True).gpu]
    assert decoded


def test_slam_cli_on_png_folder_equals_arrays(tmp_path):
    """python -m must3r_b200.slam on a PNG folder: the same poses and keyframes as the run fed the same pixels as
    BMP frames (which Pillow decodes)."""
    import PIL.Image
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_slam_golden as mk
    chkpt = str(tmp_path / "tiny.pth")
    mk.write_checkpoint(chkpt)
    base = pr.content(240, 320, "smooth")
    outs = {}
    for kind in ("png", "bmp"):
        d = tmp_path / kind
        d.mkdir()
        for k in range(6):
            img = np.roll(base, 6 * k, axis=1)
            if kind == "png":
                (d / f"{k:03d}.png").write_bytes(pr.png_bytes(img, 2))
            else:
                PIL.Image.fromarray(img).save(d / f"{k:03d}.bmp")
        o = tmp_path / f"out_{kind}"
        cmd = [sys.executable, "-m", "must3r_b200.slam", "--chkpt", chkpt, "--res", "224", "--input", str(d),
               "--output", str(o), "--device", "cuda:0"]
        r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-3000:]
        outs[kind] = o
    names = sorted(f for f in os.listdir(outs["png"]) if f.endswith(".npz"))
    assert names and names == sorted(f for f in os.listdir(outs["bmp"]) if f.endswith(".npz"))
    for f in names:
        a, b = np.load(outs["png"] / f, allow_pickle=True), np.load(outs["bmp"] / f, allow_pickle=True)
        assert sorted(a.files) == sorted(b.files)
        for k in set(a.files) - {"fps", "gpumem"}:
            np.testing.assert_array_equal(a[k], b[k], err_msg=f"{f}:{k}")
