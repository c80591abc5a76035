"""GPU input preprocessing against the reference's outputs (tests/golden/images.npz): the SLAM path (PIL resize, crop,
ImgNorm) bitwise, the demo path (CenterCrop + antialiased bilinear Resize) within 1e-5, batching and pitched inputs
bitwise, and a model run over the preprocessed images."""
import os
import sys

import numpy as np
import pytest
import torch

from must3r_b200 import synthetic as syn
from must3r_b200.engine import images

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from images_golden import DEMO, SLAM, assert_close_to_demo, assert_resized_is_pils, case, frame, sha  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", SLAM)
def test_slam_path_is_bitwise_the_reference(name):
    c = case("slam", name)
    f = frame(c)
    H1, W1, res = (int(v) for v in c["input"])
    d, focal = images.preproc_frame(f, 7, res=res)
    assert d["img"].is_cuda and d["img"].dtype == torch.float32 and list(d["img"].shape) == list(c["img_shape"])
    assert sha(d["img"]) == str(c["img_sha256"])
    assert np.array_equal(d["true_shape"], c["true_shape"]) and d["true_shape"].dtype == np.int32
    assert np.array_equal(d["offset"], c["offset"]) and d["offset"].dtype == np.int32
    assert d["idx"] == 7 and d["instance"] == "7" and focal == float(c["focal"])
    # the uint8 intermediate, from a device-resident frame
    H, W = (int(v) for v in c["resized_shape"][:2])
    u8, img = images.resize_pil(torch.from_numpy(f).cuda(), (H, W), str(c["filter"]), crop=tuple(int(v) for v in c["crop"]))
    assert_resized_is_pils(u8[0].cpu().numpy(), c)
    assert sha(img) == str(c["img_sha256"])


@pytest.mark.parametrize("name", DEMO)
def test_demo_path_matches_the_reference(name):
    c = case("demo", name)
    f = frame(c)
    H, W, size = (int(v) for v in c["input"])
    d = images.load_images([f], size, verbose=False)[0]
    assert np.array_equal(d["true_shape"], c["true_shape"]) and d["true_shape"].dtype == np.int32
    assert_close_to_demo(d["img"].cpu().numpy(), c)
    op, to_rescaled, to_orig = images.get_resize_function(size, 16, H, W)
    assert np.array_equal(to_orig, c["to_orig"]) and np.array_equal(to_rescaled, c["to_rescaled"])
    assert torch.equal(op(f).cpu(), d["img"].cpu())


def _frames(n, H, W, seed0=50):
    return [syn.synthetic_frame(H, W, seed=seed0 + i) for i in range(n)]


@pytest.mark.parametrize("HW,res", [((480, 640), 512), ((300, 400), 512), ((480, 640), 224)])
def test_batch_equals_single_calls(HW, res):
    fs = _frames(5, *HW)
    (h, w), filt, crop, _ = images._slam_geometry(HW[0], HW[1], res)
    _, batch = images.resize_pil(np.stack(fs), (h, w), filt, crop=crop)
    for i, f in enumerate(fs):
        assert torch.equal(batch[i:i + 1], images.preproc_frame(f, i, res=res)[0]["img"])
    # the demo path: one launch per size group, in input order
    imgs = images.load_images(fs + _frames(2, 700, 1000), res, verbose=False)
    op, _, _ = images.get_resize_function(res, 16, *HW)
    batch = op(np.stack(fs))
    for i in range(len(fs)):
        assert torch.equal(imgs[i]["img"], batch[i])
        assert torch.equal(imgs[i]["img"], op(fs[i]))


def test_pitched_and_cropped_views_equal_their_contiguous_copies():
    big = torch.from_numpy(syn.synthetic_frame(1100, 2000, seed=77)).cuda()
    view = big[7:7 + 1080, 33:33 + 1920]                      # row pitch 6000 bytes, offset origin
    assert not view.is_contiguous()
    dense = view.contiguous()
    for res in (512, 224):
        a = images.preproc_frame(view, 0, res=res)[0]["img"]
        b = images.preproc_frame(dense, 0, res=res)[0]["img"]
        c = images.preproc_frame(dense.cpu().numpy(), 0, res=res)[0]["img"]
        assert torch.equal(a, b) and torch.equal(a, c)
    op, _, _ = images.get_resize_function(512, 16, 1080, 1920)
    assert torch.equal(op(view), op(dense)) and torch.equal(op(view), op(dense.cpu().numpy()))
    # frames of a batch with a frame stride larger than the frame
    frames = torch.from_numpy(np.stack(_frames(3, 490, 650))).cuda()[:, 5:485, 3:643]
    (h, w), filt, crop, _ = images._slam_geometry(480, 640, 512)
    assert torch.equal(images.resize_pil(frames, (h, w), filt, crop=crop)[1],
                       images.resize_pil(frames.contiguous(), (h, w), filt, crop=crop)[1])
    op480, _, _ = images.get_resize_function(512, 16, 480, 640)
    assert torch.equal(op480(frames), op480(frames.contiguous()))


def test_side_stream_matches_default_stream():
    f = _frames(1, 480, 640)[0]
    ref = images.preproc_frame(f, 0)[0]["img"]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = images.preproc_frame(f, 0)[0]["img"]
    s.synchronize()
    assert torch.equal(got, ref)


def test_inference_multi_ar_over_loaded_images_equals_fixture_images():
    """224x224 views: the GPU PIL path's uint8 crops, passed through load_images (a 224x224 input is only normalised),
    against the fixture's images: bitwise equal inputs, so the whole model run is bitwise equal."""
    from must3r_b200 import engine
    from must3r_b200.model import Dust3rEncoder, MUSt3R, set_precision
    names = ["s224", "s224portrait", "s224square"]
    crops, fixture = [], []
    for n in names:
        c = case("slam", n)
        H, W = (int(v) for v in c["resized_shape"][:2])
        x0, y0, w, h = (int(v) for v in c["crop"])
        u8, _ = images.resize_pil(torch.from_numpy(frame(c)).cuda(), (H, W), str(c["filter"]))
        resized = u8[0].cpu().numpy()
        assert_resized_is_pils(resized, c)
        crops.append(u8[0, y0:y0 + h, x0:x0 + w])                 # a cropped CUDA view
        t = torch.from_numpy(np.ascontiguousarray(resized[y0:y0 + h, x0:x0 + w])).permute(2, 0, 1).float()
        t = ((t / 255) - 0.5) / 0.5
        assert sha(t[None]) == str(c["img_sha256"])
        fixture.append(t.cuda())
    loaded = images.load_images(crops, 224, verbose=False)
    for d in loaded:
        assert list(d["true_shape"]) == [224, 224]
    set_precision(torch.float16)
    enc = Dust3rEncoder(img_size=(224, 224), depth=2)
    dec = MUSt3R(img_size=(224, 224), depth=2, feedback_type="single_mlp", memory_mode="kv", landscape_only=False)
    enc.load_state_dict(syn.encoder_state_dict(3, depth=2))
    dec.load_state_dict(syn.decoder_state_dict(3, depth=2))
    enc, dec = enc.cuda().eval(), dec.cuda().eval()
    raw = lambda pm: {"raw": pm}  # noqa: E731
    outs = []
    for views in ([d["img"] for d in loaded], fixture):
        tss = [torch.tensor([224, 224]) for _ in views]
        ids = [torch.tensor(i) for i in range(len(views))]
        _, pm = engine.inference_multi_ar(enc, dec, views, ids, tss, [2, 1], post_process_function=raw, device="cuda")
        outs.append(torch.stack([p["raw"] for p in pm]))
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])
