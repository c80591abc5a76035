"""The demo's reconstruction modes end to end on the GPU (must3r_b200/engine/demo.py) against the reference's own run
(tests/golden/demo.npz, made by tests/golden/make_demo_golden.py), and `python -m must3r_b200.reconstruct`.

Tolerances, those of the existing goldens for the fp16 CUDA model against the fp32 reference: pointmaps within 1.5e-3
relative L2 (the parity gate of smoke()); camera poses 3e-2 absolute and focals 3e-2 relative (20x that, as the SLAM
golden's poses: they come from a weighted fit over those points); keyframe lists, view order and point counts exactly
(the golden's thresholds sit in gaps of the reference's confidences, and every vidslam overlap score is >= 5 % from its
threshold)."""
import os
import pickle
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from must3r_b200 import synthetic as syn
from must3r_b200.engine import demo
from must3r_b200.model import load_model

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_demo_golden as mk  # noqa: E402  (checkpoint, images and cases of the fixture; the reference is not imported)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(HERE, "golden", "demo.npz"))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("demo")
    chkpt = str(d / "tiny.pth")
    mk.mk.write_checkpoint(chkpt)
    img_dir = d / "images"
    img_dir.mkdir()
    return chkpt, mk.write_images(str(img_dir))


@pytest.fixture(scope="module")
def model(files):
    return load_model(files[0], device="cuda", img_size=mk.IMAGE_SIZE, verbose=False)


def _run(model, paths, name, g, monkeypatch):
    kw = dict(mk.CASES[name])
    mode = kw.pop("execution_mode")
    full = dict(num_mem_images=4, render_once=False, vidseq_local_context_size=0, keyframe_interval=3,
                slam_local_context_size=0, subsample=2, min_conf_keyframe=1.5, keyframe_overlap_thr=0.05,
                overlap_percentile=85.0)
    full.update(kw)
    if mode == "vidslam":
        full["keyframe_overlap_thr"] = float(g["vidslam_keyframe_overlap_thr"])
    keyframes = []
    if mode in ("vidseq", "vidslam"):
        orig = demo.inference_video_multi_ar

        def recording(*a, **k):
            f = k["is_keyframe_function"]

            def kf(id, res, scene_state):
                r = bool(f(id, res, scene_state))
                if r:
                    keyframes.append(int(id))
                return r
            k["is_keyframe_function"] = kf
            return orig(*a, **k)
        monkeypatch.setattr(demo, "inference_video_multi_ar", recording)
    scene, outfile = demo.get_reconstructed_scene(None, None, False, model, None, "cuda", False, mk.IMAGE_SIZE, False,
                                                  paths, 1, 0, mode, min_conf_thr=1.05, as_pointcloud=True,
                                                  transparent_cams=False, local_pointmaps=False, cam_size=0.05, **full)
    assert outfile is None
    keyframes = [0, 1] + keyframes if mode != "linseq" else demo._linspace_keyframes(len(paths), full["num_mem_images"])
    return scene, keyframes


@pytest.mark.parametrize("name", list(mk.CASES))
def test_mode_against_the_reference(name, g, files, model, monkeypatch):
    chkpt, paths = files
    scene, keyframes = _run(model, paths, name, g, monkeypatch)
    assert keyframes == g[f"{name}_keyframes"].tolist()
    assert [paths.index(p) for p in scene.image_list] == g[f"{name}_order"].tolist()
    n = len(paths)
    assert len(scene.x_out) == len(scene.imgs) == len(scene.focals) == len(scene.cams2world) == len(scene.true_shape) == n
    for i in range(n):
        o = scene.x_out[i]
        assert not o["pts3d"].is_cuda and not o["conf"].is_cuda and not scene.cams2world[i].is_cuda
        assert isinstance(scene.imgs[i], np.ndarray) and scene.imgs[i].shape == tuple(o["conf"].shape) + (3,)
        assert tuple(scene.true_shape[i].tolist()) == tuple(o["conf"].shape)
        e = syn.rel_l2(o["pts3d"][::mk.SUB, ::mk.SUB], torch.from_numpy(g[f"{name}_pts3d_{i}"]))
        assert e < 1.5e-3, (i, e)
        e = syn.rel_l2(o["conf"][::mk.SUB, ::mk.SUB], torch.from_numpy(g[f"{name}_conf_{i}"]))
        assert e < 1.5e-3, (i, e)
    np.testing.assert_allclose(np.array(scene.focals), g[f"{name}_focal"], rtol=3e-2)
    np.testing.assert_allclose(np.stack([m.numpy() for m in scene.cams2world]), g[f"{name}_c2w"], atol=3e-2)
    clouds = demo.get_3D_models_from_scene(scene, g[f"{name}_thr"].tolist())
    assert [p.shape[0] for p, _ in clouds] == g[f"{name}_count"].tolist()
    for (p, c), mean in zip(clouds, g[f"{name}_cloud_mean"]):
        if p.shape[0]:
            np.testing.assert_allclose(np.concatenate([p.mean(0), c.mean(0)]), mean, rtol=2e-2, atol=2e-2)
    # the point clouds are exactly the reference's masking (gradio.py:147-151, :91-92) of this run's own scene, and a
    # scene reloaded from its pickle (no device copies) gives the same ones
    thr = demo.THRESHOLDS
    clouds = demo.get_3D_models_from_scene(scene, thr)
    reloaded = pickle.loads(pickle.dumps(scene))
    again = demo.get_3D_models_from_scene(reloaded, thr)
    for t, (p, c), (p2, c2) in zip(thr, clouds, again):
        msk = [(o["conf"] >= t).numpy() for o in scene.x_out]
        want_p = np.concatenate([o["pts3d"].numpy()[m] for o, m in zip(scene.x_out, msk)])
        want_c = np.concatenate([im[m] for im, m in zip(scene.imgs, msk)])
        assert np.array_equal(p, want_p) and np.array_equal(c, want_c), t
        assert np.array_equal(p2, want_p) and np.array_equal(c2, want_c), t
    pl = demo.get_3D_model_from_scene(None, False, scene, min_conf_thr=2.0, as_pointcloud=True, local_pointmaps=True)
    msk = [(o["conf"] >= 2.0).numpy() for o in scene.x_out]
    want = np.concatenate([(o["pts3d_local"].double() @ m[:3, :3].double().T + m[:3, 3].double()).numpy()[k]
                           for o, m, k in zip(scene.x_out, scene.cams2world, msk)])
    np.testing.assert_allclose(pl[0], want, rtol=1e-5, atol=1e-5)


def test_vidseq_syncs_only_where_the_engine_does(files, model, monkeypatch):
    """A vidseq run adds no synchronising call of its own to the engine's schedule: inside the demo it makes no more than
    inference_video_multi_ar run alone with the same keyframe rule and max_bs on the same views (on an H100, 16 against
    17: the engine's own up-front encoder batches and per-step postprocess)."""
    _, paths = files
    views = demo.load_images(paths, size=mk.IMAGE_SIZE, verbose=False)
    imgs = [v["img"] for v in views]
    ts = [torch.from_numpy(v["true_shape"]) for v in views]
    pp = lambda x: demo.postprocess(x, compute_cam=True)      # noqa: E731
    torch.cuda.synchronize()

    def syncs(fn):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                fn()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        return sum("synchroniz" in str(x.message) for x in w)

    def engine():
        return demo.inference_video_multi_ar(model[0], model[1], imgs, ts, demo._mem_batches(len(paths), 2, 1, len(paths),
                                             len(paths)), max_bs=1, device="cuda", post_process_function=pp,
                                             local_context_size=3)
    engine()                               # one-time set-up (streams, tables) is not counted
    torch.cuda.synchronize()
    engine_alone = syncs(engine)
    calls = []
    orig = demo.inference_video_multi_ar

    def counted(*a, **k):
        out = []
        calls.append(syncs(lambda: out.append(orig(*a, **k))))
        return out[0]
    monkeypatch.setattr(demo, "inference_video_multi_ar", counted)
    demo.must3r_inference_video(model, "cuda", mk.IMAGE_SIZE, False, paths, 1, 2, 1, local_context_size=3,
                                is_keyframe_function=lambda id, res, scene_state: id % 3 == 0, verbose=False)
    assert len(calls) == 1 and calls[0] <= engine_alone, (calls, engine_alone)


def test_reconstruct_cli(files, tmp_path):
    chkpt, paths = files
    img_dir = os.path.dirname(paths[0])
    out = tmp_path / "out"
    r = subprocess.run([sys.executable, "-m", "must3r_b200.reconstruct", "--weights", chkpt, "--image_dir", img_dir,
                        "--output", str(out), "--image_size", "224", "--num_mem_imgs", "4"], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    with open(out / "scene.pkl", "rb") as f:
        scene = pickle.load(f)
    assert len(scene.x_out) == len(paths)
    sys.path.insert(0, HERE)
    from test_demo_cpu import read_ply
    for thr in demo.THRESHOLDS:
        p, c = read_ply(str(out / f"scene_{thr}.ply"))
        want, want_c = demo.get_3D_model_from_scene(None, False, scene, min_conf_thr=thr, as_pointcloud=True)
        assert p.shape[0] == want.shape[0] and np.array_equal(p, want), thr
        assert np.array_equal(c, np.rint(want_c * 255).astype(np.uint8)), thr
