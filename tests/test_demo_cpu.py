"""Host-side logic of the demo's inference layer (must3r_b200/engine/demo.py) and of `python -m must3r_b200.reconstruct`:
the memory schedule, keyframe choice, SceneState, argument handling and the PLY writer.  The reference's own run is
reproduced from tests/golden/make_demo_golden.py when a reference checkout is present."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from must3r_b200 import reconstruct
from must3r_b200.engine import demo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def read_ply(path):
    """The binary little-endian vertex list write_ply makes -> (pts [N,3] float32, rgb [N,3] uint8)."""
    with open(path, "rb") as f:
        data = f.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    assert header[:2] == ["ply", "format binary_little_endian 1.0"]
    n = int(next(line for line in header if line.startswith("element vertex")).split()[-1])
    props = [tuple(line.split()[1:]) for line in header if line.startswith("property")]
    assert props == [("float", "x"), ("float", "y"), ("float", "z"), ("uchar", "red"), ("uchar", "green"), ("uchar", "blue")]
    rec = np.frombuffer(data[end:], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"),
                                           ("blue", "u1")], count=n)
    assert len(data) == end + 15 * n
    return np.stack([rec["x"], rec["y"], rec["z"]], 1), np.stack([rec["red"], rec["green"], rec["blue"]], 1)


@pytest.mark.parametrize("nimgs,num_mem,init,bnv,want", [
    (10, 4, 2, 1, [2, 1, 1]),
    (10, 10, 2, 3, [2, 3, 3, 2]),
    (5, 1, 2, 1, [2]),                 # fewer memory images than the init batch: the init batch alone
    (200, 50, 2, 1, [2] + [1] * 48),
])
def test_mem_batches(nimgs, num_mem, init, bnv, want):
    """must3r_inference's schedule (inference.py:188-191)."""
    assert demo._mem_batches(nimgs, init, bnv, max(num_mem, init), num_mem) == want


@pytest.mark.parametrize("nimgs,init,bnv,want", [(8, 2, 1, [2, 1, 1, 1, 1, 1, 1]), (3, 5, 1, [3]), (7, 2, 3, [2, 3, 2])])
def test_video_mem_batches(nimgs, init, bnv, want):
    """must3r_inference_video's schedule (inference.py:282-285): every view, init_num_images first."""
    assert demo._mem_batches(nimgs, init, bnv, nimgs, nimgs) == want


@pytest.mark.parametrize("nimgs,num_mem,init", [(1, 1, 2), (3, 3, 5)])
def test_mem_batches_rejects_an_unreachable_memory(nimgs, num_mem, init):
    with pytest.raises(ValueError):        # the reference's loop would never end here
        demo._mem_batches(nimgs, init, 1, max(num_mem, init), num_mem)


def test_to_render():
    assert demo._to_render(False, 4, 8) is None
    assert demo._to_render(True, 4, 8) == [4, 5, 6, 7]
    assert demo._to_render(True, 8, 8) == []


@pytest.mark.parametrize("nimgs,num_mem", [(8, 4), (200, 50), (7, 7), (5, 1), (13, 6)])
def test_linspace_keyframes(nimgs, num_mem):
    kf = demo._linspace_keyframes(nimgs, num_mem)
    assert kf == np.linspace(0, nimgs - 1, num_mem, dtype=int).tolist()
    assert kf[0] == 0 and (num_mem == 1 or kf[-1] == nimgs - 1) and len(set(kf)) == num_mem


def test_golden_keyframes_are_linspace():
    g = np.load(os.path.join(HERE, "golden", "demo.npz"))
    for case in ("linseq_render", "linseq_once"):
        kf = g[f"{case}_keyframes"].tolist()
        assert kf == demo._linspace_keyframes(8, 4)
        rest = sorted(set(range(8)) - set(kf))
        assert g[f"{case}_order"].tolist() == kf + rest


def _scene():
    x_out = [{"pts3d": torch.randn(4, 6, 3), "pts3d_local": torch.randn(4, 6, 3), "conf": 1 + torch.rand(4, 6),
              "focal": torch.tensor(5.0), "c2w": torch.eye(4)} for _ in range(2)]
    return demo.SceneState(x_out, [np.random.rand(4, 6, 3).astype(np.float32) for _ in range(2)],
                           [torch.tensor([4, 6], dtype=torch.int32)] * 2, [5.0, 5.0], [torch.eye(4)] * 2, ["a", "b"])


def test_scene_state_fields_and_pickle():
    s = _scene()
    s._device = {"pts3d": [object()]}          # device copies are never written to scene.pkl
    for name in ("x_out", "imgs", "true_shape", "focals", "cams2world", "image_list"):
        assert hasattr(s, name)
    t = pickle.loads(pickle.dumps(s))
    assert not hasattr(t, "_device")
    assert t.image_list == ["a", "b"] and t.focals == [5.0, 5.0]
    assert torch.equal(t.x_out[1]["conf"], s.x_out[1]["conf"]) and np.array_equal(t.imgs[0], s.imgs[0])


def test_get_3D_model_rejects_what_needs_trimesh():
    s = _scene()
    with pytest.raises(NotImplementedError):
        demo.get_3D_model_from_scene("/nonexistent", False, s, as_pointcloud=False)
    with pytest.raises(NotImplementedError):
        demo.get_3D_model_from_scene("/nonexistent", False, s, as_pointcloud=True, filename="scene.glb")
    assert demo.get_3D_model_from_scene("/nonexistent", False, None) is None


def test_retrieval_and_viser_are_rejected():
    with pytest.raises(NotImplementedError, match="asmk"):
        demo.must3r_inference((None, None), "retrieval.pth", "cuda", 512, False, [], 1, 1, 2, 1, False, is_sequence=False)
    with pytest.raises(NotImplementedError, match="viser"):
        demo.must3r_inference_video((None, None), "cuda", 512, False, [], 1, 2, 1, viser_server=object())


def test_cli_arguments():
    a = reconstruct.parse_args(["--image_dir", "d", "--output", "o"])
    assert (a.execution_mode, a.num_mem_imgs, a.file_type, a.amp, a.image_size) == ("linseq", 50, "ply", False, 512)
    assert (a.subsample, a.min_conf_keyframe, a.keyframe_overlap_thr, a.overlap_percentile) == (2, 1.5, 0.05, 85)
    a = reconstruct.parse_args(["--image_dir", "d", "--output", "o", "--execution_mode", "vidslam", "--amp", "bf16",
                                "--local_context_size", "5", "--render_once"])
    assert a.execution_mode == "vidslam" and a.amp == "bf16" and a.local_context_size == 5 and a.render_once
    for bad in (["--retrieval", "r.pth"], ["--execution_mode", "retrieval"], ["--file_type", "glb"], ["--image_size", "384"]):
        with pytest.raises(SystemExit):
            reconstruct.parse_args(["--image_dir", "d", "--output", "o"] + bad)
    with pytest.raises(SystemExit):
        reconstruct.parse_args(["--output", "o"])


def test_cli_rejects_retrieval_before_loading_anything(tmp_path):
    r = subprocess.run([sys.executable, "-m", "must3r_b200.reconstruct", "--image_dir", str(tmp_path), "--output",
                        str(tmp_path / "out"), "--retrieval", "r.pth"], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 2 and "--retrieval is not supported" in r.stderr
    assert not (tmp_path / "out").exists()


def test_list_images_sorted_files_only(tmp_path):
    for n in ("b.png", "a.png", "c.jpg"):
        (tmp_path / n).write_bytes(b"")
    (tmp_path / "sub").mkdir()
    assert [os.path.basename(p) for p in reconstruct.list_images(str(tmp_path))] == ["a.png", "b.png", "c.jpg"]


def test_ply_round_trip(tmp_path):
    gen = np.random.default_rng(0)
    pts = gen.standard_normal((1000, 3)).astype(np.float32)
    pts[3] = [np.inf, -np.inf, 1e30]
    col = gen.random((1000, 3)).astype(np.float32)
    col[:4] = [[0, 1, 0.5], [1 / 255, 0.5 / 255, 1.5 / 255], [0.999, 0.001, 0.25], [254.5 / 255, 0, 1]]
    p = demo.write_ply(str(tmp_path / "c.ply"), pts, col)
    rp, rc = read_ply(p)
    assert np.array_equal(rp, pts)
    assert np.array_equal(rc, np.rint(col * 255).astype(np.uint8))
    assert rc[0].tolist() == [0, 255, 128] and rc[1].tolist() == [1, 0, 2]
    demo.write_ply(str(tmp_path / "e.ply"), np.zeros((0, 3)), np.zeros((0, 3)))
    rp, rc = read_ply(str(tmp_path / "e.ply"))
    assert rp.shape == (0, 3) and rc.shape == (0, 3)


def test_golden_reproduces_from_the_reference():
    from oracle.install_reference import source
    if source() is None:
        pytest.skip("no reference checkout")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_demo_golden.py"), "--check"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "reproduced" in r.stdout
