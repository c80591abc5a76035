"""Multi-camera SLAM without a GPU (must3r_b200/engine/slam_cameras.py, must3r_b200/slam_cameras.py): the step schedule
against the reference's loaders and main (oracle/_ref), the batching plan, the row arithmetic of the ordered keyframe
commit, and the command line against `python -m must3r_b200.slam`."""
import os
import subprocess
import sys

import numpy as np
import pytest

from must3r_b200 import slam as single
from must3r_b200 import slam_cameras as cli
from must3r_b200.engine import frames
from must3r_b200.engine.slam_cameras import commit_rows, steps_of
from must3r_b200.engine.lockstep import plan_batch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_slam_cli_golden as mkc  # noqa: E402


def _folders(tmp_path, lengths):
    """One folder per length with tiny PNG frames whose pixel [0, 0] encodes (folder, index)."""
    import PIL.Image
    dirs = []
    for s, n in enumerate(lengths):
        d = tmp_path / f"src{s}"
        d.mkdir()
        for i in range(n):
            PIL.Image.fromarray(np.full((2, 3, 3), (s, i, 7), np.uint8)).save(d / f"img_{i:03d}.png")
        dirs.append(str(d))
    return dirs


def _path_tag(path):
    return int(os.path.basename(os.path.dirname(path))[3:]), int(path[-7:-4])


# ------------------------------------------------------------------------------------------------ step schedule
@pytest.mark.parametrize("lengths", [[5], [4, 4], [4, 2], [3, 5, 1], [2, 2, 3], [1, 6, 2, 4]])
@pytest.mark.parametrize("skip", [1, 2])
def test_steps_are_the_next_frame_of_every_camera_left(lengths, skip, tmp_path):
    dirs = _folders(tmp_path, lengths)
    items, _ = frames.schedule(frames.AutoMultiLoader(dirs), skip)
    steps = steps_of(items)
    assert [it for st in steps for it in st] == items                  # the reference's order, timestamps untouched
    assert [t for _, _, t in items] == [k * skip for k in range(len(items))]
    used = [0] * len(lengths)
    for k, st in enumerate(steps):
        cams = [c for _, c, _ in st]
        left = [c for c, n in enumerate(lengths) if used[c] < n]
        # camera order, one frame of every camera that still has frames (the last step: those left within the frames
        # skip_every keeps)
        assert cams == (left if k < len(steps) - 1 else left[:len(cams)])
        for p, c, _ in st:
            assert _path_tag(p) == (c, used[c])
            used[c] += 1


@pytest.fixture(scope="module")
def ref():
    """The reference's slam.py and data.py from oracle/_ref (cv2 / open3d / roma stand-ins installed)."""
    if not os.path.isfile(os.path.join(REF, "must3r", "slam", "slam.py")):
        pytest.skip("no reference under oracle/_ref")
    saved = {k: sys.modules.get(k) for k in ("cv2", "open3d", "open3d.visualization", "open3d.visualization.gui",
                                             "open3d.visualization.rendering", "roma")}
    sys.path.insert(0, REF)
    mkc.install_stubs()
    import must3r.slam.slam as ref_slam
    yield ref_slam
    for k, v in saved.items():
        if v is None:
            sys.modules.pop(k, None)
        else:
            sys.modules[k] = v


@pytest.mark.parametrize("lengths", [[4, 4], [3, 5, 1], [1, 6, 2, 4]])
def test_step_order_is_the_reference_main(ref, lengths, tmp_path, monkeypatch):
    """The (frame, cam_id, timestamp) sequence of the reference's headless main, cut into steps, is what the command
    line feeds step by step."""
    dirs = _folders(tmp_path, lengths)
    calls = []

    class Recorder:
        def __init__(self, **kw):
            pass

        def __call__(self, frame, frame_id, cam_id):
            calls.append(((int(frame[0, 0, 0]), int(frame[0, 0, 1])), cam_id, frame_id))

        def write_all_poses(self, path, **kw):
            pass

        def save_memory(self, path):
            pass
    monkeypatch.setattr(ref, "SLAM_MUSt3R", Recorder)
    monkeypatch.setattr(sys, "argv", ["slam.py", "--chkpt", "c", "--input"] + dirs + ["--output", str(tmp_path / "o")])
    ref.main()
    items, _ = frames.schedule(frames.AutoMultiLoader(dirs), 1)
    got = [(_path_tag(p), c, t) for st in steps_of(items) for p, c, t in st]
    assert got == calls


# ------------------------------------------------------------------------------------------------ batching plan
def test_batching_plan():
    assert plan_batch({0: (384, 512), 1: (384, 512), 2: (512, 384)}) == ([0, 1], [2])
    assert plan_batch({0: (384, 512), 1: None, 2: (384, 512)}) == ([0, 2], [1])
    assert plan_batch({0: None, 1: None}) == ([], [0, 1])
    assert plan_batch({0: (160, 224), 1: (224, 224)}) == ([0], [1])     # a tie: the first shape
    assert plan_batch({3: (160, 224)}) == ([3], [])


# ------------------------------------------------------------------------------------------------ ordered commit rows
def _restated(keyframe, row0, N, depth=2, width=8, cap=64, seed=0):
    """The ordered commit applied to a numpy memory the way sequential m3r_mem_commit_rows calls would: frame after frame,
    a keyframe's rows at the current end."""
    rng = np.random.default_rng(seed)
    mem = rng.standard_normal((depth, cap, width))
    staged = rng.standard_normal((depth, len(keyframe), N, width))
    seq, n = mem.copy(), row0
    for k, kf in enumerate(keyframe):
        if kf:
            seq[:, n:n + N] = staged[:, k]
            n += N
    return mem, staged, seq, n


@pytest.mark.parametrize("keyframe", [[1, 1, 1, 1], [0, 0, 0, 0], [1, 0, 1, 0], [0, 1, 0, 1], [0, 0, 0, 1], [1], [0]])
def test_commit_rows_are_the_sequential_commits(keyframe):
    row0, N = 5, 3
    mem, staged, seq, n_seq = _restated(keyframe, row0, N)
    rows, n = commit_rows(keyframe, row0, N)
    assert n == n_seq
    out = mem.copy()
    for k, r in enumerate(rows):
        if r is not None:
            out[:, r:r + N] = staged[:, k]
    assert np.array_equal(out, seq)
    assert np.array_equal(out[:, n:], mem[:, n:])                       # nothing past the new length


# ------------------------------------------------------------------------------------------------ command line
def test_arguments_and_defaults_are_the_single_camera_commands(tmp_path):
    argv = ["--chkpt", "c", "--input", str(tmp_path), str(tmp_path), "--output", "o", "--res", "512", "--varying_focals"]
    assert vars(cli.parse_args(argv)) == vars(single.parse_args(argv))
    defaults = ["--chkpt", "c", "--input", str(tmp_path), "--output", "o"]
    assert vars(cli.parse_args(defaults)) == vars(single.parse_args(defaults))


@pytest.mark.parametrize("case, message", [
    ("rerender", "--rerender with several --input folders is not supported"),
    ("gui", "--gui is not supported"),
    ("camera", "camera streams are not supported"),
    ("cpu", "runs on CUDA devices only"),
    ("no_output", "--output is required"),
])
def test_rejected_with_a_message(case, message, tmp_path, capsys):
    inp = ["cam:0"] if case == "camera" else [str(tmp_path), str(tmp_path)]
    argv = ["--chkpt", "c", "--input"] + inp + ([] if case == "no_output" else ["--output", str(tmp_path / "o")])
    argv += {"rerender": ["--rerender"], "gui": ["--gui"], "cpu": ["--device", "cpu"]}.get(case, [])
    with pytest.raises(SystemExit) as e:
        cli.parse_args(argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_one_folder_may_rerender(tmp_path):
    assert cli.parse_args(["--chkpt", "c", "--input", str(tmp_path), "--output", "o", "--rerender"]).rerender


def test_cli_rejects_before_loading_anything(tmp_path):
    r = subprocess.run([sys.executable, "-m", "must3r_b200.slam_cameras", "--chkpt", "missing.pth", "--input", str(tmp_path),
                        str(tmp_path), "--output", str(tmp_path / "out"), "--rerender"], cwd=ROOT, capture_output=True,
                       text=True)
    assert r.returncode == 2 and "--rerender with several --input folders" in r.stderr
    assert not (tmp_path / "out").exists()


def test_main_builds_one_run_with_the_single_camera_arguments(tmp_path, monkeypatch):
    """The run gets SLAM_MUSt3R's arguments as `python -m must3r_b200.slam` passes them, one agent per folder."""
    dirs = _folders(tmp_path, [3, 2])
    argv = ["--chkpt", "c.pth", "--input"] + dirs + ["--output", str(tmp_path / "out"), "--subsamp", "3",
                                                     "--varying_focals"]
    got, want = {}, {}

    class Stop(Exception):
        pass

    def take(store):
        def build(*a, **kw):
            store.update(kw)
            store.update(dict(zip(("chkpt", "num_agents"), a)))
            raise Stop
        return build
    monkeypatch.setattr(cli, "MultiCameraSLAM", take(got))
    monkeypatch.setattr(single, "SLAM_MUSt3R", take(want))
    for m in (cli, single):
        with pytest.raises(Stop):
            m.main(argv)
    assert got.pop("num_agents") == want.pop("num_agents") == 2
    assert got == want


def test_golden_reproduces_from_the_reference():
    from oracle.install_reference import source
    if source() is None:
        pytest.skip("no reference checkout")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_slam_cameras_golden.py"), "--check"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "reproduced" in r.stdout
