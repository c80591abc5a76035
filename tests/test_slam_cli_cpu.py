"""Host-side logic of `python -m must3r_b200.slam` (must3r_b200/slam.py, must3r_b200/engine/frames.py): the parser, the
rejected inputs, the frame sequencing against the reference's own loaders and headless main (oracle/_ref, with the
stand-ins of tests/golden/make_slam_cli_golden.py), the memory file naming, and the golden's reproduction."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest

from must3r_b200 import slam as cli
from must3r_b200.engine import frames

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_slam_cli_golden as mkc  # noqa: E402


@pytest.fixture(scope="module")
def ref():
    """The reference's slam.py and data.py from oracle/_ref (cv2 / open3d / roma stand-ins installed)."""
    if not os.path.isfile(os.path.join(REF, "must3r", "slam", "slam.py")):
        pytest.skip("no reference under oracle/_ref")
    saved = {k: sys.modules.get(k) for k in ("cv2", "open3d", "open3d.visualization", "open3d.visualization.gui",
                                             "open3d.visualization.rendering", "roma")}
    sys.path.insert(0, REF)
    mkc.install_stubs()
    import must3r.slam.data as ref_data
    import must3r.slam.slam as ref_slam
    yield ref_slam, ref_data
    for k, v in saved.items():
        if v is None:
            sys.modules.pop(k, None)
        else:
            sys.modules[k] = v


def _reference_parser(ref_slam, monkeypatch):
    """The parser built inside the reference's main (stopped at parse_args)."""
    class Got(Exception):
        pass

    def grab(self, *a, **k):
        raise Got(self)
    monkeypatch.setattr(argparse.ArgumentParser, "parse_args", grab)
    with pytest.raises(Got) as e:
        ref_slam.main()
    monkeypatch.undo()
    return e.value.args[0]


def _actions(parser):
    return {a.dest: (a.option_strings, a.default, a.nargs, a.type, a.choices, a.required, type(a).__name__)
            for a in parser._actions if a.dest != "help"}


def test_parser_names_and_defaults_are_the_references(ref, monkeypatch):
    want = _actions(_reference_parser(ref[0], monkeypatch))
    assert _actions(cli.get_args_parser()) == want


def test_parser_defaults():
    a = cli.parse_args(["--chkpt", "c", "--input", HERE, "--output", "o"])
    assert (a.device, a.res, a.skip_every, a.subsamp, a.keyframe_overlap_thr, a.min_conf_keyframe, a.overlap_percentile,
            a.num_init_frames, a.rerender_bs) == ("cuda:0", 224, 1, 2, .1, 1.2, 85., 2, 64)
    assert (a.searcher, a.overlap_mode, a.force_first_keyframes, a.viz_conf) == ("kdtree-scipy-quadrant_x2", "nn-norm", None, 4.)


@pytest.mark.parametrize("case, message", [
    ("gui", "--gui is not supported"),
    ("no_output", "--output is required"),
    ("camera", "camera streams are not supported"),
    ("video", "video files are not supported"),
    ("missing", "no such folder"),
    ("cpu", "runs on CUDA devices only"),
])
def test_rejected_with_a_message(case, message, tmp_path, capsys):
    video = tmp_path / "clip.mp4"
    video.write_bytes(b"\0")
    inp = {"camera": "cam:0", "video": str(video), "missing": str(tmp_path / "nope")}.get(case, str(tmp_path))
    argv = ["--chkpt", "c", "--input", inp]
    argv += [] if case == "no_output" else ["--output", str(tmp_path / "o")]
    argv += {"gui": ["--gui"], "cpu": ["--device", "cpu"]}.get(case, [])
    with pytest.raises(SystemExit) as e:
        cli.parse_args(argv)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_cli_rejects_before_loading_anything(tmp_path):
    r = subprocess.run([sys.executable, "-m", "must3r_b200.slam", "--chkpt", "missing.pth", "--input", str(tmp_path),
                        "--output", str(tmp_path / "out"), "--gui"], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 2 and "--gui is not supported" in r.stderr
    assert not (tmp_path / "out").exists()


def _folders(tmp_path, lengths):
    """One folder per length with tiny PNG frames whose pixel [0, 0] encodes (folder, index), plus decoys."""
    import PIL.Image
    dirs = []
    for s, n in enumerate(lengths):
        d = tmp_path / f"src{s}"
        d.mkdir()
        for i in range(n):
            PIL.Image.fromarray(np.full((2, 3, 3), (s, i, 7), np.uint8)).save(d / f"img_{i:03d}.png")
        for decoy in ("notes.txt", "img_000.png.bak", "Thumbs.db"):
            (d / decoy).write_text("x")
        dirs.append(str(d))
    return dirs


def _tag(frame):
    return None if frame is None else (int(frame[0, 0, 0]), int(frame[0, 0, 1]))


def _path_tag(path):
    return None if path is None else (int(os.path.basename(os.path.dirname(path))[3:]), int(path[-7:-4]))


def test_list_frames_filters(tmp_path):
    for n in ("b.PNG", "a.jpg", "c.png.bak", "notes.txt", "d.tiff", "x_frame.webp", "frame_list.txt"):
        (tmp_path / n).write_text("")
    assert frames.list_frames(str(tmp_path)) == ["a.jpg", "b.PNG", "d.tiff", "x_frame.webp"]
    assert frames.list_frames(str(tmp_path), "frame") == ["x_frame.webp"]


@pytest.mark.parametrize("lengths", [[5], [4, 2], [3, 5, 1], [2, 2, 3]])
@pytest.mark.parametrize("skip", [1, 2, 3])
def test_reads_and_grabs_match_the_reference(ref, lengths, skip, tmp_path, monkeypatch):
    """grab_frame with skip_every - 1 grabs after each read, on 1-3 folders of unequal lengths, past the end."""
    ref_slam, ref_data = ref
    dirs = _folders(tmp_path, lengths)
    monkeypatch.setattr(ref_slam, "SKIP_EVERY", skip)
    rcam = ref_data.AutoMultiLoader(dirs)
    mcam = frames.AutoMultiLoader(dirs)
    assert len(mcam) == len(rcam) == sum(lengths)
    for _ in range(sum(lengths) + 3):
        f, rc = ref_slam.grab_frame(rcam)
        p, mc = frames.grab_frame(mcam, skip)
        assert (_path_tag(p), mc) == (_tag(f), rc)


def _reference_run(ref_slam, argv, monkeypatch):
    """The reference's headless main with a SLAM_MUSt3R that records its arguments and calls."""
    rec = {"calls": []}

    class Recorder:
        def __init__(self, **kw):
            rec["kw"] = kw

        def __call__(self, frame, frame_id, cam_id):
            rec["calls"].append((_tag(frame), cam_id, frame_id))

        def write_all_poses(self, path, **kw):
            rec["poses"] = (os.path.basename(path), kw)

        def save_memory(self, path):
            rec["memory"] = path
    monkeypatch.setattr(ref_slam, "SLAM_MUSt3R", Recorder)
    monkeypatch.setattr(sys, "argv", ["slam.py"] + argv)
    ref_slam.main()
    return rec


@pytest.mark.parametrize("lengths", [[5], [4, 2], [3, 5, 1]])
@pytest.mark.parametrize("skip", [1, 2, 3])
def test_schedule_matches_the_reference_main(ref, lengths, skip, tmp_path, monkeypatch):
    """(frame, cam_id, timestamp) fed to the model, the frame sizes recorded, the model's arguments and the output
    names: must3r_b200.slam against the reference's main itself."""
    dirs = _folders(tmp_path, lengths)
    argv = ["--chkpt", "c.pth", "--input"] + dirs + ["--output", str(tmp_path / "out"), "--skip_every", str(skip),
                                                     "--subsamp", "3", "--varying_focals", "--filter"]
    want = _reference_run(ref[0], argv, monkeypatch)
    items, trailing = frames.schedule(frames.AutoMultiLoader(dirs), skip)
    assert [(_path_tag(p), c, t) for p, c, t in items] == want["calls"]
    got = {}
    monkeypatch.setattr(cli, "SLAM_MUSt3R", lambda **kw: got.update(kw))
    monkeypatch.setattr(cli, "AutoMultiLoader", lambda *a: (_ for _ in ()).throw(StopIteration))
    with pytest.raises(StopIteration):
        cli.main(argv)
    assert {**got, "device": "cuda:0"} == {**want["kw"], "device": "cuda:0"}
    # the sizes the reference records: every frame fed, then the one read after the last if any
    hw = [(2, 3)] * (len(items) + (trailing is not None))
    assert np.array_equal(np.array(hw), np.array(want["poses"][1]["imgHWs"]))
    assert want["poses"][0] == os.path.basename(
        f"all_poses{cli.FILTERING_MODE}_{cli.FILTERING_STEPS}-steps_{cli.FILTERING_ALPHA}-alpha.npz")
    assert {k: want["poses"][1][k] for k in ("filtering_mode", "filtering_steps", "filtering_alpha")} == dict(
        filtering_mode=cli.FILTERING_MODE, filtering_steps=cli.FILTERING_STEPS, filtering_alpha=cli.FILTERING_ALPHA)


def test_memory_file_naming(tmp_path):
    out = str(tmp_path)
    mem = os.path.join(out, "memory.pkl")
    assert cli.memory_path(out) == mem
    assert cli.memory_path(out, os.path.join(out, "other.pkl")) == mem
    assert cli.memory_path(out, "/elsewhere/memory.pkl") == mem
    assert cli.memory_path(out, mem) == os.path.join(out, "memory_0.pkl")
    assert cli.memory_path(out, os.path.join(out, ".", "memory.pkl")) == os.path.join(out, "memory_0.pkl")
    for c in (0, 1):
        open(os.path.join(out, f"memory_{c}.pkl"), "w").close()
    assert cli.memory_path(out, mem) == os.path.join(out, "memory_2.pkl")


def test_golden_reproduces_from_the_reference():
    from oracle.install_reference import source
    if source() is None:
        pytest.skip("no reference checkout")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_slam_cli_golden.py"), "--check"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "reproduced" in r.stdout
