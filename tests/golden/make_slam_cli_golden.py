#!/usr/bin/env python
"""Generate tests/golden/slam_cli.npz by running the UNMODIFIED reference's headless SLAM command line
(must3r/slam/slam.py:main, with a patched sys.argv) on the CPU in fp32 (--device cpu).  Needs a reference checkout
(oracle/install_reference.py finds it):

    python tests/golden/make_slam_cli_golden.py [--check]

--check regenerates the arrays and compares them with the stored file instead of writing it.

The model is make_slam_golden.py's tiny random checkpoint, `roma` its stand-in.  slam.py imports cv2 and open3d at
module level: `cv2` gets a stand-in whose imread decodes with PIL and returns BGR (what cv2.imread returns for PNG),
with cvtColor, VideoCapture and the CAP_PROP_* constants; `open3d` gets empty modules (the GUI is never started).
A subclass of the reference's SLAM_MUSt3R that only records each instance, and a wrapper of postproc_pred that only
records each frame's overlap score and median confidence, observe the run.

Frames are seeded PNG crops of make_slam_golden.py's sliding panorama, with decoy files that the extension and
--image_string filters must skip.  Runs (RUNS):
  * a: one folder, --res 224 --skip_every 2 --rerender --filter;
  * b: two folders of different frame sizes and lengths (two agents), --varying_focals;
  * c: a's memory.pkl passed back with --load_memory.
Each stores the poses file's arrays except fps and gpumem (the focal dict as one array per agent), the keyframe list,
the argument list, and of memory.pkl: the shape of each memory level, the labels, the counters, the number of keyframe
point maps with their point counts, and a float64 digest (sum, sum of |x|, sum of squares) of each level.  Each run's
keyframe_overlap_thr and min_conf_keyframe are the first of THRESHOLDS / MIN_CONFS that every overlap score and median
confidence of the run clears by MARGIN (relative); the script asserts it.
"""
import argparse
import contextlib
import os
import pickle
import shutil
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_slam_golden as mk  # noqa: E402

MARGIN = 0.05
THRESHOLDS = [0.1, 0.08, 0.12, 0.06, 0.15, 0.05, 0.2, 0.04, 0.3]
MIN_CONFS = [1.2, 1.3, 1.1, 1.5, 1.05]
IMAGE_STRING = "frame"
DECOYS = ["notes.txt", "frame_list.txt", "mask_000.png", "frame_000.png.bak", "Thumbs.db"]
# run -> (folders, arguments besides --chkpt / --device / --input / --output / thresholds); folders are written by
# write_folders, "@a" is run a's output directory
RUNS = {
    "a": (["seq"], ["--res", "224", "--image_string", IMAGE_STRING, "--skip_every", "2", "--rerender", "--filter"]),
    "b": (["cam0", "cam1"], ["--res", "224", "--image_string", IMAGE_STRING, "--varying_focals"]),
    "c": (["seq"], ["--res", "224", "--image_string", IMAGE_STRING, "--load_memory", "@a/memory.pkl"]),
}
POSES = {"a": "all_poseslaplacian_256-steps_0.1-alpha.npz", "b": "all_poses.npz", "c": "all_poses.npz"}


def write_folders(d):
    """The frame folders of RUNS under d: 'seq' (12 frames 240x320), 'cam0' (7 frames 240x320), 'cam1' (4 frames
    192x256, upper-case extension), each with the decoys."""
    import PIL.Image
    spec = {"seq": (mk.frames(), ".png"), "cam0": (mk.frames(7, seed=5), ".png"),
            "cam1": (mk.frames(4, seed=6, H=192, W=256, step=16), ".PNG")}
    for name, (imgs, ext) in spec.items():
        os.makedirs(os.path.join(d, name), exist_ok=True)
        for i, im in enumerate(imgs):
            PIL.Image.fromarray(im).save(os.path.join(d, name, f"{IMAGE_STRING}_{i:03d}{ext}"))
        for n in DECOYS:
            p = os.path.join(d, name, n)
            if n.endswith(".png"):
                PIL.Image.fromarray(imgs[0][::-1].copy()).save(p)
            else:
                open(p, "w").write("not a frame\n")
    return {n: os.path.join(d, n) for n in spec}


def argv_of(run, folders, outdir, chkpt, device, thr, min_conf):
    """The command line of one run (without the program name)."""
    dirs, extra = RUNS[run]
    extra = [x.replace("@a", outdir("a")) for x in extra]
    return (["--chkpt", chkpt, "--device", device, "--input"] + [folders[f] for f in dirs] + ["--output", outdir(run)]
            + extra + ["--keyframe_overlap_thr", str(thr), "--min_conf_keyframe", str(min_conf)])


# --------------------------------------------------------------------------------------------- stand-ins
def install_stubs():
    """cv2 and open3d stand-ins (and make_slam_golden.py's roma) in sys.modules."""
    mk._install_roma()
    cv2 = types.ModuleType("cv2")
    cv2.COLOR_BGR2RGB = 4
    cv2.CAP_PROP_POS_FRAMES = 1
    cv2.CAP_PROP_FRAME_COUNT = 7
    cv2.IMREAD_COLOR, cv2.IMREAD_ANYDEPTH = 1, 2        # dust3r/utils/image.py reads them at import

    def imread(path, flags=1):
        assert flags == cv2.IMREAD_COLOR
        import PIL.Image
        try:
            with PIL.Image.open(path) as im:
                return np.ascontiguousarray(np.asarray(im.convert("RGB"))[..., ::-1])
        except OSError:
            return None

    def cvtColor(img, code):
        assert code == cv2.COLOR_BGR2RGB
        return np.ascontiguousarray(img[..., ::-1])

    class VideoCapture:
        def __init__(self, *a, **k):
            raise NotImplementedError("cv2 stand-in: no video")

    cv2.imread, cv2.cvtColor, cv2.VideoCapture = imread, cvtColor, VideoCapture
    sys.modules["cv2"] = cv2
    o3d = types.ModuleType("open3d")
    vis = types.ModuleType("open3d.visualization")
    vis.gui = types.ModuleType("open3d.visualization.gui")
    vis.rendering = types.ModuleType("open3d.visualization.rendering")
    o3d.visualization, o3d.cpu = vis, types.SimpleNamespace()
    sys.modules.update({"open3d": o3d, "open3d.visualization": vis, "open3d.visualization.gui": vis.gui,
                        "open3d.visualization.rendering": vis.rendering})


def import_reference():
    from oracle.install_reference import source
    ref = source()
    assert ref is not None, "no reference checkout found (set MUST3R_REFERENCE)"
    if ref not in sys.path:
        sys.path.insert(0, ref)
    install_stubs()
    import must3r.slam.model as ref_model
    import must3r.slam.slam as ref_slam
    return ref_model, ref_slam


@contextlib.contextmanager
def observed(ref_model, ref_slam):
    """Record every SLAM_MUSt3R built by main and every frame's (overlap score, median confidence, first-frame flag)."""
    rec = {"instances": [], "calls": []}
    orig_cls, orig_pp = ref_slam.SLAM_MUSt3R, ref_model.postproc_pred

    class Recorded(orig_cls):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            rec["instances"].append(self)

    def recording_postproc_pred(img, res, is_first_frame, *a, **k):
        out = orig_pp(img, res, is_first_frame, *a, **k)
        rec["calls"].append((float(res["overlap_score"]), float(res["conf"][0, 0].median()), bool(is_first_frame)))
        return out

    ref_slam.SLAM_MUSt3R, ref_model.postproc_pred = Recorded, recording_postproc_pred
    try:
        yield rec
    finally:
        ref_slam.SLAM_MUSt3R, ref_model.postproc_pred = orig_cls, orig_pp


def memory_record(path):
    """Shapes, labels, counters, keyframe point maps and a float64 digest of each level of a memory.pkl."""
    with open(path, "rb") as f:
        mem, data, _ = pickle.load(f)
    vals, labels = mem[0], mem[1]
    out = {"mem_shapes": np.array([list(v.shape) for v in vals]), "mem_labels": labels.cpu().numpy().astype(np.int64),
           "mem_counters": np.array([int(x) for x in mem[2:]]),
           "mem_digest": np.array([[v.double().sum().item(), v.double().abs().sum().item(), v.double().square().sum().item()]
                                   for v in vals]),
           "kf_points": np.array([int(np.prod(p.shape[:-1])) for p, _, _ in data], dtype=np.int64).reshape(-1)}
    return out


def record(run, outdir, slam, argv):
    z = np.load(os.path.join(outdir, POSES[run]), allow_pickle=True)
    out = {k: z[k] for k in z.files if k not in ("fps", "gpumem", "focal")}
    for agid, f in z["focal"].item().items():
        out[f"focal_{agid}"] = np.asarray(f, dtype=np.float64).reshape(-1)
    out["keyframes"] = np.array(slam.keyframes, dtype=np.int64)
    out["argv"] = np.array(argv)
    out.update(memory_record(os.path.join(outdir, "memory.pkl")))
    return {f"{run}_{k}": v for k, v in out.items()}


def run_reference(ref_model, ref_slam, argv):
    old = sys.argv
    sys.argv = ["slam.py"] + argv
    try:
        with observed(ref_model, ref_slam) as rec:
            ref_slam.main()
    finally:
        sys.argv = old
    assert len(rec["instances"]) == 1
    return rec["instances"][0], rec["calls"]


def generate(d):
    ref_model, ref_slam = import_reference()
    torch.set_grad_enabled(False)
    folders = write_folders(os.path.join(d, "frames"))
    chkpt = os.path.join(d, "tiny.pth")
    mk.write_checkpoint(chkpt)

    def outdir(run):
        return os.path.join(d, f"out_{run}")
    out = {}
    for run in RUNS:
        for thr in THRESHOLDS:
            for min_conf in MIN_CONFS:
                shutil.rmtree(outdir(run), ignore_errors=True)
                argv = argv_of(run, folders, outdir, chkpt, "cpu", thr, min_conf)
                slam, calls = run_reference(ref_model, ref_slam, argv)
                if all(abs(s - thr) >= MARGIN * thr and abs(m - min_conf) >= MARGIN * min_conf
                       for s, m, first in calls if not first):
                    break
            else:
                continue
            break
        else:
            raise AssertionError(f"run {run}: no threshold pair clears every score and median confidence by {MARGIN}")
        # paths are stored relative to the run's temporary directory
        rel = [a.replace(d + os.sep, "") for a in argv]
        out.update(record(run, outdir(run), slam, rel))
        print(run, "thr", thr, "min_conf", min_conf, "keyframes", slam.keyframes, "timestamps",
              out[f"{run}_timestamps"].tolist(), "scores", [round(s, 4) for s, _, _ in calls])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true", help="compare with the stored slam_cli.npz instead of writing it")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        out = generate(d)
    path = os.path.join(HERE, "slam_cli.npz")
    if args.check:
        g = np.load(path)
        assert sorted(g.files) == sorted(out), (sorted(g.files), sorted(out))
        for k, v in out.items():
            if v.dtype.kind in "iubU":
                assert np.array_equal(g[k], v), k
            else:
                np.testing.assert_allclose(g[k], v, rtol=1e-4, atol=1e-5, err_msg=k)
        print(path, "reproduced")
        return
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
