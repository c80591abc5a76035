"""Several videos on one GPU (must3r_b200/engine/videos.py): the in-place compaction (m3r_mem_compact_rows) against
sequential torch edits, then whole videos against get_reconstructed_scene run alone on each of them and against the
reference's run (tests/golden/demo.npz), other precisions, the host synchronisations of a batched run, and
`python -m must3r_b200.reconstruct_videos` against `python -m must3r_b200.reconstruct` per folder."""
import ctypes as C
import os
import pickle
import shutil
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from must3r_b200 import _lib
from must3r_b200 import synthetic as syn
from must3r_b200.engine import demo, videos
from must3r_b200.engine.slam_sessions import SessionArena
from must3r_b200.model import common as cm
from must3r_b200.model import load_model

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_demo_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 3e-3, torch.bfloat16: 2.5e-2}        # tests/test_reconstruct_scenes_gpu.py
TOL[torch.float8_e4m3fn] = TOL[torch.bfloat16]


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(HERE, "golden", "demo.npz"))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("videos")
    chkpt = str(d / "tiny.pth")
    mk.mk.write_checkpoint(chkpt)
    img_dir = d / "images"
    img_dir.mkdir()
    return chkpt, mk.write_images(str(img_dir))


@pytest.fixture(scope="module")
def model(files):
    m = load_model(files[0], device="cuda", img_size=mk.IMAGE_SIZE, verbose=False)
    assert m[1].memory_mode == "kv"
    return m


@pytest.fixture
def precision():
    prev = cm.get_precision()
    yield cm.set_precision
    cm.set_precision(prev)


# ------------------------------------------------------------------------------------------------ compaction kernel
def compact(arena, base, runs, cap, B=None, width=None, ptrs=None):
    lib = _lib.lib()
    a = (C.c_void_p * len(arena))(*(ptrs or [t.data_ptr() for t in arena]))
    B = len(base) if B is None else B
    off, flat = [0], []
    for rs in runs:
        flat += [v for r in rs for v in r]
        off.append(off[-1] + len(rs))
    return lib.m3r_mem_compact_rows(a, len(arena), B, arena[0].shape[-1] if width is None else width, cap,
                                    (C.c_int64 * max(1, len(base)))(*base), (C.c_int32 * len(off))(*off),
                                    (C.c_int32 * max(1, len(flat)))(*flat), cm.stream_ptr(torch.device("cuda")))


def runs_of_holes(length, holes):
    """The kept runs (src_row, dst_row, rows) of rows [0, length) without the hole ranges [a, b) (shift-0 runs kept)."""
    keep = np.ones(length, bool)
    for a, b in holes:
        keep[a:b] = False
    edges = np.flatnonzero(np.diff(np.concatenate(([False], keep, [False])).astype(np.int8)))
    runs, pos = [], 0
    for a, b in zip(edges[0::2].tolist(), edges[1::2].tolist()):
        runs.append((a, pos, b - a))
        pos += b - a
    return runs


def check_compaction(dtype, S, cap, width, runs_per_slot, slots, depth=2, seed=0):
    """m3r_mem_compact_rows of runs_per_slot[i] in slot slots[i] against the runs applied one by one with clone(); every
    other row and slot keeps its random bits."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    arena = [torch.randint(-32768, 32767, (S, cap, width), dtype=torch.int16, device="cuda", generator=gen).view(dtype)
             for _ in range(depth)]
    want = [a.clone() for a in arena]
    for w in want:
        for s, rs in zip(slots, runs_per_slot):
            for src, dst, n in rs:
                w[s, dst:dst + n] = w[s, src:src + n].clone()
    assert compact(arena, [s * cap for s in slots], runs_per_slot, cap) == 0, _lib.lib().m3r_last_error()
    torch.cuda.synchronize()
    for a, w in zip(arena, want):
        assert torch.equal(a.view(torch.int16), w.view(torch.int16))


CASES = {
    "hole_shorter_than_the_rows_behind": [[(300, 100, 2000)]],
    "adjacent_holes": [runs_of_holes(1500, [(100, 150), (160, 210)])],
    "growing_shifts": [runs_of_holes(3000, [(100, 110), (160, 190), (250, 340), (900, 1400)])],
    "hole_at_the_end_and_at_row_0": [runs_of_holes(768, [(500, 768)]), runs_of_holes(2304, [(0, 768)])],
    "shift_of_one_row": [[(101, 100, 2500)]],
}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
@pytest.mark.parametrize("case", list(CASES))
def test_compaction_is_sequential_clone(dtype, case):
    runs = CASES[case]
    S = len(runs) + 2
    check_compaction(dtype, S, 3200, 1536, runs, [1 + i for i in range(len(runs))])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_compaction_of_64_slots(dtype):
    """64 slots (the most one launch takes), each with its own random holes, at a narrow and the full memory width."""
    rng = np.random.default_rng(1)
    cap = 900
    runs = []
    for s in range(64):
        length = int(rng.integers(1, cap))
        holes = [tuple(sorted(rng.integers(0, length, 2).tolist())) for _ in range(int(rng.integers(0, 4)))]
        runs.append(runs_of_holes(length, holes))
    runs = [rs[:128 // 64] for rs in runs]             # at most M3R_MAX_COMPACT_RUNS in all
    for width in (24, 1536):
        check_compaction(dtype, 64, cap, width, runs, list(range(64)), seed=width)


def test_compaction_runs_past_one_launch():
    """videos._compact_rows cuts 300 runs of one scene and 5 of another over launches; the result is the sequential one."""
    arena = SessionArena(3, 2, 64, torch.float16, "cuda")
    arena.ensure(4000)
    for b in arena.bufs:
        b.copy_(torch.randint(-32768, 32767, b.shape, dtype=torch.int16, device="cuda").view(torch.float16))
    want = [b.clone() for b in arena.bufs]
    runs_of = {0: runs_of_holes(3000, [(10 * k, 10 * k + 3) for k in range(300)]), 2: runs_of_holes(400, [(5, 9)] * 5)}
    for w in want:
        for s, rs in runs_of.items():
            for src, dst, n in rs:
                w[s, dst:dst + n] = w[s, src:src + n].clone()
    videos._compact_rows(arena, runs_of, cm.stream_ptr(torch.device("cuda")))
    torch.cuda.synchronize()
    for a, w in zip(arena.bufs, want):
        assert torch.equal(a.view(torch.int16), w.view(torch.int16))


def test_compaction_argument_errors():
    cap = 64
    arena = [torch.zeros((4, cap, 32), dtype=torch.float16, device="cuda") for _ in range(2)]
    before = [a.clone() for a in arena]
    lib = _lib.lib()
    ok = [[(10, 5, 20)]]
    bad = {
        "null": dict(ptrs=[arena[0].data_ptr(), 0]),
        "aligned": dict(ptrs=[arena[0].data_ptr() + 2, arena[1].data_ptr()]),
        "dst_row <= src_row": dict(runs=[[(5, 10, 20)]]),
        "cap": dict(runs=[[(50, 40, 20)]]),
        "order": dict(runs=[[(20, 10, 5), (22, 15, 5)]]),
        "multiple of 8": dict(width=30),
        "B in": dict(B=65, base=[64 * s for s in range(65)], runs=[[]] * 65),
        "cap apart": dict(base=[0, 10], runs=[[(10, 5, 2)], []]),
        "run_offset": dict(runs=[[(2 * k + 1, k, 1) for k in range(129)]], base=[0], cap=1000),
    }
    for msg, kw in bad.items():
        runs = kw.pop("runs", ok)
        base = kw.pop("base", [0] if len(runs) == 1 else [cap * s for s in range(len(runs))])
        c = kw.pop("cap", cap)
        rc = compact(arena, base, runs, c, **kw)
        assert rc != 0 and msg.encode() in lib.m3r_last_error(), (msg, lib.m3r_last_error())
    torch.cuda.synchronize()
    for a, b in zip(arena, before):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ engine
def four_videos(paths):
    """Eight frames (six landscape, two portrait), five landscape frames, a landscape and a portrait frame, one frame."""
    return [list(paths), list(paths[1:6]), list(paths[5:7]), [paths[7]]]


def alone(model, filelist, mode, context, refinements, thr, monkeypatch):
    """get_reconstructed_scene on one list -> (scene, keyframes as test_demo_gpu.py records them)."""
    keyframes = []
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
    try:
        scene, _ = demo.get_reconstructed_scene(
            None, None, False, model, None, "cuda", False, mk.IMAGE_SIZE, False, filelist, 1, refinements, mode,
            num_mem_images=4, render_once=False, vidseq_local_context_size=context, keyframe_interval=3,
            slam_local_context_size=context, subsample=2, min_conf_keyframe=1.5, keyframe_overlap_thr=thr,
            overlap_percentile=85.0, min_conf_thr=1.05, as_pointcloud=True, transparent_cams=False,
            local_pointmaps=False, cam_size=0.05)
    finally:
        monkeypatch.setattr(demo, "inference_video_multi_ar", orig)
    return scene, list(range(min(2, len(filelist)))) + keyframes


def batched(model, lists, mode, context, refinements, thr, monkeypatch, amp=False):
    """reconstruct_videos -> (scenes, each video's keyframes)."""
    plans = []

    class Recorded(videos.VideoPlan):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            plans.append(self)
    monkeypatch.setattr(videos, "VideoPlan", Recorded)
    try:
        got = videos.reconstruct_videos(model, "cuda", mk.IMAGE_SIZE, amp, lists, mode, 1, local_context_size=context,
                                        keyframe_overlap_thr=thr, num_refinements_iterations=refinements, verbose=False)
    finally:
        monkeypatch.setattr(videos, "VideoPlan", Recorded.__base__)
    return got, [p.keyframes for p in plans]


def assert_same_scene(got, want, tol):
    assert got.image_list == want.image_list
    assert len(got.x_out) == len(want.x_out)
    for o, w in zip(got.x_out, want.x_out):
        for k in ("pts3d", "pts3d_local", "conf"):
            assert not o[k].is_cuda and o[k].shape == w[k].shape
            assert rel(o[k], w[k]) < tol, k
    np.testing.assert_allclose(np.array(got.focals), np.array(want.focals), rtol=3e-2)
    np.testing.assert_allclose(np.stack([m.numpy() for m in got.cams2world]),
                               np.stack([m.numpy() for m in want.cams2world]), atol=3e-2)
    assert [tuple(t.tolist()) for t in got.true_shape] == [tuple(t.tolist()) for t in want.true_shape]
    for a, b in zip(got.imgs, want.imgs):
        assert np.array_equal(a, b)


def assert_bitwise(got, want):
    assert got.image_list == want.image_list and got.focals == want.focals
    for o, w in zip(got.x_out, want.x_out):
        for k in ("pts3d", "pts3d_local", "conf", "c2w"):
            assert torch.equal(o[k], w[k]), k


MODES = [("vidseq", 0, 0), ("vidseq", 3, 0), ("vidseq", 0, 1), ("vidseq", 3, 1), ("vidslam", 0, 0), ("vidslam", 0, 1)]
MODE_IDS = [f"{m}_window{c}_refine{r}" for m, c, r in MODES]


def threshold(mode, g):
    return float(g["vidslam_keyframe_overlap_thr"]) if mode == "vidslam" else 0.05


@pytest.mark.parametrize("mode,context,refinements", MODES, ids=MODE_IDS)
def test_videos_match_each_video_alone(files, model, g, mode, context, refinements, monkeypatch):
    _, paths = files
    lists = four_videos(paths)
    thr = threshold(mode, g)
    got, kfs = batched(model, lists, mode, context, refinements, thr, monkeypatch)
    assert len(got) == len(lists)
    for s, fl in enumerate(lists):
        want, want_kf = alone(model, fl, mode, context, refinements, thr, monkeypatch)
        assert kfs[s] == want_kf, s
        assert_same_scene(got[s], want, TOL[torch.float16])


@pytest.mark.parametrize("mode,context,refinements", [MODES[i] for i in (1, 3, 5)],
                         ids=[MODE_IDS[i] for i in (1, 3, 5)])
def test_one_video_batched_alone_is_bitwise_the_engine(files, model, g, mode, context, refinements, monkeypatch):
    """At S = 1 the memory rows, their order and every call are the single-video engine's: the results are bit for bit
    the same."""
    _, paths = files
    thr = threshold(mode, g)
    for fl in (list(paths), list(paths[5:7])):
        (got,), (kf,) = batched(model, [fl], mode, context, refinements, thr, monkeypatch)
        want, want_kf = alone(model, fl, mode, context, refinements, thr, monkeypatch)
        assert kf == want_kf
        assert_bitwise(got, want)


@pytest.mark.parametrize("name", ["vidseq", "vidslam"])
def test_videos_reproduce_the_reference(files, model, g, name, monkeypatch):
    """The golden's video between two others reproduces the reference's run (vidseq: window 3, so frames leave from the
    middle of the memory)."""
    _, paths = files
    kw = mk.CASES[name]
    context = kw.get("vidseq_local_context_size", kw.get("slam_local_context_size", 0))
    got, kfs = batched(model, [paths[:3], paths, paths[2:7]], name, context, 0, threshold(name, g), monkeypatch)
    scene = got[1]
    assert kfs[1] == g[f"{name}_keyframes"].tolist()
    assert [paths.index(p) for p in scene.image_list] == g[f"{name}_order"].tolist()
    for i, o in enumerate(scene.x_out):
        assert syn.rel_l2(o["pts3d"][::mk.SUB, ::mk.SUB], torch.from_numpy(g[f"{name}_pts3d_{i}"])) < 1.5e-3, i
        assert syn.rel_l2(o["conf"][::mk.SUB, ::mk.SUB], torch.from_numpy(g[f"{name}_conf_{i}"])) < 1.5e-3, i
    np.testing.assert_allclose(np.array(scene.focals), g[f"{name}_focal"], rtol=3e-2)
    np.testing.assert_allclose(np.stack([m.numpy() for m in scene.cams2world]), g[f"{name}_c2w"], atol=3e-2)
    clouds = demo.get_3D_models_from_scene(scene, g[f"{name}_thr"].tolist())
    assert [p.shape[0] for p, _ in clouds] == g[f"{name}_count"].tolist()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float8_e4m3fn], ids=["bf16", "fp8"])
def test_other_precisions_match_alone(files, model, dtype, precision, monkeypatch):
    _, paths = files
    precision(dtype)
    lists = [list(paths), list(paths[1:6])]
    got, kfs = batched(model, lists, "vidseq", 3, 0, 0.05, monkeypatch)
    for s, fl in enumerate(lists):
        want, want_kf = alone(model, fl, "vidseq", 3, 0, 0.05, monkeypatch)
        assert kfs[s] == want_kf
        assert_same_scene(got[s], want, TOL[dtype])


def cached_load(monkeypatch):
    loaded = {}

    def cached(filelist, image_size, encoder, verbose, device):
        key = tuple(filelist)
        if key not in loaded:
            loaded[key] = demo._load(filelist, image_size, encoder, verbose, device)
        return loaded[key]
    monkeypatch.setattr(videos, "_load", cached)


def test_vidseq_host_syncs_do_not_grow_with_the_video_count(files, model, monkeypatch):
    """A batched vidseq run of three landscape videos of different lengths, with frames leaving the middle of the memory,
    synchronises as often as a run of one (image loading, which is per video, is left out)."""
    _, paths = files
    land = paths[:6]
    cached_load(monkeypatch)

    def syncs(lists):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                videos.reconstruct_videos(model, "cuda", mk.IMAGE_SIZE, False, lists, "vidseq", 1, local_context_size=3,
                                          keyframe_interval=2, verbose=False)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        return sum("synchroniz" in str(x.message) for x in w)
    batched_lists = [land, land[:4], land[1:]]
    syncs(batched_lists)
    syncs([land])                          # one-time set-up (streams, tables, workspaces) is not counted
    one, three = syncs([land]), syncs(batched_lists)
    print(f"\n[videos] vidseq host synchronisations: 1 video {one}, 3 videos {three}")
    assert three == one, (one, three)


def test_vidslam_waits_once_per_step(files, model, g, monkeypatch):
    """The keyframe scores of every video's frame come back with one wait per step, whatever the number of videos."""
    _, paths = files
    cached_load(monkeypatch)
    waits = []
    real = videos._wait_scores

    def counted():
        waits.append(1)
        real()
    monkeypatch.setattr(videos, "_wait_scores", counted)
    land = paths[:6]
    counts = []
    for lists in ([land], [land, land[:4], land[1:]]):
        waits.clear()
        videos.reconstruct_videos(model, "cuda", mk.IMAGE_SIZE, False, lists, "vidslam", 1,
                                  keyframe_overlap_thr=threshold("vidslam", g), verbose=False)
        counts.append(len(waits))
    assert counts == [len(land) - 2] * 2, counts


def test_engine_refuses_other_memory_modes(files, model):
    dec = model[1]
    dec.change_memory_mode("norm_y")
    try:
        with pytest.raises(NotImplementedError, match="kv"):
            videos.reconstruct_videos(model, "cuda", mk.IMAGE_SIZE, False, [files[1][:2]], "vidseq", 1, verbose=False)
    finally:
        dec.change_memory_mode("kv")


# ------------------------------------------------------------------------------------------------ command line
@pytest.mark.parametrize("mode", ["vidseq", "vidslam"])
def test_cli_matches_reconstruct_per_folder(files, g, tmp_path, mode):
    chkpt, paths = files
    sys.path.insert(0, HERE)
    from test_demo_cpu import read_ply
    dirs = []
    for i, sel in enumerate([paths, paths[1:5]]):
        d = tmp_path / f"in{i}"
        d.mkdir()
        for p in sel:
            shutil.copy(p, d / os.path.basename(p))
        dirs.append(str(d))
    common = ["--weights", chkpt, "--image_size", "224", "--execution_mode", mode, "--local_context_size", "2"]
    r = subprocess.run([sys.executable, "-m", "must3r_b200.reconstruct_videos", "--scenes", *dirs,
                        "--output", str(tmp_path / "out")] + common, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for i, d in enumerate(dirs):
        ref_out = tmp_path / f"ref{i}"
        r = subprocess.run([sys.executable, "-m", "must3r_b200.reconstruct", "--image_dir", d, "--output", str(ref_out)]
                           + common, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        out = tmp_path / "out" / f"scene_{i}"
        assert sorted(os.listdir(out)) == sorted(os.listdir(ref_out))
        with open(out / "scene.pkl", "rb") as f:
            got = pickle.load(f)
        with open(ref_out / "scene.pkl", "rb") as f:
            want = pickle.load(f)
        assert_same_scene(got, want, TOL[torch.float16])
        for thr in demo.THRESHOLDS:
            p, _ = read_ply(str(out / f"scene_{thr}.ply"))
            q, _ = read_ply(str(ref_out / f"scene_{thr}.ply"))
            assert abs(p.shape[0] - q.shape[0]) <= max(2, 1e-3 * q.shape[0]), (i, thr, p.shape[0], q.shape[0])
