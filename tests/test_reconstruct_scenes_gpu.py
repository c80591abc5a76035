"""Several offline reconstructions on one GPU (must3r_b200/engine/scenes.py): the ragged render call
(m3r_decoder_render_ragged) and the partial commit (m3r_mem_commit_rows), then whole scenes against must3r_inference run
alone on each of them and against the reference's run (tests/golden/demo.npz), the host synchronisations of a batched
run, and `python -m must3r_b200.reconstruct_scenes` against `python -m must3r_b200.reconstruct` per folder."""
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
from must3r_b200.engine import demo, scenes
from must3r_b200.model import common as cm
from must3r_b200.model import load_model

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_demo_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 3e-3, torch.bfloat16: 2.5e-2}        # tests/test_slam_sessions_gpu.py
TOL[torch.float8_e4m3fn] = TOL[torch.bfloat16]             # fp8 runs the bf16 attention and memory
PRECISIONS = [torch.float16, torch.bfloat16, torch.float8_e4m3fn]


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    d = tmp_path_factory.mktemp("scenes")
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


@pytest.fixture(scope="module")
def feats(files, model):
    """Encoder features of the six landscape views (fp16 encoder; the decoder tests set their own precision)."""
    views = demo.load_images(files[1][:6], size=mk.IMAGE_SIZE, verbose=False)
    ts = torch.as_tensor(np.stack([v["true_shape"] for v in views]))
    assert bool((ts == ts[:1]).all())
    x, pos = model[0](torch.stack([v["img"] for v in views]), ts)
    return x, pos, tuple(int(v) for v in ts[0])


def shape(hw, B, n):
    return scenes._host_shape(hw, B, n)


def memories(dec, feats, n_views):
    """One memory per scene, scene b built from n_views[b] views, in a [B, cap, 2D] arena whose other rows are NaN."""
    x, pos, hw = feats
    mems, k = [], 0
    for n in n_views:
        idx = [(k + j) % 6 for j in range(n)]
        mem, _ = dec(x[idx][None], pos[idx][None], shape(hw, 1, n), None)
        mems.append(mem[0])
        k += 1
    lens = [m[0].shape[1] for m in mems]
    cap = max(lens) + 40
    arena = [torch.full((len(n_views), cap, 2 * dec.embed_dim), float("nan"), dtype=dec.memory_dtype(), device="cuda")
             for _ in range(dec.depth)]
    for b, m in enumerate(mems):
        for l in range(dec.depth):
            arena[l][b, :lens[b]] = m[l][0]
    return arena, lens


def queries(feats, B, n):
    x, pos, hw = feats
    idx = [(3 + j) % 6 for j in range(B * n)]
    return x[idx].view(B, n, *x.shape[1:]), pos[idx].view(B, n, *pos.shape[1:]), shape(hw, B, n)


@pytest.fixture
def precision():
    prev = cm.get_precision()
    yield cm.set_precision
    cm.set_precision(prev)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dtype", PRECISIONS, ids=["fp16", "bf16", "fp8"])
def test_render_tokens_equal_lengths_is_forward_render(model, feats, dtype, precision):
    precision(dtype)
    dec = model[1]
    arena, lens = memories(dec, feats, [2, 2, 2])
    x, pos, ts = queries(feats, 3, 2)
    n = lens[0]
    mem = [a[:, :n] for a in arena]
    got = dec.render_tokens(x, pos, ts, (arena, None, 0, 0, 0), lens)
    _, want = dec(x, pos, ts, (mem, None, 0, 0, 0), render=True)
    assert got.shape == want.shape == (3, 2, *feats[2], 7)
    assert torch.equal(got, want)


@pytest.mark.parametrize("dtype", PRECISIONS, ids=["fp16", "bf16", "fp8"])
def test_render_tokens_unequal_lengths_match_each_scene_alone(model, feats, dtype, precision):
    """Scenes of 1, 4, 2 and 3 views, rows past each length NaN (then +inf, then -inf: the same bits); each scene's render
    is its own render against its memory truncated to its length, and the memory is bitwise unchanged."""
    precision(dtype)
    dec = model[1]
    arena, lens = memories(dec, feats, [1, 4, 2, 3])
    before = [a.clone() for a in arena]
    x, pos, ts = queries(feats, 4, 2)
    got = dec.render_tokens(x, pos, ts, (arena, None, 0, 0, 0), lens)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(got).all())
    for a, b in zip(arena, before):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    for b, n in enumerate(lens):
        _, alone = dec(x[b:b + 1], pos[b:b + 1], shape(feats[2], 1, 2), ([a[b:b + 1, :n] for a in arena], None, 0, 0, 0),
                       render=True)
        assert rel(got[b:b + 1], alone) < TOL[dtype], b
    for fill in (float("inf"), float("-inf"), 0.0):
        other = [a.clone() for a in arena]
        for a in other:
            for b, n in enumerate(lens):
                a[b, n:] = fill
        again = dec.render_tokens(x, pos, ts, (other, None, 0, 0, 0), lens)
        assert torch.equal(again, got), fill


def test_render_tokens_argument_checks(model, feats):
    dec = model[1]
    arena, lens = memories(dec, feats, [1, 2])
    x, pos, ts = queries(feats, 2, 1)
    for bad in ([1], [0, 0], [lens[0], arena[0].shape[1] + 1], [-1, lens[1]]):
        with pytest.raises(ValueError):
            dec.render_tokens(x, pos, ts, (arena, None, 0, 0, 0), bad)


def test_render_ragged_argument_errors(model):
    dec = model[1]
    w = dec._packed(cm.get_precision())
    nm = torch.ones(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    lib = _lib.lib()
    stream = cm.stream_ptr(torch.device("cuda"))

    def call_with(**fields):
        call = cm.DecoderCall()
        call.B, call.G, call.Nm, call.render, call.mem_mode = 1, 1, 10, 1, 0
        for k, v in fields.items():
            setattr(call, k, v)
        return call
    for fields, msg in ((dict(render=0), b"render"), (dict(mem_mode=1), b"kv"), (dict(mem_mode=2), b"kv"),
                        (dict(n_peers=1), b"peers"), (dict(cp_world=2), b"context parallel"), (dict(is_init=1), b"is_init"),
                        (dict(Nm=0), b"Nm")):
        rc = lib.m3r_decoder_render_ragged(C.byref(w), None, C.byref(call_with(**fields)), C.c_void_p(nm.data_ptr()),
                                           C.c_void_p(ws.data_ptr()), ws.numel(), stream)
        assert rc != 0 and msg in lib.m3r_last_error(), fields
    assert lib.m3r_decoder_render_ragged(C.byref(w), None, C.byref(call_with()), None, C.c_void_p(ws.data_ptr()),
                                         ws.numel(), stream) != 0
    assert b"null" in lib.m3r_last_error()
    w8 = cm.DecoderE4M3()                                       # no per-block scales
    rc = lib.m3r_decoder_render_ragged(C.byref(w), C.byref(w8), C.byref(call_with()), C.c_void_p(nm.data_ptr()),
                                       C.c_void_p(ws.data_ptr()), ws.numel(), stream)
    assert rc != 0 and b"e4m3" in lib.m3r_last_error()
    # the update entry point keeps refusing render
    call = call_with(new_only=1)
    assert lib.m3r_decoder_forward_ragged(C.byref(w), C.byref(call), C.c_void_p(nm.data_ptr()), C.c_void_p(ws.data_ptr()),
                                          ws.numel(), stream) != 0


def commit_rows(arena, staged, row0, rows, dst_rows, keep):
    lib = _lib.lib()
    a = (C.c_void_p * len(arena))(*[t.data_ptr() for t in arena])
    s = (C.c_void_p * len(staged))(*[t.data_ptr() for t in staged])
    d = (C.c_int64 * len(dst_rows))(*dst_rows)
    return lib.m3r_mem_commit_rows(a, s, len(arena), staged[0].shape[0], row0, rows, staged[0].shape[1],
                                   staged[0].shape[2], d, C.c_void_p(keep.data_ptr()), 0,
                                   cm.stream_ptr(torch.device("cuda")))


def test_mem_commit_rows_writes_exactly_the_selected_rows():
    """Rows [row0, row0 + rows) of every scene's staged block, Nt rows apart, land at its destination row; nothing else
    of the arena changes."""
    S, cap, W, B, Nt, depth, row0, rows = 4, 40, 256, 3, 9, 2, 4, 5
    sentinel = 7.0
    arena = [torch.full((S, cap, W), sentinel, dtype=torch.float16, device="cuda") for _ in range(depth)]
    staged = [torch.randn(B, Nt, W, device="cuda").half() for _ in range(depth)]
    keep = torch.ones(1, dtype=torch.int32, device="cuda")
    dst = [0 * cap + 3, 1 * cap + 0, 3 * cap + cap - rows]
    assert commit_rows(arena, staged, row0, rows, dst, keep) == 0
    torch.cuda.synchronize()
    for l in range(depth):
        want = torch.full((S * cap, W), sentinel, dtype=torch.float16, device="cuda")
        for b in range(B):
            want[dst[b]:dst[b] + rows] = staged[l][b, row0:row0 + rows]
        assert torch.equal(arena[l].view(S * cap, W), want), l
    lib = _lib.lib()
    assert commit_rows(arena, staged, 5, 5, dst, keep) != 0 and b"outside" in lib.m3r_last_error()
    assert commit_rows(arena, staged, -1, 2, dst, keep) != 0 and b"outside" in lib.m3r_last_error()


# ------------------------------------------------------------------------------------------------ engine
def three_scenes(paths):
    """All eight views (two portrait), five landscape views, two views (shorter than num_mem_images = 4), one view."""
    return [list(paths), list(paths[:5]), list(paths[2:4]), [paths[1]]]


def alone(model, filelist, render_once, refinements):
    n = len(filelist)
    return demo.must3r_inference(model, None, "cuda", mk.IMAGE_SIZE, False, filelist, min(4, n), 1, min(2, n), 1,
                                 render_once, is_sequence=True, num_refinements_iterations=refinements, verbose=False)


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


@pytest.mark.parametrize("render_once,refinements", [(False, 0), (True, 0), (False, 1)],
                         ids=["render", "render_once", "refine"])
def test_scenes_match_must3r_inference_alone(files, model, render_once, refinements):
    _, paths = files
    lists = three_scenes(paths)
    got = scenes.reconstruct_scenes(model, "cuda", mk.IMAGE_SIZE, False, lists, 4, 1, render_once=render_once,
                                    num_refinements_iterations=refinements, verbose=False)
    assert len(got) == len(lists)
    for s, fl in enumerate(lists):
        want = alone(model, fl, render_once, refinements)
        nmi = min(4, len(fl))
        assert got[s].image_list[:nmi] == [fl[k] for k in demo._linspace_keyframes(len(fl), nmi)]
        assert_same_scene(got[s], want, TOL[torch.float16])
    # the scenes keep their device tensors: the point clouds come out as the scene's own masking
    clouds = demo.get_3D_models_from_scene(got[0], [1.5])
    msk = [(o["conf"] >= 1.5).numpy() for o in got[0].x_out]
    assert np.array_equal(clouds[0][0], np.concatenate([o["pts3d"].numpy()[m] for o, m in zip(got[0].x_out, msk)]))


@pytest.mark.parametrize("name", ["linseq_render", "linseq_once"])
def test_scenes_reproduce_the_reference(files, model, name):
    """Two copies of the golden's scene next to a shorter one: each copy reproduces the reference's run."""
    g = np.load(os.path.join(HERE, "golden", "demo.npz"))
    _, paths = files
    kw = mk.CASES[name]
    got = scenes.reconstruct_scenes(model, "cuda", mk.IMAGE_SIZE, False, [paths, paths[:3], paths], kw["num_mem_images"],
                                    1, render_once=kw["render_once"], verbose=False)
    for scene in (got[0], got[2]):
        assert [paths.index(p) for p in scene.image_list] == g[f"{name}_order"].tolist()
        for i, o in enumerate(scene.x_out):
            assert syn.rel_l2(o["pts3d"][::mk.SUB, ::mk.SUB], torch.from_numpy(g[f"{name}_pts3d_{i}"])) < 1.5e-3, i
            assert syn.rel_l2(o["conf"][::mk.SUB, ::mk.SUB], torch.from_numpy(g[f"{name}_conf_{i}"])) < 1.5e-3, i
        np.testing.assert_allclose(np.array(scene.focals), g[f"{name}_focal"], rtol=3e-2)
        np.testing.assert_allclose(np.stack([m.numpy() for m in scene.cams2world]), g[f"{name}_c2w"], atol=3e-2)
        clouds = demo.get_3D_models_from_scene(scene, g[f"{name}_thr"].tolist())
        assert [p.shape[0] for p, _ in clouds] == g[f"{name}_count"].tolist()


def test_host_syncs_do_not_grow_with_the_scene_count(files, model, monkeypatch):
    """The engine of a batched run of three landscape scenes of different lengths synchronises as often as a run of one
    (image loading, which is per scene, is left out)."""
    _, paths = files
    land = paths[:6]
    loaded = {}

    def cached(filelist, image_size, encoder, verbose, device):
        key = tuple(filelist)
        if key not in loaded:
            loaded[key] = demo._load(filelist, image_size, encoder, verbose, device)
        return loaded[key]
    monkeypatch.setattr(scenes, "_load", cached)

    def syncs(lists):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                scenes.reconstruct_scenes(model, "cuda", mk.IMAGE_SIZE, False, lists, 4, 1, verbose=False)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        return sum("synchroniz" in str(x.message) for x in w)
    batched = [land, land[:4], land[1:]]
    syncs(batched)
    syncs([land])                          # one-time set-up (streams, tables, workspaces) is not counted
    one, three = syncs([land]), syncs(batched)
    print(f"\n[scenes] host synchronisations: 1 scene {one}, 3 scenes {three}")
    assert three == one, (one, three)


def test_engine_refuses_other_memory_modes(files, model):
    dec = model[1]
    dec.change_memory_mode("norm_y")
    try:
        with pytest.raises(NotImplementedError, match="kv"):
            scenes.reconstruct_scenes(model, "cuda", mk.IMAGE_SIZE, False, [files[1][:2]], 4, 1, verbose=False)
    finally:
        dec.change_memory_mode("kv")


# ------------------------------------------------------------------------------------------------ command line
def test_cli_matches_reconstruct_per_folder(files, tmp_path):
    chkpt, paths = files
    dirs = []
    for i, sel in enumerate([paths, paths[1:4]]):
        d = tmp_path / f"in{i}"
        d.mkdir()
        for p in sel:
            shutil.copy(p, d / os.path.basename(p))
        dirs.append(str(d))
    common = ["--weights", chkpt, "--image_size", "224", "--num_mem_imgs", "4"]
    r = subprocess.run([sys.executable, "-m", "must3r_b200.reconstruct_scenes", "--scenes", *dirs,
                        "--output", str(tmp_path / "out")] + common, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    sys.path.insert(0, HERE)
    from test_demo_cpu import read_ply
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
    r = subprocess.run([sys.executable, "-m", "must3r_b200.reconstruct_scenes", "--scenes", *dirs, "--output",
                        str(tmp_path / "x"), "--execution_mode", "vidseq"] + common, cwd=ROOT, capture_output=True,
                       text=True, timeout=300)
    assert r.returncode != 0 and "must3r_b200.reconstruct" in r.stderr
