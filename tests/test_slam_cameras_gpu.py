"""One SLAM map built by several cameras (must3r_b200/engine/slam_cameras.py): the ordered keyframe commit and the
shared-memory attention (csrc), one camera against SLAM_MUSt3R bit for bit, the step semantics with several cameras, the
one wait of a batched step, and the command line."""
import ast
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from must3r_b200 import _lib, ops
from must3r_b200.engine import slam
from must3r_b200.engine.frames import AutoMultiLoader, schedule
from must3r_b200.engine.slam_cameras import MultiCameraSLAM, steps_of
from must3r_b200.model import common as cm

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_slam_cameras_golden as mkg  # noqa: E402
import make_slam_cli_golden as mkc  # noqa: E402
import make_slam_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu
E2E = mk.RUNS["e2e"]


@pytest.fixture(scope="module")
def chkpt(tmp_path_factory):
    p = str(tmp_path_factory.mktemp("cameras") / "tiny.pth")
    mk.write_checkpoint(p)
    return p


# ------------------------------------------------------------------------------------------------ kernels
def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


@pytest.mark.parametrize("flags", [[1, 1, 1, 1], [0, 0, 0, 0], [1, 0, 1, 0], [0, 0, 0, 1]],
                         ids=["all", "none", "alternating", "last"])
def test_ordered_commit_is_sequential_commit_rows(flags):
    """m3r_mem_commit_ordered with the flags in records (stride 3 ints) = m3r_mem_commit_rows frame after frame with the
    rows counted on the host; every row past the new length (guard rows) keeps its sentinel."""
    depth, cap, W, F, Nt, row0 = 3, 40, 256, len(flags), 5, 7
    arena = [torch.full((1, cap, W), 7.0, dtype=torch.float16, device="cuda") for _ in range(depth)]
    want = [a.clone() for a in arena]
    staged = [torch.randn(F, Nt, W, device="cuda").half() for _ in range(depth)]
    keep = torch.tensor([[f, -3, 11] for f in flags], dtype=torch.int32, device="cuda").reshape(-1)
    lib, stream = _lib.lib(), cm.stream_ptr(torch.device("cuda"))
    assert lib.m3r_mem_commit_ordered(_ptrs(arena), _ptrs(staged), depth, F, Nt, W, row0, C.c_void_p(keep.data_ptr()), 3,
                                      stream) == 0
    n = row0
    for k, f in enumerate(flags):
        one = [t[k:k + 1] for t in staged]
        rc = lib.m3r_mem_commit_rows(_ptrs(want), _ptrs(one), depth, 1, 0, Nt, Nt, W, (C.c_int64 * 1)(n),
                                     C.c_void_p(keep.data_ptr() + 12 * k), 0, stream)
        assert rc == 0
        n += Nt if f else 0
    torch.cuda.synchronize()
    for a, w in zip(arena, want):
        assert torch.equal(a, w)
        assert bool((a[0, n:] == 7.0).all())
    assert lib.m3r_mem_commit_ordered(_ptrs(arena), _ptrs(staged), depth, F, Nt, W, row0,
                                      C.c_void_p(keep.data_ptr() + 2), 3, stream) != 0
    assert b"aligned" in lib.m3r_last_error()
    assert lib.m3r_mem_commit_ordered(_ptrs(arena), _ptrs(staged), depth, 65, Nt, W, row0, C.c_void_p(keep.data_ptr()), 3,
                                      stream) != 0


@pytest.mark.parametrize("splits", [None, "3"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_shared_memory_attention_is_attention_to_copies(dtype, splits, monkeypatch):
    """F frames against one memory through kv_bstride0 = 0 (the frames launched next to each other) = the same frames
    against F physical copies of it, bit for bit; each frame's own new keys are skipped, as in the decoder."""
    if splits:
        monkeypatch.setenv("M3R_ATTN_SPLITS", splits)
    torch.manual_seed(0)
    F, H, N, Nm = 3, 2, 200, 700
    D = H * 64
    q = torch.randn(F * N, D, device="cuda").to(dtype)
    mem = torch.randn(Nm, 2 * D, device="cuda").to(dtype)
    new = torch.randn(F * N, 2 * D, device="cuda").to(dtype)
    copies = mem[None].expand(F, -1, -1).contiguous().view(F * Nm, 2 * D)
    seg1 = dict(k1=new[:, :D], v1=new[:, D:], Nk1=N, kv_bstride1=N, skip_lo=Nm, skip_step=N, skip_len=N)
    shared = ops.attention(q, mem[:, :D], mem[:, D:], B=F, H=H, Nq=N, Nk0=Nm, kv_bstride0=0, **seg1)
    copied = ops.attention(q, copies[:, :D], copies[:, D:], B=F, H=H, Nq=N, Nk0=Nm, kv_bstride0=Nm, **seg1)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(shared.float()).all())
    assert torch.equal(shared, copied)


def _views(F=3, H=48, W=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    loc = torch.rand(F, H, W, 3, generator=g) * 2 - 1
    loc[..., 2] = 1 + torch.rand(F, H, W, generator=g)
    ang = torch.rand(F, generator=g)
    R = torch.stack([torch.stack([ang.cos(), -ang.sin(), 0 * ang], -1), torch.stack([ang.sin(), ang.cos(), 0 * ang], -1),
                     torch.tensor([[0., 0., 1.]]).expand(F, 3)], 1)
    pts = torch.einsum("fij,fhwj->fhwi", R, loc) + torch.rand(F, 1, 1, 3, generator=g) + 0.01 * torch.randn(F, H, W, 3, generator=g)
    conf = 1 + 2 * torch.rand(F, H, W, generator=g)
    return pts.cuda().contiguous(), loc.cuda().contiguous(), conf.cuda().contiguous()


def test_pose_views_is_per_view_slam_pose():
    """m3r_slam_pose_views with a focal state per view = m3r_slam_pose of each view alone, bit for bit (the records and
    the depth rectified in place)."""
    pts, loc, conf = _views()
    seqs, first = [None, 55.0, 41.5], [False, False, True]
    loc_b = loc.clone()
    rec = ops.slam_pose_views(pts, loc_b, conf, seqs, first)
    for v in range(3):
        loc_v = loc[v:v + 1].clone()
        one = ops.slam_pose(pts[v:v + 1], loc_v, conf[v:v + 1], seq_focal=seqs[v], is_first=first[v])
        torch.cuda.synchronize()
        assert torch.equal(rec[v:v + 1], one), v
        assert torch.equal(loc_b[v:v + 1], loc_v), v
    assert not torch.equal(loc_b[1], loc[1])                              # view 1 was rectified
    with pytest.raises(RuntimeError):
        ops.slam_pose_views(*_views(F=65, H=4, W=4), [None] * 65, [False] * 65)


@pytest.mark.parametrize("mode", ["nn-norm", "nn", "meanconf"])
def test_keyframe_frames_is_single_calls(mode):
    """m3r_slam_keyframe_frames over F frames = m3r_slam_keyframe frame after frame, bit for bit, record by record."""
    F, H, W, s = 3, 48, 64, 4
    pts, loc, conf = _views(F, H, W, seed=1)
    rec = ops.slam_pose_views(pts, loc, conf, [None] * F, [False] * F)
    Q = (H // s) * (W // s)
    dists = (torch.rand(F, Q, device="cuda") * 0.5).contiguous()
    dists[1, ::7] = float("inf")
    kw = dict(subsamp=s, mode=mode, percentile=70., thr=0.1, min_conf_keyframe=1.5)
    singles = rec.clone()
    for f in range(F):
        ops.slam_keyframe(dists[f].contiguous() if mode != "meanconf" else None, conf[f], loc[f], singles[f:f + 1],
                          is_first=f == 2, **kw)
    ops.slam_keyframe_frames(dists if mode != "meanconf" else None, conf, loc, rec, is_first=[False, False, True], **kw)
    torch.cuda.synchronize()
    assert torch.equal(rec, singles)
    assert rec.cpu().numpy().view(ops.SLAM_RECORD)[2, 0]["keyframe"] == 1


# ------------------------------------------------------------------------------------------------ against the reference
@pytest.fixture(scope="module")
def gc():
    return np.load(os.path.join(HERE, "golden", "slam_cameras.npz"))


@pytest.fixture(scope="module")
def golden_runs(chkpt, gc, tmp_path_factory):
    """The golden runs of make_slam_cameras_golden.py through MultiCameraSLAM on the fp16 test model."""
    d = tmp_path_factory.mktemp("golden_runs")
    runs = {}
    for run in ("equal", "mixed", "cont"):
        seqs = mkg.sequences(run)
        kw = mkg.run_kwargs(run, float(gc[f"{run}_thr"]), float(gc[f"{run}_min_conf"]))
        load = str(d / "equal.pkl") if run == "cont" else None
        mc = MultiCameraSLAM(chkpt, len(seqs), device="cuda:0", load_memory=load, **kw)
        for st in mkg.steps(seqs):
            mc.step({c: (seqs[c][k], t) for c, k, t in st})
        if run == "equal":
            mc.save_memory(str(d / "equal.pkl"))
        runs[run] = mc
    return runs


@pytest.mark.parametrize("run", ["equal", "mixed", "cont"])
def test_runs_match_the_reference_steps(golden_runs, gc, run):
    mc = golden_runs[run]
    assert mc.keyframes == gc[f"{run}_keyframes"].tolist()
    assert mc.all_timestamps == gc[f"{run}_timestamps"].tolist()
    np.testing.assert_allclose(torch.stack(mc.all_poses).cpu().numpy(), gc[f"{run}_poses"], atol=3e-2)
    vals, labels, nimgs = mc.memory[0], mc.memory[1], mc.memory[2]
    assert [list(v.shape) for v in vals] == gc[f"{run}_mem_shapes"].tolist()
    assert np.array_equal(labels.cpu().numpy(), gc[f"{run}_mem_labels"]) and nimgs == int(gc[f"{run}_mem_nimgs"])
    digest = np.array([[v.double().sum().item(), v.double().abs().sum().item(), v.double().square().sum().item()]
                       for v in vals])
    np.testing.assert_allclose(digest[:, 1:], gc[f"{run}_mem_digest"][:, 1:], rtol=2e-2)
    for agid, f in mc.get_true_focals().items():
        np.testing.assert_allclose(np.asarray(f, dtype=np.float64).reshape(-1), gc[f"{run}_focal_{agid}"], rtol=3e-2)
    if run == "mixed":
        assert mc.stats["alone"] > 3 and mc.stats["batched"] > 0        # the square camera runs alone in mixed steps


# ------------------------------------------------------------------------------------------------ whole runs
def _memory_state(s):
    vals, labels, nimgs, _, n = s.memory
    return [v.clone() for v in vals], labels.clone(), nimgs, n


def test_one_camera_is_slam_bit_for_bit(chkpt):
    frames = mk.frames()
    alone = slam.SLAM_MUSt3R(chkpt, device="cuda:0", keep_memory=True, **E2E)
    aouts = [alone(im, i, 0) for i, im in enumerate(frames)]
    mc = MultiCameraSLAM(chkpt, 1, device="cuda:0", keep_memory=True, **E2E)
    outs = [mc.step({0: (im, i)})[0] for i, im in enumerate(frames)]
    assert mc.stats["batched"] > 0
    assert mc.keyframes == alone.keyframes
    assert mc.all_timestamps == alone.all_timestamps
    for o, a in zip(outs, aouts):
        assert o[-1] == a[-1]
        assert np.array_equal(o[0], a[0]) and np.array_equal(o[1], a[1])
        assert torch.equal(o[2], a[2]) and torch.equal(o[3], a[3]) and torch.equal(o[5], a[5])
        assert np.array_equal(np.asarray(o[4]), np.asarray(a[4]))
    assert torch.equal(torch.stack(mc.all_poses), torch.stack(alone.all_poses))
    assert torch.equal(torch.stack(mc.all_confs), torch.stack(alone.all_confs))
    mv, ml, mn, mlen = _memory_state(mc)
    av, al, an, alen = _memory_state(alone)
    assert (mn, mlen) == (an, alen) and torch.equal(ml, al)
    for x, y in zip(mv, av):
        assert torch.equal(x, y)
    assert len(mc.keyframe_pointmaps) == len(alone.keyframe_pointmaps)
    assert mc.get_true_focals() == alone.get_true_focals()
    mc.rerender_all_frames(maxbs=5)
    alone.rerender_all_frames(maxbs=5)
    assert torch.equal(torch.stack(mc.all_poses), torch.stack(alone.all_poses))


def test_a_step_decodes_against_the_memory_before_it(chkpt):
    """Two cameras given the same frames: in every batched step both frames are decoded against the same pre-step memory
    and searcher (varying focals: no per-agent focal state enters the pose), so both give the same result - and both are
    keyframes together, where the reference would let the second frame see the first's keyframe."""
    frames = mk.frames()
    mc = MultiCameraSLAM(chkpt, 2, device="cuda:0", keep_memory=True, **{**E2E, "rerender": False, "fixed_focal": False})
    kf_steps = 0
    for i, im in enumerate(frames):
        before = mc.stats["batched"]
        out = mc.step({0: (im, 2 * i), 1: (im, 2 * i + 1)})
        if mc.stats["batched"] - before == 2:
            a, b = out[0], out[1]
            assert a[-1] == b[-1]
            assert np.array_equal(a[0], b[0]) and torch.equal(a[5], b[5]) and torch.equal(a[3], b[3])
            kf_steps += a[-1]
    assert mc.stats["batched"] > 0
    n = mc.memory[0][0].shape[1]
    labels = mc.memory[1][0].tolist()
    assert mc.memory[4] == n == len(labels) and mc.memory[2] == labels[-1] + 1
    assert labels == sorted(labels)                                      # images appended in order
    if kf_steps:
        assert any(mc.keyframes[j] + 1 == mc.keyframes[j + 1] for j in range(len(mc.keyframes) - 1))


def test_saved_memory_continues(chkpt, tmp_path):
    frames = mk.frames()
    mc = MultiCameraSLAM(chkpt, 2, device="cuda:0", keep_memory=True, **{**E2E, "rerender": False})
    for i in range(0, 8, 2):
        mc.step({0: (frames[i], i), 1: (frames[i + 1], i + 1)})
    p = str(tmp_path / "m.pkl")
    mc.save_memory(p)
    more = MultiCameraSLAM(chkpt, 2, device="cuda:0", load_memory=p, keep_memory=True, **{**E2E, "rerender": False})
    assert more.memory[0][0].shape == mc.memory[0][0].shape and more.memory[2:] == mc.memory[2:]
    for i in range(8, 12, 2):
        more.step({0: (frames[i], i), 1: (frames[i + 1], i + 1)})
    assert more.stats["alone"] >= 2 and more.stats["batched"] > 0
    assert more.all_timestamps == [8, 9, 10, 11]          # the two initialisation re-runs, then one batched step


def test_step_without_keyframe_waits_once(chkpt, monkeypatch):
    frames = mk.frames()
    mc = MultiCameraSLAM(chkpt, 2, device="cuda:0", **{**E2E, "rerender": False, "keyframe_overlap_thr": 1e9})
    for i in range(3):
        mc.step({0: (frames[i], 2 * i), 1: (frames[i + 1], 2 * i + 1)})
    waits = []
    dec, wait = MultiCameraSLAM._decode_shared, slam._wait_host_copies

    def decode_then_strict(self, *a, **k):
        out = dec(self, *a, **k)
        torch.cuda.set_sync_debug_mode("error")
        return out

    def named_wait():
        torch.cuda.set_sync_debug_mode(0)
        waits.append(1)
        wait()
        torch.cuda.set_sync_debug_mode("error")

    monkeypatch.setattr(MultiCameraSLAM, "_decode_shared", decode_then_strict)
    monkeypatch.setattr(slam, "_wait_host_copies", named_wait)
    try:
        out = mc.step({0: (frames[4], 8), 1: (frames[5], 9)})
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not out[0][-1] and not out[1][-1]
    assert waits == [1]


# ------------------------------------------------------------------------------------------------ command line
def test_cli_over_two_folders(chkpt, tmp_path):
    d = str(tmp_path)
    mkc.write_folders(os.path.join(d, "frames"))
    folders = [os.path.join(d, "frames", n) for n in ("cam0", "cam1")]
    common = ["--chkpt", chkpt, "--device", "cuda:0", "--image_string", mkc.IMAGE_STRING, "--res", "224",
              "--varying_focals", "--input"] + folders

    def sh(mod, out):
        r = subprocess.run([sys.executable, "-m", mod] + common + ["--output", out], cwd=ROOT, capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        return ast.literal_eval([x for x in r.stdout.splitlines() if " keyframes: [" in x][-1].split("keyframes: ")[1])

    kf = sh("must3r_b200.slam_cameras", os.path.join(d, "cams"))
    sh("must3r_b200.slam", os.path.join(d, "one"))
    zc = np.load(os.path.join(d, "cams", "all_poses.npz"), allow_pickle=True)
    zo = np.load(os.path.join(d, "one", "all_poses.npz"), allow_pickle=True)
    assert np.array_equal(zc["timestamps"], zo["timestamps"]) and np.array_equal(zc["imgHWs"], zo["imgHWs"])
    assert zc["poses"].shape == zo["poses"].shape and set(zc.files) == set(zo.files)
    assert os.path.exists(os.path.join(d, "cams", "memory.pkl"))

    # the same steps driven through the engine give the command's keyframes
    from must3r_b200.engine.frames import decode
    mc = MultiCameraSLAM(chkpt, 2, device="cuda:0", res=224, kf_x_subsamp=2, keyframe_overlap_thr=.1,
                         min_conf_keyframe=1.2, overlap_percentile=85., keep_memory=True, fixed_focal=False)
    items, _ = schedule(AutoMultiLoader(folders, mkc.IMAGE_STRING), 1)
    for st in steps_of(items):
        mc.step({c: (torch.from_numpy(decode(p)).cuda(), t) for p, c, t in st})
    assert mc.keyframes == kf
    assert np.array_equal(np.array(mc.all_timestamps), zc["timestamps"])
