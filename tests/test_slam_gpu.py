"""The SLAM front end on the GPU (csrc/slam.cu, must3r_b200/engine/slam.py) against engine/camera.py, torch / numpy
order statistics and the reference's own run (tests/golden/slam.npz, made by tests/golden/make_slam_golden.py)."""
import os
import sys

import numpy as np
import pytest
import torch

from must3r_b200 import ops
from must3r_b200.engine import camera, slam
from must3r_b200.engine.keyframes import get_searcher
from oracle import must3r_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_slam_golden as mk  # noqa: E402  (checkpoint and frames of the fixture; the reference is not imported)

pytestmark = pytest.mark.gpu
FLT_MAX = float(np.finfo(np.float32).max)


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(HERE, "golden", "slam.npz"))


@pytest.fixture(scope="module")
def chkpt(tmp_path_factory):
    p = str(tmp_path_factory.mktemp("slam") / "tiny.pth")
    mk.write_checkpoint(p)
    return p


def _records(rec):
    return rec.cpu().numpy().view(ops.SLAM_RECORD)[:, 0]


def _check_pose(pts, loc, conf, seq=None):
    """Kernel vs camera.py (focal) and the SVD Procrustes in float64, on a batch of views."""
    B, H, W = conf.shape
    loc_before = loc.clone()
    rec = _records(ops.slam_pose(pts, loc, conf, seq_focal=seq))
    pp = torch.tensor((W / 2, H / 2), device=pts.device)
    focal = camera.estimate_focal_weiszfeld(loc_before, pp)
    np.testing.assert_allclose(rec["focal"], focal.cpu().numpy(), rtol=2e-4)      # fp32 torch vs double sums
    ratio = torch.ones(B, device=pts.device) if seq is None else \
        torch.tensor(np.float32(seq) / rec["focal"], device=pts.device)
    want_z = loc_before[..., 2] * ratio.view(B, 1, 1)
    assert torch.equal(loc[..., 2], want_z) and torch.equal(loc[..., :2], loc_before[..., :2])      # in place, fp32
    for b in range(B):                  # the weighted Kabsch / SVD solution in float64
        R, t = orc.rigid_registration(loc[b].reshape(-1, 3).cpu(), pts[b].reshape(-1, 3).cpu(), (conf[b] - 1).reshape(-1).cpu())
        np.testing.assert_allclose(rec["c2w"][b, :3, :3], R.numpy(), atol=2e-5)
        np.testing.assert_allclose(rec["c2w"][b, :3, 3], t.numpy(), atol=2e-5)
    Rs, _ = camera.rigid_points_registration(loc.reshape(B, -1, 3), pts.reshape(B, -1, 3), (conf - 1).reshape(B, -1),
                                             method="svd")
    np.testing.assert_allclose(rec["c2w"][:, :3, :3], Rs.cpu().numpy(), atol=1e-3)      # camera.py solves in fp32
    np.testing.assert_allclose(np.einsum("bij,bjk->bik", rec["w2c"], rec["c2w"]), np.broadcast_to(np.eye(4), (B, 4, 4)), atol=2e-6)
    assert np.array_equal(rec["conf_median"], conf.reshape(B, -1).median(dim=1).values.cpu().numpy())
    np.testing.assert_allclose(rec["conf_mean"], conf.reshape(B, -1).double().mean(1).cpu().numpy(), rtol=1e-6)
    return rec


def test_pose_kernel_on_the_reference_predictions(g):
    pts = torch.from_numpy(g["tf_pts3d"]).cuda().contiguous()
    loc = torch.from_numpy(g["tf_pts3d_local"]).cuda().contiguous()
    conf = torch.from_numpy(g["tf_conf"]).cuda().contiguous()
    _check_pose(pts, loc, conf)
    _check_pose(pts, loc.clone(), conf, seq=11.5)


def test_pose_kernel_adversarial():
    """z <= 0 pixels, confidence exactly 1 on most pixels, H x W not a multiple of the CTA size, B > 1."""
    gen = torch.Generator().manual_seed(5)
    B, H, W = 3, 37, 53
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    z = 1 + torch.rand(B, H, W, generator=gen)
    loc = torch.stack([(xs - W / 2) * z / 40, (ys - H / 2) * z / 40, z], -1) + 0.01 * torch.randn(B, H, W, 3, generator=gen)
    loc[:, ::7, ::5, 2] = 0.0
    loc[:, 3::11, 2::9, 2] *= -1
    ang = 0.3
    R = torch.tensor([[np.cos(ang), -np.sin(ang), 0], [np.sin(ang), np.cos(ang), 0], [0, 0, 1]], dtype=torch.float32)
    pts = loc @ R.T + torch.tensor([0.5, -0.2, 1.0]) + 0.01 * torch.randn(B, H, W, 3, generator=gen)
    conf = torch.ones(B, H, W)
    sel = torch.rand(B, H, W, generator=gen) < 0.2
    conf[sel] = 1 + 3 * torch.rand(int(sel.sum()), generator=gen)
    rec = _check_pose(pts.cuda(), loc.cuda().contiguous(), conf.cuda())
    # the first frame defines the origin: identity pose, no rectification
    loc2 = loc.cuda().contiguous()
    first = _records(ops.slam_pose(pts.cuda(), loc2, conf.cuda(), seq_focal=10.0, is_first=True))
    assert np.array_equal(first["c2w"], np.broadcast_to(np.eye(4, dtype=np.float32), (B, 4, 4)))
    assert torch.equal(loc2, loc.cuda()) and np.array_equal(first["focal"], rec["focal"])


def _keyframe(values, conf, percentile=70., min_conf=1.5, mode="nn"):
    H, W = conf.shape
    rec = ops.slam_pose(torch.zeros(1, H, W, 3, device="cuda"), torch.ones(1, H, W, 3, device="cuda"), conf[None].contiguous())
    ops.slam_keyframe(values.contiguous(), conf.contiguous(), torch.ones(H, W, 3, device="cuda"), rec, subsamp=1, mode=mode,
                      percentile=percentile, thr=0.5, min_conf_keyframe=min_conf, is_first=False)
    return _records(rec)[0]


@pytest.mark.parametrize("case", ["ties", "inf", "nan_masked", "single", "none", "nan_kept", "random"])
@pytest.mark.parametrize("percentile", [0., 33.3, 70., 100.])
def test_selection_is_np_percentile(case, percentile):
    gen = torch.Generator().manual_seed(11)
    H, W = 29, 41
    vals = torch.rand(H * W, generator=gen)
    conf = 1 + torch.rand(H, W, generator=gen)
    if case == "ties":
        vals = torch.randint(0, 4, (H * W,), generator=gen).float() / 4
    if case == "inf":
        vals[::3] = float("inf")
    if case == "nan_masked":
        vals[::5] = float("nan")
        conf.view(-1)[::5] = 1.0
    if case == "nan_kept":
        vals[7] = float("nan")
        conf.view(-1)[7] = 2.0
    if case == "single":
        conf[:] = 1.0
        conf[3, 4] = 1.9
    if case == "none":
        conf[:] = 1.2
    r = _keyframe(vals.cuda(), conf.cuda(), percentile)
    msk = conf.reshape(-1) > 1.5
    assert r["n_conf"] == int(msk.sum())
    d = vals[msk].double().numpy()
    d[np.isposinf(d)] = FLT_MAX
    want = 0.0 if d.size == 0 else np.percentile(d, percentile)
    if d.size:
        assert np.isnan(want) == np.isnan(torch.quantile(torch.from_numpy(d), percentile / 100).item())
    if np.isnan(want):
        assert np.isnan(r["score"])
    else:
        assert r["score"] == want
        if d.size and not np.isnan(d).any():
            assert r["score"] == torch.quantile(torch.from_numpy(d), percentile / 100, interpolation="linear").item()
    assert r["keyframe"] == int(bool(r["score"] > 0.5) and r["conf_median"] > 1.5)


def test_teacher_forced_against_the_reference(g):
    """Fed the reference's per-frame predictions, seq_focal and first-frame flag, each frame's focal, pose, overlap score
    and decision match the reference's.  Tolerances: focal 1e-4 relative and pose 1e-4 absolute (fp32 sums in the reference
    against double sums here, on points of magnitude ~5); the score 1e-4 relative (fp32 distances here, float64 scipy
    distances in the reference); decisions exactly (every score is >= 5 % from the threshold)."""
    kw = mk.RUNS["tf"]
    tree, epoch = None, None
    for k in range(len(g["tf_call_frame"])):
        if g["tf_call_epoch"][k] != epoch:
            epoch, tree = g["tf_call_epoch"][k], get_searcher("kdtree-scipy-quadrant_x2")
        pts = torch.from_numpy(g["tf_pts3d"][k]).cuda()
        loc = torch.from_numpy(g["tf_pts3d_local"][k]).cuda()
        conf = torch.from_numpy(g["tf_conf"][k]).cuda()
        seq = None if np.isnan(g["tf_seq_focal"][k]) else float(g["tf_seq_focal"][k])
        rec = ops.slam_pose(pts[None], loc[None], conf[None], seq_focal=seq, is_first=bool(g["tf_first"][k]))
        c2w = ops.slam_record_c2w(rec)[0]
        sub = pts[::4, ::4].reshape(-1, 3)
        d = tree.query(sub, cam_center=c2w[:3, 3])
        ops.slam_keyframe(d, conf, loc, rec, subsamp=4, mode="nn-norm", percentile=70., thr=kw["keyframe_overlap_thr"],
                          min_conf_keyframe=kw["min_conf_keyframe"], is_first=bool(g["tf_first"][k]))
        r = _records(rec)[0]
        assert r["focal"] == pytest.approx(g["tf_focal"][k], rel=1e-4), k
        np.testing.assert_allclose(r["c2w"], g["tf_c2w"][k], atol=1e-4, err_msg=str(k))
        if g["tf_score"][k] >= FLT_MAX:
            assert r["score"] == FLT_MAX
        else:
            assert r["score"] == pytest.approx(g["tf_score"][k], rel=1e-4), k
        assert bool(r["keyframe"]) == bool(g["tf_keyframe"][k]), k
        if r["keyframe"]:
            msk = conf[::4, ::4].reshape(-1) > kw["min_conf_keyframe"]
            tree.add_pts(sub[msk], cam_center=c2w[:3, 3])


def _run(chkpt, frames, **kw):
    s = slam.SLAM_MUSt3R(chkpt, device="cuda:0", **{**mk.RUNS["e2e"], **kw})
    outs = [s(im, i, 0) for i, im in enumerate(frames)]
    return s, outs


def test_end_to_end_against_the_reference(g, chkpt, tmp_path):
    """The CUDA model runs fp16 operands; its pointmaps stay within 1.5e-3 relative L2 of the fp32 reference (the parity
    gate of smoke()).  The poses come from a weighted fit over those points and are held to 20x that (3e-2 absolute on
    entries of magnitude <= ~1); keyframe decisions must match exactly (scores are >= 7 % from the threshold)."""
    s, outs = _run(chkpt, mk.frames())
    assert s.keyframes == g["e2e_keyframes"].tolist()
    last_call = [int(np.flatnonzero(g["e2e_call_frame"] == i)[-1]) for i in range(len(outs))]
    assert [bool(o[-1]) for o in outs] == [bool(g["e2e_keyframe"][k]) for k in last_call]
    poses = torch.stack(s.all_poses).cpu().numpy()
    np.testing.assert_allclose(poses, g["e2e_poses"], atol=3e-2)
    p = str(tmp_path / "poses.npz")
    s.write_all_poses(p, filtering_mode="laplacian-conf")
    z = np.load(p, allow_pickle=True)
    np.testing.assert_allclose(z["poses"], g["e2e_write_laplacian-conf_poses"], atol=3e-2)
    assert np.array_equal(z["timestamps"], g["e2e_write_timestamps"])
    np.testing.assert_allclose(z["confs"], g["e2e_write_confs"], rtol=1e-2)
    s.rerender_all_frames(maxbs=5)
    np.testing.assert_allclose(torch.stack(s.all_poses).cpu().numpy(), g["e2e_rerender_poses"], atol=3e-2)
    assert s.all_pts3d.shape == (1, 12, 224, 224, 3)
    assert outs[-1][0].shape == (224, 224, 3) and outs[-1][1].shape == (1, 1, 224, 224, 3)


def test_save_and_reload_continues_like_the_live_memory(chkpt, tmp_path):
    frames = mk.frames()
    a, _ = _run(chkpt, frames[:6], keep_memory=True)
    path = str(tmp_path / "mem.pkl")
    a.save_memory(path)
    a.memory_memory, a.memory_data, a.memory_overlap_tree = a.memory, a.keyframe_pointmaps, a.overlap_tree
    a.reset()
    b = slam.SLAM_MUSt3R(chkpt, device="cuda:0", load_memory=path, keep_memory=True, **mk.RUNS["e2e"])
    assert b.fetch_memory_map(1.5)[0].shape == a.fetch_memory_map(1.5)[0].shape
    for i, im in enumerate(frames[6:]):
        oa, ob = a(im, 6 + i, 0), b(im, 6 + i, 0)
        assert oa[-1] == ob[-1]
        np.testing.assert_allclose(oa[0], ob[0], rtol=0, atol=1e-6)
        np.testing.assert_allclose(oa[5].cpu().numpy(), ob[5].cpu().numpy(), atol=1e-6)
    assert a.keyframes == b.keyframes


def test_non_keyframe_syncs_only_at_its_one_wait(chkpt, monkeypatch, g):
    frames = mk.frames()
    s, _ = _run(chkpt, frames[:4])
    waits = []
    fwd, wait = slam.forward_must3r, slam._wait_host_copies

    def forward_then_strict(*a, **k):
        out = fwd(*a, **k)
        torch.cuda.set_sync_debug_mode("error")
        return out

    def named_wait():
        torch.cuda.set_sync_debug_mode(0)
        waits.append(1)
        wait()
        torch.cuda.set_sync_debug_mode("error")

    monkeypatch.setattr(slam, "forward_must3r", forward_then_strict)
    monkeypatch.setattr(slam, "_wait_host_copies", named_wait)
    try:
        out = s(frames[4], 4, 0)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not out[-1] and not g["e2e_keyframe"][5]
    assert waits == [1]
