"""Host-side logic of the SLAM front end (must3r_b200/engine/slam.py) against the reference's own run
(tests/golden/slam.npz, made by tests/golden/make_slam_golden.py): the trajectory smoothers, write_all_poses, the focal
bookkeeping and the order in which the initialisation window re-runs its frames."""
import os

import numpy as np
import pytest
import torch

from must3r_b200.engine import slam
from must3r_b200.engine.images import _slam_geometry

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "slam.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def _bare_slam(g, run="e2e"):
    """A SLAM_MUSt3R holding the reference run's per-frame results, without a model."""
    s = slam.SLAM_MUSt3R.__new__(slam.SLAM_MUSt3R)
    s.agents = [slam.MUSt3R_Agent(True)]
    s.all_poses = [torch.from_numpy(p) for p in g[f"{run}_write_none_poses"]]
    s.all_confs = [torch.tensor(c) for c in g[f"{run}_write_confs"]]
    s.all_timestamps = list(g[f"{run}_write_timestamps"])
    _replay_focals(g, run, s.agents[0])
    return s


def _replay_focals(g, run, agent, check=None):
    """Feed the agent the reference's per-call focals and mean confidences, in call order (a new epoch = a reset)."""
    res = {"e2e": 224, "tf": 48}[run]
    to_orig = _slam_geometry(240, 320, res)[3]
    epoch = None
    for k in range(len(g[f"{run}_call_frame"])):
        if g[f"{run}_call_epoch"][k] != epoch:
            epoch = g[f"{run}_call_epoch"][k]
            agent.reset()
        if check is not None:
            check(k, slam.mean_focal(agent.seq_focals))
        agent.seq_focals['f'].append(np.float32(g[f"{run}_focal"][k]))
        agent.seq_focals['to_orig'].append(to_orig)
        agent.seq_focals['conf'].append(np.float32(g[f"{run}_mean"][k]) - 1.)


@pytest.mark.parametrize("run", ["e2e", "tf"])
def test_mean_focal_and_true_focal(g, run):
    """seq_focal of every call = the confidence-weighted mean focal of the agent's earlier calls of the same epoch."""
    def check(k, seq):
        want = g[f"{run}_seq_focal"][k]
        if np.isnan(want):
            assert seq is None
        else:
            assert seq == pytest.approx(want, rel=1e-6)
    agent = slam.MUSt3R_Agent(True)
    _replay_focals(g, run, agent, check)
    assert agent.get_true_focal() == pytest.approx(float(g[f"{run}_true_focal"]), rel=1e-6)
    varying = slam.MUSt3R_Agent(False)
    _replay_focals(g, run, varying)
    assert len(varying.get_true_focal()) == len(varying.seq_focals['f'])


def test_smoothers_match_the_reference(g):
    traj = g["e2e_write_none_poses"][:, :3, -1]
    conf = g["e2e_write_confs"]
    plain = slam.laplacian_smoothing(traj, alpha=.5, iterations=5)
    np.testing.assert_allclose(plain, g["e2e_write_laplacian_poses"][:, :3, -1], rtol=1e-6, atol=1e-7)
    remap = (conf - conf.min()) / (conf.max() - conf.min())
    weighted = slam.laplacian_smoothing_with_confidence(traj, remap, alpha=.5, iterations=5)
    np.testing.assert_allclose(weighted, g["e2e_write_laplacian-conf_poses"][:, :3, -1], rtol=1e-6, atol=1e-7)
    assert np.array_equal(plain[[0, -1]], traj[[0, -1]])          # the end points stay


@pytest.mark.parametrize("mode", [None, "laplacian", "laplacian-conf"])
def test_write_all_poses_arrays_and_keys(g, tmp_path, mode):
    s = _bare_slam(g)
    path = str(tmp_path / "poses.npz")
    s.write_all_poses(path, filtering_mode=mode, run_name="golden")
    z = np.load(path, allow_pickle=True)
    assert sorted(z.files) == ["confs", "focal", "poses", "run_name", "timestamps"]
    np.testing.assert_allclose(z["poses"], g[f"e2e_write_{mode or 'none'}_poses"], rtol=1e-6, atol=1e-7)
    assert np.array_equal(z["timestamps"], g["e2e_write_timestamps"])
    np.testing.assert_array_equal(z["confs"], g["e2e_write_confs"])
    assert z["focal"].item()[0] == pytest.approx(float(g["e2e_true_focal"]), rel=1e-6)
    with pytest.raises(ValueError):
        s.write_all_poses(path, filtering_mode="median")


def test_init_window_reruns_earlier_frames_in_order(g, monkeypatch):
    """Before num_init_frames frames are in, a new frame resets the map and the earlier frames are re-run with it, each
    view handled in order (the first one as the first frame); the call order is the reference's."""
    calls = []
    s = slam.SLAM_MUSt3R.__new__(slam.SLAM_MUSt3R)
    s.agents, s.num_init_frames, s.res, s.device, s.model = [slam.MUSt3R_Agent(True)], 2, 224, "cpu", None
    s.searcher, s.overlap_mode, s.kf_x_subsamp = "kdtree-scipy-quadrant_x2", "meanconf", 4
    s.keyframe_overlap_thr, s.min_conf_keyframe, s.overlap_percentile = .13, 1.5, 70.
    s.rerender = s.keep_memory = False
    s.memory_memory, s.memory_map, s.memory_data, s.memory_overlap_tree = None, None, [], None
    s.reset()
    kf = dict(zip(range(len(g["e2e_call_frame"])), g["e2e_keyframe"]))
    monkeypatch.setattr(slam, "preproc_frame", lambda img, idx, res, device: ({"idx": idx, "true_shape": np.int32([[4, 4]])}, 1.))
    monkeypatch.setattr(slam, "forward_must3r", lambda model, views, mem, device: ([{} for _ in views], ("mem", len(views))))
    monkeypatch.setattr(slam, "_release_tail", lambda mem: None)

    def update(self, inp, pred, is_first_frame, **kw):
        k = len(calls)
        calls.append((inp["idx"], bool(is_first_frame), s.overlap_tree is None))
        pred["slam_c2w"], pred["slam_record"] = torch.eye(4), {"conf_mean": np.float32(2)}
        return None, torch.zeros(1), torch.zeros(1), None, None, 1., None, None, bool(kf[k])
    monkeypatch.setattr(slam.MUSt3R_Agent, "update", update)
    for i in range(len(g["e2e_write_timestamps"])):
        s(None, i, 0)
    assert [c[0] for c in calls] == g["e2e_call_frame"].tolist()
    assert [c[1] for c in calls] == g["e2e_first"].tolist()
    assert s.keyframes == g["e2e_keyframes"].tolist()
    assert s.all_timestamps == list(range(len(g["e2e_write_timestamps"])))
