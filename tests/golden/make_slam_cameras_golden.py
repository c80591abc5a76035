"""Golden data of one SLAM map built by several cameras (must3r_b200/engine/slam_cameras.py), from the UNMODIFIED
reference's functions on the CPU in fp32 (the tiny random checkpoint and the cv2 / roma stand-ins of
make_slam_cli_golden.py / make_slam_golden.py).

The reference feeds the cameras one frame at a time.  The multi-camera step is composed here from its own pieces: each
step takes the next frame of every camera that still has frames, in the reference's order.  Frames run alone through
the reference's SLAM_MUSt3R.__call__ while the memory is empty or the initialisation re-runs are not done.  Otherwise,
when the step's frames share the most common preprocessed shape:
  * each of them is decoded with forward_must3r against the memory as it stood before the step;
  * each is updated by its own camera's agent against the searcher as it stood before the step;
  * at the end of the step, each frame's timestamp and pose are recorded in camera order, and each keyframe's new memory
    rows, labels, searcher points and point map are appended in camera order.
A frame of another shape then runs alone through __call__.

Runs: 'equal' (2 folders of 6 frames), 'mixed' (3 folders of different sizes and lengths, --varying_focals), 'cont' (2
cameras continued from the memory of 'equal').  Stores keyframes, timestamps, poses, per-agent focals and memory
digests.

    python tests/golden/make_slam_cameras_golden.py [--check]
"""
import argparse
import os
import sys
import tempfile
from collections import Counter

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_slam_cli_golden as mkc  # noqa: E402
import make_slam_golden as mk  # noqa: E402

MARGIN = 0.05
THRESHOLDS = [0.13, 0.1, 0.08, 0.12, 0.06, 0.15, 0.05, 0.2]
MIN_CONFS = [1.5, 1.2, 1.3, 1.1, 1.05]


def sequences(run):
    """The frames of each camera of a run."""
    if run == "mixed":
        return [mk.frames(6, seed=5), mk.frames(4, seed=6, H=240, W=240, step=16), mk.frames(5, seed=7)]
    if run == "cont":
        return [mk.frames(4, seed=11), mk.frames(4, seed=12)]
    return [mk.frames(6, seed=5), mk.frames(6, seed=8)]


def run_kwargs(run, thr, min_conf):
    # res 224 crops every frame to a square; at 512 the square camera of 'mixed' has its own shape and runs alone
    return dict(res=512 if run == "mixed" else 224, keyframe_overlap_thr=thr, min_conf_keyframe=min_conf, fixed_focal=run != "mixed",
                keep_memory=True)


def steps(seqs):
    """[(cam, frame index, timestamp)] per step: the reference's AutoMultiLoader order cut at each camera's second frame."""
    out, t = [], 0
    for k in range(max(len(s) for s in seqs)):
        st = []
        for c, s in enumerate(seqs):
            if k < len(s):
                st.append((c, k, t))
                t += 1
        out.append(st)
    return out


def plan(cands):
    """engine/slam_sessions.py plan_batch, restated: the most common shape (the first on a tie) is batched."""
    shapes = Counter(sh for sh in cands.values() if sh is not None)
    if not shapes:
        return [], list(cands)
    best = max(shapes.values())
    shape = next(sh for sh in cands.values() if sh is not None and shapes[sh] == best)
    batch = [c for c, sh in cands.items() if sh == shape]
    return batch, [c for c in cands if c not in batch]


def step(ref_model, slam, frames):
    """One multi-camera step of the reference SLAM_MUSt3R `slam`: frames = [(cam, img, timestamp)] in camera order."""
    together = slam.memory is not None and len(slam.all_images) >= slam.num_init_frames
    cands, prepped = {}, {}
    for cam, img, fid in frames:
        if together:
            prepped[cam] = ref_model.preproc_frame(img, fid, res=slam.res, transform=slam.transform)
            cands[cam] = tuple(int(v) for v in np.asarray(prepped[cam][0]['true_shape']).reshape(-1)[:2])
        else:
            cands[cam] = None
    batch, alone = plan(cands)
    by_cam = {cam: (img, fid) for cam, img, fid in frames}
    mem0 = slam.memory
    done = []
    for cam in batch:
        view, to_orig = prepped[cam]
        preds, newmem = ref_model.forward_must3r(slam.model, [view], mem0, device=slam.device)
        out = slam.agents[cam].update(view, preds[0], False, overlap_mode=slam.overlap_mode,
                                      overlap_tree=slam.overlap_tree, kf_x_subsamp=slam.kf_x_subsamp,
                                      keyframe_overlap_thr=slam.keyframe_overlap_thr,
                                      min_conf_keyframe=slam.min_conf_keyframe,
                                      overlap_percentile=slam.overlap_percentile, to_orig_focal=to_orig)
        done.append((by_cam[cam][1], newmem, out))
    n0 = 0 if mem0 is None else mem0[0][0].shape[1]
    for fid, newmem, out in done:
        selpts3d, pts3d, colors, depth, conf, focal, w2c, cam_center, iskeyframe = out
        slam.all_timestamps.append(fid)
        slam.all_poses.append(w2c.inverse())
        slam.all_confs.append(conf.mean())
        if iskeyframe:
            vals, labels, nimgs, prot, ntok = slam.memory
            rows = [v[:, n0:] for v in newmem[0]]
            slam.memory = ([torch.cat([v, r], 1) for v, r in zip(vals, rows)],
                           torch.cat([labels, torch.full((1, rows[0].shape[1]), nimgs, dtype=labels.dtype)], 1),
                           nimgs + 1, prot + 1, ntok + rows[0].shape[1])
            slam.keyframes.append(fid)
            if slam.overlap_tree is not None:
                slam.overlap_tree.add_pts(selpts3d, cam_center=cam_center)
            if slam.keep_memory:
                slam.keyframe_pointmaps.append([pts3d.cpu(), colors.cpu(), conf.cpu()])
    for cam in alone:
        img, fid = by_cam[cam]
        slam(img, fid, cam)


def memory_record(mem):
    vals, labels = mem[0], mem[1]
    return {"mem_shapes": np.array([list(v.shape) for v in vals]), "mem_labels": labels.cpu().numpy().astype(np.int64),
            "mem_nimgs": np.array(int(mem[2])),
            "mem_digest": np.array([[v.double().sum().item(), v.double().abs().sum().item(), v.double().square().sum().item()]
                                    for v in vals])}


def run_one(ref_model, run, chkpt, thr, min_conf, load_memory=None):
    """-> (slam, the (score, median, first) of every postproc_pred call)."""
    calls = []
    orig = ref_model.postproc_pred

    def recording(img, res, is_first_frame, *a, **k):
        out = orig(img, res, is_first_frame, *a, **k)
        calls.append((float(res["overlap_score"]), float(res["conf"][0, 0].median()), bool(is_first_frame)))
        return out
    ref_model.postproc_pred = recording
    try:
        seqs = sequences(run)
        slam = ref_model.SLAM_MUSt3R(chkpt, device="cpu", num_agents=len(seqs), load_memory=load_memory,
                                     **run_kwargs(run, thr, min_conf))
        for st in steps(seqs):
            step(ref_model, slam, [(c, seqs[c][k], t) for c, k, t in st])
    finally:
        ref_model.postproc_pred = orig
    return slam, calls


def generate(d):
    ref_model, _ = mkc.import_reference()
    torch.set_grad_enabled(False)
    chkpt = os.path.join(d, "tiny.pth")
    mk.write_checkpoint(chkpt)
    out = {}
    for run in ("equal", "mixed", "cont"):
        for thr in THRESHOLDS:
            for min_conf in MIN_CONFS:
                load = os.path.join(d, "equal_memory.pkl") if run == "cont" else None
                slam, calls = run_one(ref_model, run, chkpt, thr, min_conf, load)
                if all(abs(s - thr) >= MARGIN * thr and abs(m - min_conf) >= MARGIN * min_conf
                       for s, m, first in calls if not first):
                    break
            else:
                continue
            break
        else:
            raise AssertionError(f"run {run}: no threshold pair clears every score and median confidence by {MARGIN}")
        if run == "equal":
            slam.save_memory(os.path.join(d, "equal_memory.pkl"))
        rec = {"thr": np.array(thr), "min_conf": np.array(min_conf), "keyframes": np.array(slam.keyframes, dtype=np.int64),
               "timestamps": np.array(slam.all_timestamps, dtype=np.int64),
               "poses": torch.stack(slam.all_poses).numpy(), **memory_record(slam.memory)}
        for agid, f in slam.get_true_focals().items():
            rec[f"focal_{agid}"] = np.asarray(f, dtype=np.float64).reshape(-1)
        out.update({f"{run}_{k}": v for k, v in rec.items()})
        print(run, "thr", thr, "min_conf", min_conf, "keyframes", slam.keyframes, "timestamps", slam.all_timestamps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true", help="compare with the stored slam_cameras.npz instead of writing it")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as d:
        out = generate(d)
    path = os.path.join(HERE, "slam_cameras.npz")
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
