#!/usr/bin/env python
"""Generate tests/golden/slam.npz by running the UNMODIFIED reference SLAM front end (must3r/slam/model.py SLAM_MUSt3R)
on the CPU in fp32 (device='cpu').  Needs a reference checkout (oracle/install_reference.py finds it):

    python tests/golden/make_slam_golden.py

The model is a tiny random checkpoint (weights from must3r_b200/synthetic.py, constructor strings of the reference's
classes) written to a temporary file; the tests write the same checkpoint again with `write_checkpoint`.  The frames are
seeded uint8 crops of a panorama that slides to the right (`frames`).

`roma` is not installed.  A module of that name is provided whose `rigid_points_registration` is roma's documented
algorithm, the weighted orthogonal Procrustes (Kabsch) solution with det R = +1, evaluated in float64 by the oracle
(oracle/must3r_oracle.py rigid_registration).

Two runs:
  * 'e2e' at res=224 (rerender=True): per-frame focal, c2w, overlap score, median / mean confidence and keyframe flag,
    the keyframe list, the write_all_poses arrays (plain and both smoothers) and the poses after rerender_all_frames;
  * 'tf' at res=48: the same per-frame records plus each frame's pts3d / pts3d_local / conf as the reference's
    postprocess produced them (before the in-place rectification), for the teacher-forced tests; small maps keep the
    file well under 1 MB.
The thresholds are chosen so that every score is at least 5 % away from keyframe_overlap_thr and every median confidence
at least 5 % away from min_conf_keyframe; the script asserts these margins.
"""
import argparse
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from must3r_b200 import synthetic as syn  # noqa: E402

ENCODER = "Dust3rEncoder(img_size=(224, 224), patch_size=16, embed_dim=128, depth=2, num_heads=2, pos_embed='RoPE100')"
DECODER = ("MUSt3R(img_size=(224, 224), enc_embed_dim=128, embed_dim=128, depth=2, num_heads=2, "
           "feedback_type='single_mlp', memory_mode='kv', landscape_only=False)")
SEED = 3
N_FRAMES = 12
MARGIN = 0.05
RUNS = {  # name -> SLAM_MUSt3R arguments besides chkpt / device
    "e2e": dict(res=224, keyframe_overlap_thr=0.13, min_conf_keyframe=1.5, rerender=True),
    "tf": dict(res=48, keyframe_overlap_thr=0.1, min_conf_keyframe=1.5),
}


def write_checkpoint(path, seed=SEED):
    esd = syn.encoder_state_dict(seed, embed_dim=128, depth=2)
    dsd = syn.decoder_state_dict(seed, enc_embed_dim=128, embed_dim=128, depth=2, feedback_type="single_mlp")
    syn.camera_like_head_bias(dsd)           # positive depth and a positive focal from a random network
    torch.save({"args": argparse.Namespace(encoder=ENCODER, decoder=DECODER), "encoder": esd, "decoder": dsd}, path)


def frames(n=N_FRAMES, seed=SEED, H=240, W=320, step=12):
    pano = syn.synthetic_frame(H, W + step * n, seed=seed)
    return [np.ascontiguousarray(pano[:, step * i:step * i + W]) for i in range(n)]


def _install_roma():
    from oracle.must3r_oracle import rigid_registration

    def rigid_points_registration(x, y, weights=None, compute_scaling=False):
        assert not compute_scaling
        B = x.shape[0]
        w = torch.ones(x.shape[:-1]) if weights is None else weights
        Rs, ts = zip(*[rigid_registration(x[b].cpu(), y[b].cpu(), w[b].cpu()) for b in range(B)])
        return torch.stack(Rs).float().to(x.device), torch.stack(ts).float().to(x.device)

    sys.modules["roma"] = types.SimpleNamespace(rigid_points_registration=rigid_points_registration)


def run(ref_model, chkpt, imgs, kw, keep_preds):
    """One reference run; returns the arrays recorded under the run's prefix."""
    calls = []
    orig = ref_model.postproc_pred

    def recording_postproc_pred(img, res, is_first_frame, seq_focals, fixed_focal=True, **k):
        seq = ref_model.mean_focal(seq_focals) if fixed_focal else None
        pred = {n: res[n][0, 0].clone().numpy() for n in ("pts3d", "pts3d_local", "conf")}
        out = orig(img, res, is_first_frame, seq_focals, fixed_focal=fixed_focal, **k)
        conf = res["conf"][0, 0]
        calls.append(dict(pred=pred, first=bool(is_first_frame), seq=np.nan if seq is None else float(seq),
                          focal=float(out[5][0]), c2w=torch.inverse(out[6]).numpy(), score=float(res["overlap_score"]),
                          median=float(conf.median()), mean=float(conf.mean()), kf=bool(out[8])))
        return out

    ref_model.postproc_pred = recording_postproc_pred
    try:
        slam = ref_model.SLAM_MUSt3R(chkpt, device="cpu", **kw)
        frame_of_call, epochs, epoch, tree = [], [], -1, None
        for i, im in enumerate(imgs):
            n0 = len(calls)
            slam(im, i, 0)
            ids = list(range(i - (len(calls) - n0) + 1, i + 1))
            frame_of_call += ids
            if slam.overlap_tree is not tree:
                tree, epoch = slam.overlap_tree, epoch + 1
            epochs += [epoch] * len(ids)
    finally:
        ref_model.postproc_pred = orig
    out = {
        "call_frame": np.array(frame_of_call), "call_epoch": np.array(epochs),
        "first": np.array([c["first"] for c in calls]), "seq_focal": np.array([c["seq"] for c in calls]),
        "focal": np.array([c["focal"] for c in calls]), "c2w": np.stack([c["c2w"] for c in calls]),
        "score": np.array([c["score"] for c in calls]), "median": np.array([c["median"] for c in calls]),
        "mean": np.array([c["mean"] for c in calls]), "keyframe": np.array([c["kf"] for c in calls]),
        "keyframes": np.array(slam.keyframes), "true_focal": np.array(slam.get_true_focals()[0]),
        "poses": torch.stack(slam.all_poses).numpy(), "confs": torch.stack(slam.all_confs).numpy(),
    }
    print(kw, "keyframes", slam.keyframes, "scores", np.round(out["score"], 4).tolist(),
          "medians", np.round(out["median"], 4).tolist())
    for c in calls:                     # no decision may hinge on rounding
        if not c["first"]:
            assert abs(c["score"] - kw["keyframe_overlap_thr"]) >= MARGIN * kw["keyframe_overlap_thr"], (c["score"], kw)
            assert abs(c["median"] - kw["min_conf_keyframe"]) >= MARGIN * kw["min_conf_keyframe"], (c["median"], kw)
    if keep_preds:
        for n in ("pts3d", "pts3d_local", "conf"):
            out[n] = np.stack([c["pred"][n] for c in calls])
    if kw.get("rerender"):
        with tempfile.TemporaryDirectory() as d:
            for mode in (None, "laplacian", "laplacian-conf"):
                p = os.path.join(d, "poses.npz")
                slam.write_all_poses(p, filtering_mode=mode)
                z = np.load(p, allow_pickle=True)
                out[f"write_{mode or 'none'}_poses"] = z["poses"]
                if mode is None:
                    out["write_timestamps"], out["write_confs"] = z["timestamps"], z["confs"]
        slam.rerender_all_frames(maxbs=5)
        out["rerender_poses"] = torch.stack(slam.all_poses).numpy()
    return out


def main():
    from oracle.install_reference import source
    ref = source()
    assert ref is not None, "no reference checkout found (set MUST3R_REFERENCE)"
    sys.path.insert(0, ref)
    _install_roma()
    torch.set_grad_enabled(False)
    import must3r.slam.model as ref_model
    imgs = frames()
    out = {}
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "tiny.pth")
        write_checkpoint(chkpt)
        for name, kw in RUNS.items():
            rec = run(ref_model, chkpt, imgs, kw, keep_preds=name == "tf")
            out.update({f"{name}_{k}": v for k, v in rec.items()})
    path = os.path.join(HERE, "slam.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
