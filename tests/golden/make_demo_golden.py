#!/usr/bin/env python
"""Generate tests/golden/demo.npz by running the UNMODIFIED reference demo inference (must3r/demo/inference.py) on the CPU
in fp32 (device='cpu').  Needs a reference checkout (oracle/install_reference.py finds it):

    python tests/golden/make_demo_golden.py [--check]

--check regenerates the arrays and compares them with the stored file instead of writing it.

The model is make_slam_golden.py's tiny random checkpoint, loaded at image_size 384.  The images are seeded crops of a
sliding synthetic panorama written as PNG files to a temporary directory: six landscape 384x288 and two portrait 288x384
frames, so two aspect ratios occur and load_images keeps them at their size (no resampling).  `roma` gets
make_slam_golden.py's stand-in; `faiss` and `asmk`, imported at module level by must3r.retrieval.processor, get empty
stand-ins (retrieval is never run).  gradio.py imports gradio and trimesh, so get_reconstructed_scene's mode dispatch
(gradio.py:177-203) and the point-cloud masking (gradio.py:147-151, :91-92) are restated here.

Cases ('linseq' with render_once False and True, 'vidseq', 'vidslam'), each recording: the order of the views in the
scene (indices into the sorted file list), the keyframe list, per view pts3d and conf subsampled by SUB in both axes
(full-size maps would make the file several MB), focal and c2w, and the point cloud's count at two thresholds.  The
thresholds are placed in gaps of the scene's confidences, at least CONF_MARGIN (relative) from every confidence, so the
counts are a stable target; 'vidslam' uses a keyframe_overlap_thr that every overlap score clears by 5 %.  The script
asserts both margins.
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
sys.path.insert(0, HERE)

import make_slam_golden as mk  # noqa: E402
from must3r_b200 import synthetic as syn  # noqa: E402

IMAGE_SIZE = 384
SUB = 8
CONF_MARGIN = 0.0025
MARGIN = 0.05
SEED = 7
SLAM_THRESHOLDS = [0.05, 0.03, 0.08, 0.12, 0.02, 0.2]       # the first every score clears by MARGIN is used
CASES = {  # name -> get_reconstructed_scene execution arguments
    "linseq_render": dict(execution_mode="linseq", num_mem_images=4, render_once=False),
    "linseq_once": dict(execution_mode="linseq", num_mem_images=4, render_once=True),
    "vidseq": dict(execution_mode="vidseq", vidseq_local_context_size=3, keyframe_interval=3),
    "vidslam": dict(execution_mode="vidslam", slam_local_context_size=0, subsample=2, min_conf_keyframe=1.5,
                    overlap_percentile=85.0),
}


def images(n_land=6, n_port=2, seed=SEED, step=16):
    """RGB uint8 frames in sequence order: landscape crops of a panorama sliding right, then portrait crops."""
    pano = syn.synthetic_frame(384, 384 + step * (n_land + n_port), seed=seed)
    out = [np.ascontiguousarray(pano[48:336, step * i:step * i + 384]) for i in range(n_land)]
    out += [np.ascontiguousarray(pano[:, step * i:step * i + 288]) for i in range(n_land, n_land + n_port)]
    return out


def write_images(d):
    import PIL.Image
    paths = []
    for i, im in enumerate(images()):
        p = os.path.join(d, f"{i:03d}.png")
        PIL.Image.fromarray(im).save(p)
        paths.append(p)
    return paths


def gap_thresholds(confs, n=2, margin=CONF_MARGIN):
    """n thresholds, each at least `margin` (relative) from every confidence, inside the 10-90 % quantile band if
    possible: the centres of the widest relative gaps between consecutive sorted confidences."""
    c = np.unique(np.concatenate([x.reshape(-1) for x in confs]).astype(np.float64))
    c = c[np.isfinite(c)]
    lo, hi = np.quantile(c, 0.1), np.quantile(c, 0.9)
    mid = np.sqrt(c[:-1] * c[1:])
    width = np.log(c[1:] / c[:-1])
    for band in ((mid > lo) & (mid < hi), np.ones_like(mid, dtype=bool)):
        idx = np.flatnonzero(band)
        idx = idx[np.argsort(-width[idx])][:n]
        if len(idx) == n and (width[idx] >= 2 * np.log1p(margin)).all():
            thr = np.sort(mid[idx].astype(np.float32))
            for t in thr:
                assert np.abs(c / t - 1).min() >= margin, t
            return thr
    raise AssertionError("no confidence gap wide enough for a stable point-cloud count")


def _install_stubs():
    mk._install_roma()
    sys.modules.setdefault("faiss", types.SimpleNamespace(StandardGpuResources=lambda: None))
    sys.modules.setdefault("asmk", types.SimpleNamespace(asmk_method=None))


def run_case(ref, model, paths, kw, keyframe_overlap_thr=None):
    """get_reconstructed_scene (gradio.py:177-203) with the reference's functions; returns (scene, keyframes, scores)."""
    import functools
    from must3r.slam.model import get_searcher
    inf = ref
    mode = kw["execution_mode"]
    keyframes, scores = [], []
    if mode in ("vidseq", "vidslam"):
        if mode == "vidseq":
            def is_kf(id, res, scene_state): return (id % kw["keyframe_interval"] == 0)
            scene_state, update = None, (lambda res, scene_state: scene_state)
            local = kw["vidseq_local_context_size"]
        else:
            orig = inf.get_overlap_score

            def recording_score(*a, **k):
                s = orig(*a, **k)
                scores.append(float(s))
                return s
            inf.get_overlap_score = recording_score
            is_kf = functools.partial(inf.slam_is_keyframe, kw["subsample"], kw["min_conf_keyframe"],
                                      keyframe_overlap_thr, kw["overlap_percentile"], "nn-norm")
            scene_state = get_searcher("kdtree-scipy-quadrant_x2")
            update = functools.partial(inf.slam_update_scene_state, kw["subsample"], kw["min_conf_keyframe"])
            local = kw["slam_local_context_size"]

        def recording_kf(id, res, scene_state):
            r = bool(is_kf(id, res, scene_state))
            if r:
                keyframes.append(int(id))
            return r
        try:
            scene = inf.must3r_inference_video(model, "cpu", IMAGE_SIZE, False, paths, 1, init_num_images=2,
                                               batch_num_views=1, local_context_size=local,
                                               is_keyframe_function=recording_kf, scene_state=scene_state,
                                               scene_state_update_function=update, verbose=False)
        finally:
            if mode == "vidslam":
                inf.get_overlap_score = orig
        keyframes = [0, 1] + keyframes
    else:
        scene = inf.must3r_inference(model, None, "cpu", IMAGE_SIZE, False, paths, kw["num_mem_images"], 1,
                                     init_num_images=2, batch_num_views=1, render_once=kw["render_once"],
                                     is_sequence=True, verbose=False)
        keyframes = np.linspace(0, len(paths) - 1, kw["num_mem_images"], dtype=int).tolist()
    return scene, keyframes, scores


def record(name, scene, keyframes, scores, paths):
    out = {f"{name}_order": np.array([paths.index(p) for p in scene.image_list]),
           f"{name}_keyframes": np.array(keyframes),
           f"{name}_focal": np.array(scene.focals, dtype=np.float32),
           f"{name}_c2w": np.stack([np.asarray(m) for m in scene.cams2world]).astype(np.float32)}
    confs = [o["conf"].numpy() for o in scene.x_out]
    for i, o in enumerate(scene.x_out):
        out[f"{name}_pts3d_{i}"] = o["pts3d"].numpy()[::SUB, ::SUB]
        out[f"{name}_conf_{i}"] = confs[i][::SUB, ::SUB]
    thr = gap_thresholds(confs)
    counts, means = [], []
    for t in thr:
        # gradio.py:150-151 then :91-92
        pts3d = [o["pts3d"].numpy() for o in scene.x_out]
        msk = [(o["conf"] >= float(t)).numpy() for o in scene.x_out]
        pts = np.concatenate([p[m] for p, m in zip(pts3d, msk)])
        col = np.concatenate([p[m] for p, m in zip(scene.imgs, msk)])
        counts.append(pts.shape[0])
        means.append(np.concatenate([pts.mean(0), col.mean(0)]))
    out[f"{name}_thr"] = thr
    out[f"{name}_count"] = np.array(counts)
    out[f"{name}_cloud_mean"] = np.stack(means)
    if scores:
        out[f"{name}_scores"] = np.array(scores)
    return out


def generate():
    from oracle.install_reference import source
    ref_dir = source()
    assert ref_dir is not None, "no reference checkout found (set MUST3R_REFERENCE)"
    sys.path.insert(0, ref_dir)
    _install_stubs()
    torch.set_grad_enabled(False)
    import must3r.demo.inference as ref
    from must3r.model import load_model
    out = {}
    with tempfile.TemporaryDirectory() as d:
        chkpt = os.path.join(d, "tiny.pth")
        mk.write_checkpoint(chkpt)
        model = load_model(chkpt, device="cpu", img_size=IMAGE_SIZE, verbose=False)
        paths = write_images(d)
        for name, kw in CASES.items():
            if kw["execution_mode"] == "vidslam":
                for thr in SLAM_THRESHOLDS:
                    scene, kf, scores = run_case(ref, model, paths, kw, keyframe_overlap_thr=thr)
                    if all(abs(s - thr) >= MARGIN * thr for s in scores):
                        break
                else:
                    raise AssertionError(f"no keyframe_overlap_thr of {SLAM_THRESHOLDS} clears every score by {MARGIN}")
                out["vidslam_keyframe_overlap_thr"] = np.array(thr)
            else:
                scene, kf, scores = run_case(ref, model, paths, kw)
            out.update(record(name, scene, kf, scores, paths))
            print(name, "order", out[f"{name}_order"].tolist(), "keyframes", kf, "counts", out[f"{name}_count"].tolist(),
                  "scores", np.round(scores, 4).tolist())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--check", action="store_true", help="compare with the stored demo.npz instead of writing it")
    args = ap.parse_args()
    out = generate()
    path = os.path.join(HERE, "demo.npz")
    if args.check:
        g = np.load(path)
        assert sorted(g.files) == sorted(out), (sorted(g.files), sorted(out))
        for k, v in out.items():
            if v.dtype.kind in "iub":
                assert np.array_equal(g[k], v), k
            else:
                np.testing.assert_allclose(g[k], v, rtol=1e-4, atol=1e-5, err_msg=k)
        print(path, "reproduced")
        return
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
