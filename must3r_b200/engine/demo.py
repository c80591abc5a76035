"""The reconstruction front end of the reference's demo (must3r/demo/inference.py and the scene functions of
must3r/demo/gradio.py) with the same names, arguments and results, on the CUDA model: `SceneState`, `load_images`,
`slam_is_keyframe`, `slam_update_scene_state`, `must3r_inference`, `must3r_inference_video`, `get_reconstructed_scene`
and `get_3D_model_from_scene`.

The engine runs with its results on the device.  Once the last view is predicted, every array the `SceneState` holds is
copied to the host in one batch of asynchronous copies followed by one wait; the device tensors stay attached to the
scene (not pickled), so the point clouds are gathered on the GPU by `m3r_scene_points` (csrc/scene.cu), up to 8
confidence thresholds per pass, and only the selected points travel to the host.

Deliberate differences from the reference:
  * Retrieval (the unordered mode with a retrieval checkpoint) needs `asmk` and `faiss`, which this package does not
    vendor, so its keyframe choice cannot be reproduced: a retrieval checkpoint raises NotImplementedError.  Without one
    the unordered mode takes linspace keyframes, as the reference does.
  * No viser, gradio or trimesh: `viser_server` must be None, `get_3D_model_from_scene` needs as_pointcloud=True and
    returns the point cloud (pts, col) [N,3] float32 arrays (gradio.py:91-92); it writes them as a PLY file only when
    given a `filename` ending in '.ply' (cameras are not exported, as in the reference's PLY export).
  * The `vidslam` keyframe test reads one host value per frame: the overlap score from the SLAM keyframe kernel
    (`m3r_slam_keyframe`) over the searcher's distances of every subsampled pixel.
  * `amp` selects the CUDA model's 16-bit operand format for the call ('fp16', 'bf16'); False keeps the current one.
  * The scene's true_shape is a list of host int32 tensors (the reference leaves device tensors in it).
"""
from __future__ import annotations

import datetime
import functools
import os
from contextlib import contextmanager

import numpy as np
import torch

from .. import ops
from ..model import get_dtype, get_pointmaps_activation
from ..model.common import get_precision, set_precision
from .images import load_images  # noqa: F401  (the reference's name; decodes and resizes on the GPU)
from .inference import _sync_host_copies, _to_out, inference_multi_ar, inference_video_multi_ar, postprocess
from .keyframes import choose_keyframe_from_overlap, get_overlap_score, get_searcher

# get_reconstruction.py:85,106: the thresholds its point clouds are written at
THRESHOLDS = [6.0, 5.0, 4.0, 3.0, 2.5, 2.0, 1.5, 1.05]


class SceneState:
    """must3r/demo/inference.py:21-28: what scene.pkl holds.  x_out: per view {'pts3d', 'pts3d_local', 'conf', 'focal',
    'c2w'} host tensors; imgs: per view [H,W,3] float32 colours in [0, 1]; true_shape: per view int32 (H, W); focals:
    floats; cams2world: [4,4] host tensors; image_list: the file names in x_out's order."""

    def __init__(self, x_out, imgs, true_shape, focals, cams2world, image_list):
        self.x_out = x_out
        self.imgs = imgs
        self.true_shape = true_shape
        self.focals = focals
        self.cams2world = cams2world
        self.image_list = image_list

    def __getstate__(self):
        return {k: v for k, v in self.__dict__.items() if k != "_device"}      # the device copies are not saved


@contextmanager
def _amp(amp):
    prev = get_precision()
    if amp:
        set_precision(get_dtype(amp))
    try:
        yield
    finally:
        set_precision(prev)


def _no_viser(viser_server):
    if viser_server is not None:
        raise NotImplementedError("must3r_b200's demo has no viser visualisation: pass viser_server=None")


def _rgb(img):
    """dust3r.utils.image.rgb of an ImgNorm image [3,H,W]: [H,W,3], (x * 0.5) + 0.5 clipped to [0, 1] (NaN stays)."""
    return img.permute(1, 2, 0).mul(0.5).add_(0.5).clamp_(0, 1).contiguous()


def _scene_from_device(x_out, imgs, true_shape, filenames):
    """Copy the results to the host in one batch of asynchronous copies and one wait; keep the device tensors on the scene
    for the point-cloud gather (inference.py:224-236 copies each tensor with a synchronising .cpu())."""
    copies = _launch_scene_copies(x_out, imgs)
    _sync_host_copies()
    return _finish_scene(copies, true_shape, filenames)


def _launch_scene_copies(x_out, imgs):
    """Enqueue the host copies of one scene's results (no wait) -> what _finish_scene takes once they are waited for."""
    dev = {"pts3d": [o["pts3d"] for o in x_out], "pts3d_local": [o["pts3d_local"] for o in x_out],
           "conf": [o["conf"] for o in x_out], "c2w": [o["c2w"] for o in x_out], "img": list(imgs)}
    host = [{k: _to_out(v, "cpu") for k, v in o.items()} for o in x_out]
    cols = [_to_out(_rgb(im), "cpu") for im in imgs]
    return dev, host, cols


def _finish_scene(copies, true_shape, filenames):
    dev, host, cols = copies
    focals = [float(o["focal"]) for o in host]
    cams2world = [o["c2w"] for o in host]
    scene = SceneState(host, [c.numpy() for c in cols], true_shape, focals, cams2world, filenames)
    scene._device = dev
    return scene


def _mem_batches(nimgs, init_num_images, batch_num_views, total, last):
    """inference.py:188-191 (total = max(num_mem_images, init_num_images), last = num_mem_images) and :282-285 (both
    nimgs): init_num_images views first, then batch_num_views at a time until `total`.  Where the reference's loop
    would never end, this raises."""
    batches = [min(init_num_images, nimgs)]
    while (sum_b := sum(batches)) != total:
        size_b = min(batch_num_views, last - sum_b)
        if size_b <= 0:
            raise ValueError(f"cannot build a memory of {total} views from {nimgs} images "
                             f"with init_num_images={init_num_images}")
        batches.append(size_b)
    return batches


def _to_render(render_once, num_mem_images, nimgs):
    """inference.py:193-196: render only the views outside the memory (render_once), or all of them (None)."""
    return list(range(num_mem_images, nimgs)) if render_once else None


def _linspace_keyframes(nimgs, num_mem_images):
    """inference.py:140"""
    return np.linspace(0, nimgs - 1, num_mem_images, dtype=int).tolist()


def _load(filelist, image_size, encoder, verbose, device):
    p = getattr(encoder, "patch_size", 16)
    return load_images(filelist, size=image_size, patch_size=p[0] if isinstance(p, (tuple, list)) else p,
                       verbose=verbose, device=device)


def _report(verbose, what, start, device):
    if verbose:
        print(f'{what} in {datetime.datetime.now() - start}')
        try:
            print(str(int(torch.cuda.max_memory_reserved(device) / (1024 ** 2))) + " MB")
        except Exception:  # noqa: BLE001  (as the reference: the memory report is optional)
            pass


# ------------------------------------------------------------------------------------------- the vidslam callbacks
def slam_is_keyframe(subsample, min_conf_keyframe, keyframe_overlap_thr, overlap_percentile, overlap_mode, id, res,
                     scene_state):
    """inference.py:79-92.  The nearest-neighbour modes score every subsampled pixel's distance in the SLAM keyframe
    kernel and read the score back once; the confidence modes use get_overlap_score as the reference does."""
    cam_center = res['c2w'][:3, -1]
    if ops.overlap_mode_id(overlap_mode) > 1:
        res_unsqueeze = {k: v.unsqueeze(0).unsqueeze(0) for k, v in res.items()}
        overlap_score = get_overlap_score(res_unsqueeze, scene_state, cam_center=cam_center, mode=overlap_mode,
                                          kf_x_subsamp=subsample, min_conf_keyframe=min_conf_keyframe,
                                          percentile=overlap_percentile)
    else:
        s = subsample or 1
        conf, loc = res['conf'].contiguous(), res['pts3d_local'].contiguous()
        dists = scene_state.query(res['pts3d'][::s, ::s].reshape(-1, 3), cam_center=cam_center).float().contiguous()
        rec = torch.zeros((1, ops.SLAM_RECORD.itemsize), dtype=torch.uint8, device=conf.device)
        with torch.cuda.device(conf.device):
            ops.slam_keyframe(dists, conf, loc, rec, subsamp=s, mode=overlap_mode, percentile=overlap_percentile,
                              thr=keyframe_overlap_thr, min_conf_keyframe=min_conf_keyframe, is_first=False)
        host = _to_out(rec, "cpu")
        _sync_host_copies()
        overlap_score = float(host.numpy().view(ops.SLAM_RECORD)[0, 0]['score'])
    assert not np.isnan(overlap_score)
    return choose_keyframe_from_overlap(overlap_score, keyframe_overlap_thr, overlap_mode)


def slam_update_scene_state(subsample, min_conf_keyframe, res, scene_state):
    """inference.py:95-106: add the keyframe's confident (subsampled) points to the searcher."""
    cam_center = res['c2w'][:3, -1]
    msk = res['conf'] > min_conf_keyframe
    if subsample:
        msk = msk[::subsample, ::subsample]
        pts = res['pts3d'][::subsample, ::subsample][msk]
    else:
        pts = res['pts3d'][msk]
    scene_state.add_pts(pts, cam_center=cam_center)
    return scene_state


# ------------------------------------------------------------------------------------------- inference
@torch.no_grad()
def must3r_inference(model, retrieval, device, image_size, amp,
                     filelist, num_mem_images, max_bs, init_num_images, batch_num_views, render_once,
                     is_sequence, viser_server=None, num_refinements_iterations=0, verbose=True):
    """inference.py:109-241: linspace keyframes build the memory (init_num_images, then batch_num_views at a time), then
    every view is rendered (or, with render_once, only those outside the memory) -> SceneState."""
    _no_viser(viser_server)
    if not is_sequence and retrieval is not None:
        raise NotImplementedError("retrieval keyframes need the asmk and faiss packages, which must3r_b200 does not "
                                  "vendor, so the reference's keyframe choice cannot be reproduced; run without a "
                                  "retrieval checkpoint (linspace keyframes) or in a sequence mode")
    max_bs = None if max_bs == 0 else max_bs
    encoder, decoder = model
    pointmaps_activation = get_pointmaps_activation(decoder, verbose=verbose)
    def post_process_function(x): return postprocess(x, pointmaps_activation=pointmaps_activation, compute_cam=True)

    if verbose:
        print('loading images')
    time_start = datetime.datetime.now()
    views = _load(filelist, image_size, encoder, verbose, device)
    nimgs = len(views)
    if verbose:
        print(f'loaded in {datetime.datetime.now() - time_start}')
        print('running inference')
    time_start = datetime.datetime.now()

    keyframes = _linspace_keyframes(nimgs, num_mem_images)
    not_keyframes = sorted(set(range(nimgs)).difference(set(keyframes)))
    assert (len(keyframes) + len(not_keyframes)) == nimgs
    order = keyframes + not_keyframes
    imgs = [views[i]['img'] for i in order]
    true_shape = [torch.from_numpy(views[i]['true_shape']) for i in order]      # host: the engine reads it there
    filenames = [filelist[i] for i in order]
    img_ids = [torch.tensor(v) for v in order]
    mem_batches = _mem_batches(nimgs, init_num_images, batch_num_views, max(num_mem_images, init_num_images), num_mem_images)
    to_render = _to_render(render_once, num_mem_images, nimgs)

    with _amp(amp):
        x_out_0, x_out = inference_multi_ar(encoder, decoder, imgs, img_ids, true_shape, mem_batches,
                                            max_bs=max_bs, verbose=verbose, to_render=to_render,
                                            encoder_precomputed_features=None, device=device, preserve_gpu_mem=False,
                                            post_process_function=post_process_function,
                                            num_refinements_iterations=num_refinements_iterations)
    if to_render is not None:
        x_out = x_out_0 + x_out
    _report(verbose, 'inference', time_start, device)
    return _scene_from_device(x_out, imgs, true_shape, filenames)


@torch.no_grad()
def must3r_inference_video(model, device, image_size, amp,
                           filelist, max_bs, init_num_images, batch_num_views,
                           viser_server=None, num_refinements_iterations=0, local_context_size: int = 25,
                           is_keyframe_function=lambda id, res, scene_state: (id % 3 == 0),
                           scene_state=None,
                           scene_state_update_function=lambda res, scene_state: scene_state,
                           verbose=True):
    """inference.py:244-331: the streaming schedule (keyframes + a rolling window of local_context_size frames) over the
    views in order -> SceneState.  The callbacks see per-view results on the device."""
    _no_viser(viser_server)
    max_bs = None if max_bs == 0 else max_bs
    encoder, decoder = model
    pointmaps_activation = get_pointmaps_activation(decoder, verbose=verbose)
    def post_process_function(x): return postprocess(x, pointmaps_activation=pointmaps_activation, compute_cam=True)

    if verbose:
        print('loading images')
    time_start = datetime.datetime.now()
    views = _load(filelist, image_size, encoder, verbose, device)
    nimgs = len(views)
    if verbose:
        print(f'loaded in {datetime.datetime.now() - time_start}')
        print('running inference')
    time_start = datetime.datetime.now()

    imgs = [b['img'] for b in views]
    true_shape = [torch.from_numpy(b['true_shape']) for b in views]
    mem_batches = _mem_batches(nimgs, init_num_images, batch_num_views, nimgs, nimgs)

    with _amp(amp):
        x_out = inference_video_multi_ar(encoder, decoder, imgs, true_shape, mem_batches,
                                         max_bs=max_bs, verbose=verbose,
                                         device=device, preserve_gpu_mem=False,
                                         post_process_function=post_process_function,
                                         num_refinements_iterations=num_refinements_iterations,
                                         local_context_size=local_context_size,
                                         is_keyframe_function=is_keyframe_function,
                                         scene_state=scene_state,
                                         scene_state_update_function=scene_state_update_function)
    _report(verbose, 'inference', time_start, device)
    return _scene_from_device(x_out, imgs, true_shape, list(filelist))


# ------------------------------------------------------------------------------------------- gradio.py's scene functions
def _device_maps(scene, local_pointmaps):
    """The scene's per-view device tensors: those kept by the inference, or the host ones uploaded (a loaded scene.pkl)."""
    dev = getattr(scene, "_device", None)
    if dev is None:
        x_out = scene.x_out
        put = lambda t: torch.as_tensor(t).float().cuda(non_blocking=True).contiguous()      # noqa: E731
        # The stored colours c are rgb() outputs.  c * 2 - 1 is exact for them (for c >= 1/4 by Sterbenz's lemma; a
        # smaller c is (x * 0.5) + 0.5 with x * 0.5 in [-1/2, -3/8], a multiple of 2^-25), and so is (y * 0.5) + 0.5
        # back: the kernel's colours are the stored ones bit for bit.
        dev = {"pts3d": [put(o["pts3d"]) for o in x_out], "pts3d_local": [put(o["pts3d_local"]) for o in x_out],
               "conf": [put(o["conf"]) for o in x_out], "c2w": [put(m) for m in scene.cams2world],
               "img": [put(np.asarray(im)).permute(2, 0, 1).mul(2).sub(1).contiguous() for im in scene.imgs]}
        scene._device = dev
    pts = dev["pts3d_local"] if local_pointmaps else dev["pts3d"]
    c2w = [m.float().contiguous() for m in dev["c2w"]] if local_pointmaps else None
    return [p.float().contiguous() for p in pts], [c.float().contiguous() for c in dev["conf"]], \
        [im.float().contiguous() for im in dev["img"]], c2w


@torch.no_grad()
def get_3D_models_from_scene(scene, thresholds, local_pointmaps=False):
    """The point clouds of get_3D_model_from_scene at several thresholds, gathered on the GPU in one pass
    (m3r_scene_points, at most 8 thresholds per pass) and copied to the host with one wait: [(pts [N,3], col [N,3])]
    float32 numpy arrays, one pair per threshold, each in the reference's order (view after view, raster order)."""
    pts3d, conf, imgs, c2w = _device_maps(scene, local_pointmaps)
    out = []
    for lo in range(0, len(thresholds), ops.SCENE_MAX_THR):
        thr = list(thresholds[lo:lo + ops.SCENE_MAX_THR])
        with torch.cuda.device(conf[0].device):
            pts, col, counts = ops.scene_points(pts3d, conf, imgs, thr, c2w=c2w)
        hp, hc = _to_out(pts, "cpu"), _to_out(col, "cpu")
        _sync_host_copies()
        hp, hc = hp.numpy(), hc.numpy()
        off = np.concatenate([[0], np.cumsum(counts)])
        out += [(hp[off[t]:off[t + 1]], hc[off[t]:off[t + 1]]) for t in range(len(thr))]
    return out


def write_ply(path, pts, col):
    """Binary little-endian PLY of a point cloud: `x y z` float32 and `red green blue` uchar per vertex.  Colours in
    [0, 1] become bytes as round(255 * c) (round half to even, clipped to [0, 255]); this is not claimed to be trimesh's
    rule, which the reference's export uses."""
    pts = np.asarray(pts, dtype=np.float32).reshape(-1, 3)
    col = np.asarray(col, dtype=np.float32).reshape(-1, 3)
    assert pts.shape == col.shape
    rec = np.empty(pts.shape[0], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"),
                                        ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    rec["x"], rec["y"], rec["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
    u8 = np.clip(np.rint(np.nan_to_num(col) * 255), 0, 255).astype(np.uint8)
    rec["red"], rec["green"], rec["blue"] = u8[:, 0], u8[:, 1], u8[:, 2]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {pts.shape[0]}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              "end_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(rec.tobytes())
    return path


@torch.no_grad()
def get_3D_model_from_scene(outdir, verbose, scene, min_conf_thr=3.0, as_pointcloud=False,
                            transparent_cams=False, local_pointmaps=False, cam_size=0.05, camera_conf_thr=0.0,
                            filename=None):
    """gradio.py:131-156 with as_pointcloud=True: the points with conf >= min_conf_thr (pts3d, or pts3d_local moved by
    the view's c2w with local_pointmaps) and their colours, as (pts [N,3], col [N,3]) float32 arrays (gradio.py:91-92).
    With a filename ending in '.ply' they are also written to outdir/filename.  Camera options only concern the GLB's
    camera meshes and are ignored."""
    if scene is None:
        return None
    if not as_pointcloud:
        raise NotImplementedError("mesh export needs trimesh, which must3r_b200 does not use: pass as_pointcloud=True")
    if filename is not None and not filename.endswith(".ply"):
        raise NotImplementedError(f"{filename}: only PLY point clouds are written (GLB export needs trimesh)")
    pts, col = get_3D_models_from_scene(scene, [min_conf_thr], local_pointmaps=local_pointmaps)[0]
    if filename is not None:
        outfile = os.path.join(outdir, filename)
        if verbose:
            print('(exporting 3D scene to', outfile, ')')
        write_ply(outfile, pts, col)
    return pts, col


@torch.no_grad()
def get_reconstructed_scene(outdir, viser_server, should_save_glb, model, retrieval, device, verbose, image_size, amp,
                            filelist, max_bs, num_refinements_iterations,  # main params
                            execution_mode, num_mem_images, render_once, vidseq_local_context_size, keyframe_interval,
                            slam_local_context_size, subsample, min_conf_keyframe, keyframe_overlap_thr,
                            overlap_percentile,  # execution params
                            min_conf_thr, as_pointcloud, transparent_cams, local_pointmaps, cam_size,
                            camera_conf_thr=0.0,  # output params
                            loaded_files=""):
    """gradio.py:159-217 -> (scene, outfile).  Modes: 'linseq', 'vidseq', 'vidslam', and any other (the unordered
    mode) with linspace keyframes.  With should_save_glb the point cloud at min_conf_thr is written to
    outdir/scene.ply (there is no GLB export) and outfile is its path."""
    if filelist:
        image_list = filelist
    elif loaded_files:
        image_list = loaded_files.split("\n")
    else:
        return None, None

    if execution_mode == "vidseq" or execution_mode == "vidslam":
        if execution_mode == "vidseq":
            local_context_size = vidseq_local_context_size
            def is_keyframe_function(id, res, scene_state): return (id % keyframe_interval == 0)
            scene_state = None
            def scene_state_update_function(res, scene_state): return scene_state
        else:
            local_context_size = slam_local_context_size
            overlap_mode = "nn-norm"
            is_keyframe_function = functools.partial(
                slam_is_keyframe, subsample, min_conf_keyframe, keyframe_overlap_thr, overlap_percentile, overlap_mode)
            scene_state = get_searcher("kdtree-scipy-quadrant_x2")
            scene_state_update_function = functools.partial(slam_update_scene_state, subsample, min_conf_keyframe)
        scene = must3r_inference_video(model, device, image_size, amp, image_list, max_bs, init_num_images=2,
                                       batch_num_views=1, viser_server=viser_server,
                                       num_refinements_iterations=num_refinements_iterations,
                                       local_context_size=local_context_size, is_keyframe_function=is_keyframe_function,
                                       scene_state=scene_state, scene_state_update_function=scene_state_update_function,
                                       verbose=verbose)
    else:
        is_sequence = (execution_mode == "linseq")
        scene = must3r_inference(model, retrieval, device, image_size, amp, image_list,
                                 num_mem_images, max_bs, init_num_images=2, batch_num_views=1, render_once=render_once,
                                 is_sequence=is_sequence, viser_server=viser_server,
                                 num_refinements_iterations=num_refinements_iterations,
                                 verbose=verbose)
    if verbose:
        print('preparing pointcloud')
    time_start = datetime.datetime.now()
    outfile = None
    if should_save_glb:
        get_3D_model_from_scene(outdir, verbose, scene, min_conf_thr, as_pointcloud, transparent_cams,
                                local_pointmaps, cam_size, camera_conf_thr=camera_conf_thr, filename='scene.ply')
        outfile = os.path.join(outdir, 'scene.ply')
    if verbose:
        print(f'pointcloud prepared in {datetime.datetime.now() - time_start}')
    return scene, outfile
