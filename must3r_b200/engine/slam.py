"""Online SLAM front end of the reference (must3r/slam/model.py: SLAM_MUSt3R, MUSt3R_Agent, forward_must3r,
get_camera_pose, postproc_pred, ...) with the same names, arguments and results, on the CUDA model.

After the decoder call a frame costs two kernels of csrc/slam.cu and one wait: `m3r_slam_pose` (Weiszfeld focal, the
in-place depth rectification, weighted Procrustes, confidence mean and median), the quadrant ids and grid query of the
keyframe searcher (engine/keyframes.py), `m3r_slam_keyframe` (overlap percentile and keyframe decision), then one
asynchronous device-to-host copy of the frame's record and of the arrays `__call__` returns, and one wait for it.  A frame
that is not a keyframe synchronises nowhere else; a keyframe also adds its confident points to the searcher.  The tail
comes in two halves around that wait, `_launch_tail` and `_finish_tail` (on the agent: `launch_tail` / `finish_tail`), and
`SLAM_MUSt3R._record_frame` does the frame's host bookkeeping, so that engine/slam_sessions.py can put one wait behind
several sessions' tails.

The decoder computes a memory update for every frame; a frame that is not a keyframe gives the rows it appended back
(`_release_tail`), so the next update appends in place onto the memory that was kept.

Deliberate differences from the reference:
  * `forward_must3r` does not call `torch.cuda.empty_cache()` (the reference does, every frame): returning the caching
    allocator's blocks to the driver and allocating them again costs time and changes no result.
  * `postproc_pred` returns the full point map and the colours as (pinned) host tensors, copied with the record; the
    reference's callers only ever move them to the host.  The focal it returns is a host array.
  * The pose of a frame is kept as the record's c2w; the reference stores `inverse(inverse(c2w))`.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import ops
from ..model import get_pointmaps_activation, load_model
from . import memory_io
from .images import preproc_frame
from .inference import _release_tail, _reserve, _sync_host_copies, _to_out, _with_host_shape, postprocess
from .keyframes import choose_keyframe_from_overlap, get_overlap_score, get_searcher  # noqa: F401  (reference names)


# ------------------------------------------------------------------------------------------- trajectory smoothing
def laplacian_smoothing(trajectory, alpha=0.5, iterations=10):
    """must3r/slam/tools.py:34-41: Gauss-Seidel sweeps moving every inner point towards the mean of its neighbours
    (each sweep already sees the points it updated before); the two end points stay."""
    out = np.array(trajectory, copy=True)
    for _ in range(iterations):
        for i in range(1, len(out) - 1):
            out[i] = (1 - alpha) * out[i] + (alpha / 2) * (out[i - 1] + out[i + 1])
    return out


def laplacian_smoothing_with_confidence(trajectory, confidence, alpha=0.5, iterations=10):
    """must3r/slam/tools.py:44-63: the same sweeps with normalised weights (1 - alpha) c_i for the point itself and
    alpha (1 - c_j) / 2 for each neighbour j: a confident point moves less, a confident neighbour pulls less."""
    out = np.array(trajectory, copy=True)
    c = np.asarray(confidence)
    for _ in range(iterations):
        for i in range(1, len(out) - 1):
            w = np.array([alpha * (1 - c[i - 1]) / 2, (1 - alpha) * c[i], alpha * (1 - c[i + 1]) / 2])
            w = w / w.sum()
            out[i] = w[1] * out[i] + w[0] * out[i - 1] + w[2] * out[i + 1]
    return out


# ------------------------------------------------------------------------------------------- per-frame processing
@torch.no_grad()
def forward_must3r(model, input_views, memory, render=False, device='cuda:0'):
    """must3r/slam/model.py:22-59: encode each view, one decoder call over all of them, postprocess each prediction.
    true_shape stays on the host (the CUDA model reads it there), so the call makes no host-to-device copy of it."""
    encoder, decoder = model
    xs, poss, shapes = [], [], []
    for view in input_views:
        ts = torch.as_tensor(np.asarray(view['true_shape'])).reshape(-1, 2)
        x, pos = encoder(view['img'].to(device), ts)
        xs.append(x[None])
        poss.append(pos[None])
        shapes.append(_with_host_shape(ts, device))
    new_memory, preds = decoder(xs, poss, shapes, memory, render=render)
    act = get_pointmaps_activation(decoder, verbose=False)
    return [postprocess(pred, pointmaps_activation=act) for pred in preds], new_memory


def mean_focal(seq_focals):
    """must3r/slam/model.py:131-137: confidence-weighted mean of the focals so far (None before the first frame)."""
    if not len(seq_focals['f']):
        return None
    f, c = np.array(seq_focals['f']), np.array(seq_focals['conf'])
    return (f * c / c.sum()).sum()


def _pose_record(res, seq_focal, is_first_frame=False, rectify=True, rec=None):
    """m3r_slam_pose over the views of res (pts3d, pts3d_local, conf [1,B,H,W,...]): device records [B, 160] (into
    `rec` if given)."""
    return ops.slam_pose(res['pts3d'][0], res['pts3d_local'][0], res['conf'][0],
                         seq_focal=seq_focal if rectify else None, is_first=is_first_frame, rec=rec)


def get_camera_pose(res, seq_focal, HW, is_first_frame=False, rectify=True):
    """must3r/slam/model.py:147-172 -> (c2w [B,4,4], focal [B]) on the device.  Like the reference, pts3d_local's depth
    is scaled in place by seq_focal / focal (unless is_first_frame), so later readers see the rectified depth."""
    rec = _pose_record(res, seq_focal, is_first_frame, rectify)
    focal = rec[:, 128:132].view(torch.float32).reshape(-1)
    return ops.slam_record_c2w(rec), focal


_COLOR_NORM = {}


def prep_imgs(cimg, img_mean, img_std):
    """must3r/slam/model.py:94-96: ImgNorm images [B,3,H,W] back to colours [B,H,W,3] in [0,1].  The per-channel
    constants are uploaded once per device (the reference uploads them on every call, a synchronising copy)."""
    key = (cimg.device, tuple(img_mean), tuple(img_std))
    if key not in _COLOR_NORM:
        _COLOR_NORM[key] = (torch.tensor(img_std, device=cimg.device), torch.tensor(img_mean, device=cimg.device))
    std, mean = _COLOR_NORM[key]
    return cimg.permute(0, 2, 3, 1) * std + mean


def _wait_host_copies():
    """The one wait of a frame: the record and the returned arrays are on the host after it."""
    _sync_host_copies()


def _index_ready(tree, device):
    """Build the keyframe searcher's grid index now, on a keyframe, rather than at the next frame's query."""
    grid = getattr(tree, 'grid', None)
    if grid is not None and grid._grid is None and len(grid) > 0:
        if not hasattr(tree, 'uses_brute_force') or not tree.uses_brute_force():
            grid._build(torch.device(device))


def _launch_tail(img, res, is_first_frame, seq_focal, overlap_mode, overlap_tree, kf_x_subsamp, keyframe_overlap_thr,
                 min_conf_keyframe, overlap_percentile, img_mean, img_std, rec=None):
    """The device half of postproc_pred, which never waits: m3r_slam_pose into `rec` (a new [1, 160] record unless
    given, e.g. a row of a batch of records), the searcher query, m3r_slam_keyframe and the asynchronous host copies of
    the point map and the colours.  -> the tail that _finish_tail takes once the record is on the host."""
    assert res['pts3d'].shape[0] == 1 and res['pts3d'].shape[1] == 1, "frames come one by one here"
    conf = res['conf'][0, 0]
    s = kf_x_subsamp or 1
    rec = _pose_record(res, seq_focal, is_first_frame, rec=rec)
    c2w = ops.slam_record_c2w(rec)[0]
    sub = res['pts3d'][0, 0, ::s, ::s].reshape(-1, 3)
    dists = None
    if ops.overlap_mode_id(overlap_mode) <= 1:
        dists = overlap_tree.query(sub, cam_center=c2w[:3, -1]).float().contiguous()
    ops.slam_keyframe(dists, conf, res['pts3d_local'][0, 0], rec, subsamp=s, mode=overlap_mode,
                      percentile=overlap_percentile, thr=keyframe_overlap_thr, min_conf_keyframe=min_conf_keyframe,
                      is_first=bool(is_first_frame))
    cols = prep_imgs(img['img'], img_mean=img_mean, img_std=img_std)[None]
    host = [_to_out(t, 'cpu') for t in (res['pts3d'][0, 0], cols)]
    return rec, c2w, sub, conf[::s, ::s], min_conf_keyframe, host


def _finish_tail(res, tail, r):
    """The host half of postproc_pred: the launched `tail` and the frame's host record r -> postproc_pred's tuple; sets
    res['overlap_score'], res['slam_record'] (r) and res['slam_c2w'] (the pose on the device)."""
    rec, c2w, sub, conf_sub, min_conf_keyframe, host = tail
    # the confident subsampled points, in pixel order: a stable sort of the mask puts them first (no host sync)
    msk = conf_sub.reshape(-1) > min_conf_keyframe
    pts = sub[torch.argsort((~msk).to(torch.uint8), stable=True)[:int(r['n_conf'])]]
    res['overlap_score'] = float(r['score'])
    res['slam_record'] = r
    res['slam_c2w'] = c2w
    w2c = rec[0, 64:128].view(torch.float32).view(4, 4)
    return (pts, host[0], host[1], res['pts3d_local'][0, 0, ..., -1], res['conf'][0, 0],
            np.array([r['focal']], dtype=np.float32), w2c, c2w[:3, -1], bool(r['keyframe']))


def postproc_pred(img, res, is_first_frame, seq_focals, fixed_focal=True, overlap_mode='nn-norm', overlap_tree=None,
                  kf_x_subsamp=None, keyframe_overlap_thr=.15, min_conf_keyframe=1.5, overlap_percentile=70,
                  img_mean=[0.5, 0.5, 0.5], img_std=[0.5, 0.5, 0.5]):
    """must3r/slam/model.py:185-248 -> (pts, allpts, cols, depth, conf, focal, w2c, cam_center, iskeyframe).
    Reads the frame's record back once; also sets res['overlap_score'], res['slam_record'] (the host record) and
    res['slam_c2w'] (the pose on the device)."""
    seq_focal = mean_focal(seq_focals) if fixed_focal else None
    tail = _launch_tail(img, res, is_first_frame, seq_focal, overlap_mode, overlap_tree, kf_x_subsamp,
                        keyframe_overlap_thr, min_conf_keyframe, overlap_percentile, img_mean, img_std)
    host_rec = _to_out(tail[0], 'cpu')
    _wait_host_copies()
    return _finish_tail(res, tail, host_rec.numpy().view(ops.SLAM_RECORD)[0, 0])


class MUSt3R_Agent():
    """must3r/slam/model.py:251-317: one camera's focal bookkeeping."""

    def __init__(self, fixed_focal=True, smooth_focal_changes=False, img_mean=[0.5, 0.5, 0.5], img_std=[0.5, 0.5, 0.5]):
        assert fixed_focal or not smooth_focal_changes, "online focal smoothing with varying focals is not supported"
        self.fixed_focal = fixed_focal
        self.smooth_focal_changes = smooth_focal_changes
        self.img_mean = img_mean
        self.img_std = img_std
        self.reset()

    def reset(self):
        self.seq_focals = {'f': [], 'conf': [], 'to_orig': []}

    def get_true_focal(self):
        """The focal in the original frame's pixels: the weighted mean (fixed focal) or the per-frame list."""
        if len(self.seq_focals['f']) == 0:
            return None
        if self.fixed_focal:
            to_orig = self.seq_focals['to_orig']
            assert all(t == to_orig[0] for t in to_orig), "To orig should be constant for a single true focal"
            return mean_focal(self.seq_focals) * to_orig[0]
        return [f * t for f, t in zip(self.seq_focals['f'], self.seq_focals['to_orig'])]

    def add_focal(self, r, to_orig_focal):
        """Record the focal and confidence of a frame's host record r -> the focal the frame reports: the weighted mean
        so far (fixed focal) or its own."""
        self.seq_focals['f'].append(np.float32(r['focal']))
        self.seq_focals['to_orig'].append(to_orig_focal)
        self.seq_focals['conf'].append(np.float32(r['conf_mean']) - 1.)
        return mean_focal(self.seq_focals) if self.fixed_focal else self.seq_focals['f'][-1]

    def launch_tail(self, inp, pred, is_first_frame, overlap_mode, overlap_tree, kf_x_subsamp, keyframe_overlap_thr,
                    min_conf_keyframe, overlap_percentile, rec=None):
        """The device half of `update` (it never waits), with this agent's focal; `rec` as in _launch_tail."""
        return _launch_tail(inp, pred, is_first_frame, mean_focal(self.seq_focals) if self.fixed_focal else None,
                            overlap_mode, overlap_tree, kf_x_subsamp, keyframe_overlap_thr, min_conf_keyframe,
                            overlap_percentile, self.img_mean, self.img_std, rec=rec)

    def finish_tail(self, pred, tail, r, to_orig_focal):
        """The host half of `update` once the frame's record r is on the host -> update's tuple."""
        out = _finish_tail(pred, tail, r)
        return out[:5] + (self.add_focal(r, to_orig_focal),) + out[6:]

    @torch.no_grad()
    def update(self, inp, pred, is_first_frame, overlap_mode, overlap_tree, kf_x_subsamp, keyframe_overlap_thr,
               min_conf_keyframe, overlap_percentile, to_orig_focal):
        out = postproc_pred(
            img=inp, res=pred, is_first_frame=is_first_frame, seq_focals=self.seq_focals, fixed_focal=self.fixed_focal,
            overlap_mode=overlap_mode, overlap_tree=overlap_tree, kf_x_subsamp=kf_x_subsamp,
            keyframe_overlap_thr=keyframe_overlap_thr, min_conf_keyframe=min_conf_keyframe,
            overlap_percentile=overlap_percentile, img_mean=self.img_mean, img_std=self.img_std)
        return out[:5] + (self.add_focal(pred['slam_record'], to_orig_focal),) + out[6:]


def get_map(ptscolsconfs, confthr):
    """must3r/slam/model.py:175-182: the stored keyframes' points and colours with conf > confthr."""
    pts = [p[c > confthr] for p, _, c in ptscolsconfs]
    cols = [col[0, 0, c > confthr] for _, col, c in ptscolsconfs]
    return torch.cat(pts), torch.cat(cols)


class SLAM_MUSt3R():
    """must3r/slam/model.py:320-528: the memory manager of the online SLAM.  Frames go to their camera's agent; keyframes
    extend the decoder memory and the searcher's point map.  The memory can be saved and loaded for later runs."""

    def __init__(self, chkpt, res=512, searcher='kdtree-scipy-quadrant_x2', overlap_mode='nn-norm', kf_x_subsamp=4,
                 keyframe_overlap_thr=.15, min_conf_keyframe=1.5, overlap_percentile=70., rerender=False, fixed_focal=True,
                 keep_memory=False, load_memory=None, num_agents=1, device='cuda:0', num_init_frames=2):
        self.agents = [MUSt3R_Agent(fixed_focal) for _ in range(num_agents)]
        self.num_init_frames = num_init_frames
        self.res = res
        self.device = device
        self.model = self._load_model(chkpt, device)
        self.searcher = searcher
        self.kf_x_subsamp = kf_x_subsamp
        self.keyframe_overlap_thr = keyframe_overlap_thr
        self.min_conf_keyframe = min_conf_keyframe
        self.overlap_percentile = overlap_percentile
        self.overlap_mode = overlap_mode
        self.rerender = rerender
        self.keep_memory = keep_memory
        self.memory_memory = None
        self.memory_map = None
        self.memory_data = []
        self.memory_overlap_tree = None
        if load_memory is not None:
            self.load_memory(load_memory)
        self.reset()

    def _load_model(self, chkpt, device):
        model = load_model(chkpt, device=device)
        _reserve(model[1], 0, 1.5)               # memory buffers grow geometrically: updates append in place
        return model

    def reset(self):
        """Back to the loaded memory if there is one, else to an empty map."""
        self.all_poses = []
        self.all_confs = []
        self.all_timestamps = []
        self.memory = self.memory_memory
        self.keyframe_pointmaps = self.memory_data
        self.keyframes = []
        if self.memory_overlap_tree is None:
            self.overlap_tree = get_searcher(self.searcher if 'nn' in self.overlap_mode else 'none')
        else:
            self.overlap_tree = self.memory_overlap_tree
        self.all_images = []
        self.all_pts3d = None
        self.mem_was_loaded = self.memory_memory is not None
        for agent in self.agents:
            agent.reset()

    @property
    def num_mem_frames(self):
        return len(self.keyframes)

    def get_true_focals(self):
        return {agid: agent.get_true_focal() for agid, agent in enumerate(self.agents)}

    def write_all_poses(self, path, filtering_mode=None, filtering_steps=5, filtering_alpha=.5, **tolog):
        """must3r/slam/model.py:408-429: npz with poses [N,4,4] (c2w), timestamps, confs (mean confidence per frame),
        focal (get_true_focals) and any extra arrays; optionally the camera centres smoothed ('laplacian',
        'laplacian-conf': weights = the confidences rescaled to [0, 1])."""
        print(f"Writing full trajectory in {path}")
        all_poses = torch.stack(self.all_poses).cpu().numpy()
        timestamps = np.stack(self.all_timestamps).astype(int)
        conf = torch.stack(self.all_confs).cpu().numpy()
        focals = self.get_true_focals()
        if filtering_mode is not None:
            if 'laplacian' not in filtering_mode:
                raise ValueError(f"Unknown filtering mode {filtering_mode}")
            trajectory = all_poses[:, :3, -1]
            if 'conf' in filtering_mode:
                remap = (conf - conf.min()) / (conf.max() - conf.min())
                trajectory = laplacian_smoothing_with_confidence(trajectory, remap, alpha=filtering_alpha,
                                                                 iterations=filtering_steps)
            else:
                trajectory = laplacian_smoothing(trajectory, alpha=filtering_alpha, iterations=filtering_steps)
            all_poses[:, :3, -1] = trajectory
        np.savez(path, poses=all_poses, timestamps=timestamps, confs=conf, focal=focals, **tolog)

    def save_memory(self, output):
        memory_io.save_memory(output, self.memory, self.keyframe_pointmaps, self.overlap_tree)

    def load_memory(self, mem_file):
        self.memory_memory, self.memory_data, self.memory_overlap_tree = memory_io.load_memory(mem_file, device=self.device)
        self.memory = self.memory_memory
        self.keyframe_pointmaps = self.memory_data
        self.overlap_tree = self.memory_overlap_tree
        self.mem_was_loaded = True

    def fetch_memory_map(self, conf_thr):
        if self.mem_was_loaded:
            self.memory_map = get_map(self.memory_data, conf_thr)
            self.mem_was_loaded = False
        return self.memory_map

    @torch.no_grad()
    def rerender_all_frames(self, maxbs=64):
        """Once the sequence is done (rerender=True), predict every frame again from the full memory, in batches of
        maxbs, and recompute all poses in one batched m3r_slam_pose with the sequence's focal."""
        assert len(self.agents) == 1, "rerendering with several agents (different focal lengths) is not supported"
        if not self.rerender:
            return
        preds = []
        for lo in range(0, len(self.all_images), maxbs):
            sel = self.all_images[lo:lo + maxbs]
            batch = {'img': torch.cat([im['img'] for im in sel]),
                     'true_shape': np.concatenate([im['true_shape'] for im in sel])}
            out, _ = forward_must3r(self.model, [batch], self.memory, render=True, device=self.device)
            preds.append(out[0])
        res = {k: torch.cat([p[k] for p in preds], dim=1).contiguous() for k in ('pts3d', 'pts3d_local', 'conf')}
        c2w, _ = get_camera_pose(res, mean_focal(self.agents[0].seq_focals), HW=None, is_first_frame=False)
        self.all_pts3d = res['pts3d'].cpu()
        self.all_poses = list(c2w)

    @torch.no_grad()
    def __call__(self, img, frame_id, cam_id):
        """must3r/slam/model.py:480-528 -> (pts3d [H,W,3], colors [1,1,H,W,3] numpy, depth, conf, focal, w2c, HW,
        iskeyframe)."""
        query_view_prep, to_orig_focal = preproc_frame(img, frame_id, res=self.res, device=self.device)
        if self.memory is not None and len(self.all_images) < self.num_init_frames:
            # initialisation not complete: start again from the loaded memory with the earlier frames re-run
            other_init_images = self.all_images
            frame_ids = self.all_timestamps
            self.reset()
            self.all_images = other_init_images.copy()
        else:
            other_init_images = []
            frame_ids = []
        if self.rerender or len(self.all_images) < self.num_init_frames:
            self.all_images.append(query_view_prep)
        query_images = other_init_images + [query_view_prep]
        frame_ids = frame_ids + [frame_id]
        preds, newmem = forward_must3r(self.model, query_images, self.memory, device=self.device)
        kept = False
        for view, pred, fid in zip(query_images, preds, frame_ids):
            out = self.agents[cam_id].update(
                view, pred, self.memory is None, overlap_mode=self.overlap_mode, overlap_tree=self.overlap_tree,
                kf_x_subsamp=self.kf_x_subsamp, keyframe_overlap_thr=self.keyframe_overlap_thr,
                min_conf_keyframe=self.min_conf_keyframe, overlap_percentile=self.overlap_percentile,
                to_orig_focal=to_orig_focal)
            if out[-1]:
                self.memory = newmem
                kept = True
            ret = self._record_frame(view, pred, fid, out)
        if not kept:
            _release_tail(self.memory)        # the update of a frame that is not a keyframe is dropped
        return ret

    def _record_frame(self, view, pred, fid, out, build_index=True):
        """Host bookkeeping of a frame once its record is known (out = the agent's update tuple; the caller updates the
        memory): its timestamp, pose and confidence; on a keyframe its id, its confident points in the searcher (and,
        unless build_index is False, the searcher's index rebuilt now) and, with keep_memory, its point map.  -> what
        __call__ returns for the frame."""
        selpts3d, pts3d, colors, depth, conf, focal, w2c, cam_center, iskeyframe = out
        self.all_timestamps.append(fid)
        self.all_poses.append(pred['slam_c2w'])
        self.all_confs.append(torch.tensor(pred['slam_record']['conf_mean']))
        if iskeyframe:
            self.keyframes.append(fid)
            if self.overlap_tree is not None:
                self.overlap_tree.add_pts(selpts3d, cam_center=cam_center)
                if build_index:
                    _index_ready(self.overlap_tree, self.device)
            if self.keep_memory:
                self.keyframe_pointmaps.append([pts3d.cpu(), colors.cpu(), conf.cpu()])
        return pts3d.cpu().numpy(), colors.cpu().numpy(), depth, conf, focal, w2c, view['true_shape'][0], iskeyframe
