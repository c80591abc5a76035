"""One online SLAM run whose map several cameras build together (the reference's SLAM_MUSt3R with one agent per camera,
must3r/slam/model.py), with the frames of all cameras batched into one encoder and one decoder call per step.

The reference feeds the cameras' frames one at a time (AutoMultiLoader: camera 0, 1, ..., K-1, skipping a camera that
has run out), so each camera's frame rate is the single-camera rate divided by K.  `MultiCameraSLAM.step({cam_id: (frame,
frame_id)})` takes the next frame of every camera that still has frames and returns, per camera, what
SLAM_MUSt3R.__call__ returns for it.

Step semantics: every batched frame is decoded against the memory, and keyframe-tested against the searcher's point map,
as they stood before the step, with its own camera's agent (its focal state); at the end of the step the keyframes are
appended to the memory in camera order, as images nimgs, nimgs + 1, ..., their points go to the searcher and their point
maps (keep_memory) are kept in the same order.  With one camera this is SLAM_MUSt3R, bit for bit.  With several, the one
difference from the reference is that a frame does not see a keyframe taken earlier in the same step: two cameras that
look at new ground at the same instant may both become keyframes where the reference would take only the first.

Batching rule (plan_batch of engine/slam_sessions.py): the step's frames are batched when the memory is non-empty, the
run is past the initialisation re-runs (`num_init_frames`, after a fresh start or load_memory), the decoder keeps its
memory as K|V rows (memory_mode 'kv'), and a frame's preprocessed shape is the shape most frames of the step share.  The
batch costs one encoder call, one decoder call in which the F frames read the one memory through a stride-0 scene
dimension (no copy of it; the attention launches the frames that read the same key tiles together, csrc/attention.cu),
one pose launch over the F frames with each camera's own focal state (m3r_slam_pose_views), one searcher query over all
frames' subsampled points, one keyframe launch writing F records (m3r_slam_keyframe_frames), one
m3r_mem_commit_ordered that appends the keyframes' rows in camera order with the keyframe flags read on the device, and
one wait for all records and returned arrays.  The host then counts the keyframes, updates the labels, nimgs and the
length, and runs SLAM_MUSt3R._record_frame for each frame in camera order, rebuilding the searcher's index once if any
keyframe was taken.  Every other frame (another preprocessed shape in a step that batches the rest) runs alone through
SLAM_MUSt3R.__call__ after the batch, in camera order: its timestamp, pose and keyframe are recorded after the batch's,
and it sees the batch's keyframes.

Memory: one [1, cap, 2D] buffer per level (SessionArena of engine/slam_sessions.py with one slot), grown geometrically
before a step that could overflow it; the run's `memory` is the reference's 5-tuple of views of it, so save_memory,
pickling and load_memory work unchanged.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import numpy as np
import torch

from .. import _lib, ops
from ..model import get_pointmaps_activation
from ..model import common as cm
from . import slam
from .images import preproc_frame
from .inference import _to_out, postprocess
from .keyframes import QuadrantSearcher, get_quadrant_id
from .slam import SLAM_MUSt3R, _index_ready, mean_focal, prep_imgs
from .slam_sessions import KEYFRAME_OFFSET, SLAMSessions, plan_batch

MAX_CAMERAS = 64         # M3R_MAX_COMMIT: frames per m3r_mem_commit_ordered launch


def steps_of(items):
    """Split the reference's frame order [(path, cam_id, timestamp)] (engine/frames.py schedule) into steps: a step ends
    where a camera would give its second frame.  -> [[item, ...] per step], each step in camera order."""
    steps = []
    for it in items:
        if not steps or any(it[1] == o[1] for o in steps[-1]):
            steps.append([])
        steps[-1].append(it)
    return steps


def commit_rows(keyframe, row0, N):
    """The rows m3r_mem_commit_ordered writes frame k's N new rows to: row0 + N * (keyframes among frames < k), or None
    when frame k is not a keyframe.  -> (rows per frame, the memory's new length)."""
    rows, n = [], row0
    for kf in keyframe:
        rows.append(n if kf else None)
        n += N if kf else 0
    return rows, n


def query_frames(tree, subs, centers):
    """The keyframe searcher's distances of F frames' subsampled points subs [F, Q, 3], each frame's points bucketed by
    the viewing direction from its own camera centre centers [F, 3], in one query -> [F * Q], bitwise F `tree.query`
    calls (the distances of a point depend on nothing but the point, its bucket and the map)."""
    pts = subs.reshape(-1, 3)
    if isinstance(tree, QuadrantSearcher):
        rays = (subs.float() - centers.reshape(-1, 1, 3).to(subs.device).float()).reshape(-1, 3)
        return tree.grid.query(pts, get_quadrant_id(rays, tree.quadrant_divider))
    return tree.query(pts)


class MultiCameraSLAM(SLAMSessions):
    """K cameras building one map: one SLAM_MUSt3R (`.slam`) with num_agents = K on the shared model.  `kwargs` are
    SLAM_MUSt3R's constructor arguments without chkpt, device and num_agents.  Attributes and methods that are not the
    batched step's (save_memory, write_all_poses, load_memory, get_true_focals, keyframes, all_poses, ...) are the
    SLAM_MUSt3R's."""

    def __init__(self, chkpt, num_cameras=1, device='cuda:0', **kwargs):
        if not 1 <= num_cameras <= MAX_CAMERAS:
            raise ValueError(f"num_cameras must be in [1, {MAX_CAMERAS}]")
        if kwargs.get('rerender') and num_cameras > 1:
            raise ValueError("rerendering with several cameras (different focal lengths) is not supported")
        super().__init__(chkpt, 1, device=device, num_agents=num_cameras, **kwargs)

    @property
    def slam(self):
        return self.sessions[0]

    def __getattr__(self, name):
        if name == 'sessions':
            raise AttributeError(name)
        return getattr(self.sessions[0], name)

    @torch.no_grad()
    def step(self, frames: Dict[int, tuple]):
        """frames: {cam_id: (frame, frame_id)} -> {cam_id: SLAM_MUSt3R.__call__'s result}, in camera order."""
        s = self.slam
        cams = sorted(frames)
        for c in cams:
            if not 0 <= c < len(s.agents):
                raise ValueError(f"camera {c}: this run has {len(s.agents)} cameras")
        together = self.kv and not s.runs_alone() and self.arena.lengths[0] > 0 and self.arena.holds(0, s.memory[0])
        cands, prepped = {}, {}
        for c in cams:
            if not together:
                cands[c] = None
                continue
            img, fid = frames[c]
            view, to_orig = preproc_frame(img, fid, res=s.res, device=s.device)
            prepped[c] = (view, to_orig)
            cands[c] = tuple(int(v) for v in np.asarray(view['true_shape']).reshape(-1)[:2])
        batch, alone = plan_batch(cands)
        out = {}
        if batch:
            out.update(self._step_cameras(batch, frames, prepped))
        for c in alone:
            img, fid = frames[c]
            out[c] = SLAM_MUSt3R.__call__(s, img, fid, c)
            self._to_slot(s)
        self.stats['batched'] += len(batch)
        self.stats['alone'] += len(alone)
        return {c: out[c] for c in cams}

    def _decode_shared(self, batch, prepped):
        """One encoder call over the batch's frames, then one decoder call in which every frame attends to the one
        memory (a stride-0 view of slot 0).  -> (res {pts3d, pts3d_local, conf} [F,1,H,W,..] in batch order, staged new
        rows, list[depth] of [F, N, 2D])."""
        encoder, decoder = self.model
        views = [prepped[c][0] for c in batch]
        imgs = torch.cat([v['img'] for v in views]).to(self.device)
        ts = torch.as_tensor(np.concatenate([np.asarray(v['true_shape']).reshape(-1, 2) for v in views]))
        x, pos = encoder(imgs, ts)
        F, N = x.shape[0], x.shape[1]
        n = self.arena.lengths[0]
        if self.arena.ensure(n + F * N):            # room for every frame of the step being a keyframe
            self._repoint()
        shape = ts.view(F, 1, 2)
        shape._m3r_hw = tuple(int(v) for v in ts[0].tolist())
        mem = ([b[0:1, :n].expand(F, -1, -1) for b in self.arena.bufs], None, 0, 0, 0)
        new_tokens, pm = decoder.update_tokens(x[:, None], pos[:, None], shape, current_mem=mem)
        return postprocess(pm, pointmaps_activation=get_pointmaps_activation(decoder, verbose=False)), new_tokens

    def _commit_ordered(self, new_tokens, recs):
        """m3r_mem_commit_ordered: the rows of the frames whose record says keyframe, behind the memory in batch order."""
        depth = self.arena.depth
        arena = (C.c_void_p * depth)(*[b.data_ptr() for b in self.arena.bufs])
        src = (C.c_void_p * depth)(*[t.data_ptr() for t in new_tokens])
        F, N = new_tokens[0].shape[:2]
        _lib.check(_lib.lib().m3r_mem_commit_ordered(arena, src, depth, F, N, self.arena.width, self.arena.lengths[0],
                                                     C.c_void_p(recs.data_ptr() + KEYFRAME_OFFSET), recs.shape[1] // 4,
                                                     cm.stream_ptr(recs.device)), "mem_commit_ordered")

    def _launch_tails(self, batch, res, prepped, recs):
        """The device half of the agents' `update` for the F frames of the batch at once, which never waits: one
        m3r_slam_pose_views with each camera's focal, one searcher query over all frames' subsampled points, one
        m3r_slam_keyframe_frames into recs [F, record], and the asynchronous host copies of each frame's point map and
        colours.  -> per frame the tail MUSt3R_Agent.finish_tail takes (that of MUSt3R_Agent.launch_tail)."""
        s = self.slam
        F = len(batch)
        pts, loc, conf = res['pts3d'][:, 0], res['pts3d_local'][:, 0], res['conf'][:, 0]
        seq = [mean_focal(s.agents[c].seq_focals) if s.agents[c].fixed_focal else None for c in batch]
        ops.slam_pose_views(pts, loc, conf, seq, [False] * F, rec=recs)
        c2w = ops.slam_record_c2w(recs)
        sub = s.kf_x_subsamp or 1
        subs = pts[:, ::sub, ::sub].reshape(F, -1, 3)
        dists = None
        if ops.overlap_mode_id(s.overlap_mode) <= 1:
            dists = query_frames(s.overlap_tree, subs, c2w[:, :3, -1]).float().contiguous()
        ops.slam_keyframe_frames(dists, conf, loc, recs, subsamp=sub, mode=s.overlap_mode, percentile=s.overlap_percentile,
                                 thr=s.keyframe_overlap_thr, min_conf_keyframe=s.min_conf_keyframe, is_first=[False] * F)
        tails = []
        for i, c in enumerate(batch):
            agent = s.agents[c]
            cols = prep_imgs(prepped[c][0]['img'], img_mean=agent.img_mean, img_std=agent.img_std)[None]
            host = [_to_out(t, 'cpu') for t in (pts[i], cols)]
            tails.append((recs[i:i + 1], c2w[i], subs[i], conf[i, ::sub, ::sub], s.min_conf_keyframe, host))
        return tails

    def _step_cameras(self, batch, frames, prepped):
        s = self.slam
        res, new_tokens = self._decode_shared(batch, prepped)
        recs = torch.empty((len(batch), ops.SLAM_RECORD.itemsize), dtype=torch.uint8, device=torch.device(self.device))
        preds = [{k: res[k][i:i + 1] for k in ('pts3d', 'pts3d_local', 'conf')} for i in range(len(batch))]
        tails = self._launch_tails(batch, res, prepped, recs)
        self._commit_ordered(new_tokens, recs)
        host_recs = _to_out(recs, 'cpu')
        slam._wait_host_copies()
        records = host_recs.numpy().view(ops.SLAM_RECORD)[:, 0]
        N = new_tokens[0].shape[1]
        out, any_keyframe = {}, False
        for i, c in enumerate(batch):
            _, fid = frames[c]
            view, to_orig = prepped[c]
            frame_out = s.agents[c].finish_tail(preds[i], tails[i], records[i], to_orig)
            if s.rerender:
                s.all_images.append(view)
            if frame_out[-1]:
                self._append(s, N)                 # the rows m3r_mem_commit_ordered wrote for it (commit_rows)
                any_keyframe = True
            out[c] = s._record_frame(view, preds[i], fid, frame_out, build_index=False)
        if any_keyframe and s.overlap_tree is not None:
            _index_ready(s.overlap_tree, s.device)       # one rebuild for all the step's keyframes
        return out
