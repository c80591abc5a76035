"""Several videos (must3r_inference_video's vidseq and vidslam schedules) reconstructed in lockstep on one model and one GPU.

`reconstruct_videos(model, device, image_size, amp, filelists, execution_mode, max_bs, ...)` returns, for every image
list, the SceneState that `demo.get_reconstructed_scene(..., execution_mode=...)` returns for that list alone
(must3r_inference_video with init_num_images=2, batch_num_views=1 and the mode's keyframe test), but the scenes share
their calls:

  * All frames of all scenes are encoded up front, grouped by shape (lockstep._encode).
  * Step k of every scene that has one runs in shared decoder calls: the scenes whose step views have the same shapes
    share a call, cut into runs of consecutive slots (lockstep_calls).  Step 0 (the init views) is one
    MUSt3R.update_tokens call without a memory; every later step passes the scenes' memory lengths, so each scene attends
    only to its own rows.  The memories live in one SessionArena (engine/lockstep.py), one slot per scene.
  * Keyframes: vidseq's test (id % keyframe_interval == 0) is known on the host, so the frame loop waits for nothing and
    the arena is sized once.  vidslam postprocesses each step's frames together; every scene's searcher query and
    m3r_slam_keyframe fill one row of one record tensor, read back with one wait per step whatever the number of scenes;
    then the keyframes' points go to their scene's searcher.  Its arena grows geometrically.
  * Memory edits come from each scene's VideoPlan, a host replay of inference_video_multi_ar's label bookkeeping.  After a
    step, the rows of the frames that left the rolling window without being keyframes are closed up, in order, by one
    m3r_mem_compact_rows over every scene and level; then the step's rows that stay are written where they belong
    (m3r_mem_commit_rows): behind the scene's memory, or over a keyframe's old rows in a refinement pass (except those of
    the reference view, label 0).  A frame that leaves the window right after its own step (local_context_size=0, not a
    keyframe) is never written.  Between passes only keyframes stay; after the last pass nothing is compacted.
    lockstep.apply_edits applies every scene's StepEdit.
  * Results are those of the last pass.  postprocess(compute_cam=True) runs once per step and view group over all the
    scenes' frames (vidseq: after the frame loop), and every scene's results are copied to the host in one batch of
    asynchronous copies followed by one wait.

`max_bs` keeps its per-scene meaning; with one view per step it only splits the init step's groups (stack_views).
Only memory_mode 'kv' is supported.
"""
from __future__ import annotations

import copy
import datetime
from collections import deque
from typing import List

import numpy as np
import torch

from .. import ops
from ..model import get_pointmaps_activation
from .demo import (SceneState, _amp, _finish_scene, _launch_scene_copies, _load, _mem_batches, _report,
                   slam_update_scene_state)
from .inference import _sync_host_copies, _to_out, postprocess
from .keyframes import choose_keyframe_from_overlap, get_searcher
from .lockstep import (SessionArena, StepEdit, _call_inputs, _encode, _groups, _tokens, apply_edits, lockstep_calls,
                       signature)

OVERLAP_MODE = "nn-norm"        # demo.get_reconstructed_scene's vidslam overlap score
SEARCHER = "kdtree-scipy-quadrant_x2"


def _find(blocks, label):
    return next((i for i, b in enumerate(blocks) if b[0] == label), None)


def _extend(runs, src, dst, n):
    if runs and runs[-1][0] + runs[-1][2] == src and runs[-1][1] + runs[-1][2] == dst:
        runs[-1] = (runs[-1][0], runs[-1][1], runs[-1][2] + n)
    else:
        runs.append((src, dst, n))


class VideoPlan:
    """One video's schedule and memory layout, on the host.  steps[k]: the groups [((H, W), [frames])] of step k (the two
    init frames, then one frame per step), as stack_views groups them; step(it, k, is_keyframe) replays what
    inference_video_multi_ar does to its memory after step k of pass `it` and returns the StepEdit.  The layout (blocks:
    [label, rows] per stored view, in memory order) is the label row of the engine's memory after the same step, with
    the engine's labels: a call's views are labelled in call order, and a refinement pass relabels a non-keyframe with
    its old label."""

    def __init__(self, shapes, local_context_size=0, num_refinements_iterations=0, max_bs=None):
        n = len(shapes)
        if n == 0:
            raise ValueError("a video needs at least one frame")
        self.shapes = [tuple(int(v) for v in np.asarray(s).reshape(-1)[:2]) for s in shapes]
        self.order = list(range(n))                 # (scenes._encode's name for the views to encode)
        self.local_context_size = local_context_size
        self.passes = num_refinements_iterations + 1
        self.mem_batches = _mem_batches(n, 2, 1, n, n)
        self.step_ids, self.steps, lo = [], [], 0
        for b in self.mem_batches:
            ids = list(range(lo, lo + b))
            self.step_ids.append(ids)
            self.steps.append(_groups(self.shapes, ids, max_bs))
            lo += b
        self.blocks = []            # [label, rows] per stored view, in memory order
        self.label_of = {}          # frame -> label
        self.keyframes = []         # in the order they were decided
        self.window = deque()

    @property
    def length(self):
        return sum(n for _, n in self.blocks)

    def label_row(self, blocks=None):
        blocks = self.blocks if blocks is None else blocks
        return np.concatenate([np.full(n, lab, dtype=np.int64) for lab, n, *_ in blocks]) if blocks else \
            np.zeros(0, dtype=np.int64)

    def _evict(self, blocks, vid):
        if vid not in self.keyframes:
            i = _find(blocks, self.label_of[vid])
            if i is not None:
                del blocks[i]

    def final_label_row(self):
        """The label row inference_video_multi_ar's memory has after the last pass (the window emptied of non-keyframes),
        which this engine does not compact: the memory is discarded."""
        blocks = [list(b) for b in self.blocks]
        for vid in self.window:
            self._evict(blocks, vid)
        return self.label_row(blocks)

    def step(self, it, k, is_keyframe=None) -> StepEdit:
        """After step k of pass `it`; is_keyframe(frame) -> bool decides the frames first seen after the init step."""
        ids = self.step_ids[k]
        first = len(self.label_of)                  # the memory's image count: the first label of the call
        blocks, row = [], 0                         # [label, rows, staged?, row in the memory or in the staged block]
        for lab, n in self.blocks:
            blocks.append([lab, n, False, row])
            row += n
        srow = 0
        for j, q in enumerate(q for _, pos in self.steps[k] for q in pos):
            n = _tokens(self.shapes[q])
            blocks.append([first + j, n, True, srow])
            srow += n
        new = [first + j for j in range(len(ids))]
        if it == 0 and k == 0:                      # initialisation: every view is a keyframe
            for j, vid in enumerate(ids):
                self.label_of[vid] = new[j]
                self.window.append(vid)
                self.keyframes.append(vid)
        else:
            for j, vid in enumerate(ids):
                seen = vid in self.label_of
                is_kf = (vid in self.keyframes) if seen else bool(is_keyframe(vid))
                self.window.append(vid)
                if is_kf and seen:                  # refinement pass: the fresh rows replace the keyframe's old ones ...
                    src = _find(blocks, new[j])
                    if self.label_of[vid] != 0:     # ... except the reference view's
                        dst = _find(blocks, self.label_of[vid])
                        assert blocks[dst][1] == blocks[src][1]
                        blocks[dst][2:] = blocks[src][2:]
                    del blocks[src]
                elif seen:                          # known non-keyframe: its rows keep the old label
                    blocks[_find(blocks, new[j])][0] = self.label_of[vid]
                else:
                    self.label_of[vid] = new[j]
                    if is_kf:
                        self.keyframes.append(vid)
        while len(self.window) > self.local_context_size:
            self._evict(blocks, self.window.popleft())
        if k == len(self.steps) - 1 and it < self.passes - 1:      # between passes only keyframes stay
            while self.window:
                self._evict(blocks, self.window.popleft())
        runs, writes, row = [], [], 0
        for lab, n, staged, r in blocks:
            if staged:
                _extend(writes, r, row, n)
            elif r != row:
                _extend(runs, r, row, n)
            row += n
        assert len(writes) <= 1, writes             # one view per step, or the init views side by side
        self.blocks = [[lab, n] for lab, n, _, _ in blocks]
        return StepEdit(runs, writes[0] if writes else None, row)

    def max_rows(self, is_keyframe):
        """The largest memory of the whole schedule for a keyframe test known up front (vidseq)."""
        p, m = copy.deepcopy(self), 0
        for it in range(p.passes):
            for k in range(len(p.steps)):
                m = max(m, p.step(it, k, is_keyframe).length)
        return m


def plan_step_calls(plans: List[VideoPlan], k):
    """The lockstep calls of step k -> [(signature, [slots])] (lockstep_calls)."""
    return lockstep_calls([(s, signature(p.steps[k])) for s, p in enumerate(plans) if k < len(p.steps)])


def _postprocess(parts, act, out):
    """postprocess(compute_cam=True) of one step's pointmaps, parts [(((H, W), group), pointmaps [n, H, W, 7],
    [(scene, frame)])], once per view group of the step over all scenes -> out[scene][frame] = that frame's results.  A
    video batched alone is postprocessed in the batches inference_video_multi_ar uses (the camera fit's reductions are
    not bitwise independent of the batch size)."""
    by_group = {}
    for key, pm, members in parts:
        by_group.setdefault(key, []).append((pm, members))
    for items in by_group.values():
        pm = torch.cat([p for p, _ in items]) if len(items) > 1 else items[0][0]
        res = postprocess(pm, pointmaps_activation=act, compute_cam=True)
        k = 0
        for _, members in items:
            for s, q in members:
                out[s][q] = {key: v[k] for key, v in res.items()}
                k += 1


def _wait_scores():
    """The one wait of a vidslam step: the keyframe records of every scene's frame."""
    _sync_host_copies()


def _slam_decisions(res, searchers, members, dev, subsample, min_conf_keyframe, keyframe_overlap_thr, overlap_percentile):
    """demo.slam_is_keyframe of every (scene, frame) of a step: each scene's query and m3r_slam_keyframe into one row of
    one record tensor, one read-back -> [bool]."""
    recs = torch.zeros((len(members), ops.SLAM_RECORD.itemsize), dtype=torch.uint8, device=dev)
    sub = subsample or 1
    for i, (s, q) in enumerate(members):
        r = res[s][q]
        conf, loc = r['conf'].contiguous(), r['pts3d_local'].contiguous()
        dists = searchers[s].query(r['pts3d'][::sub, ::sub].reshape(-1, 3),
                                   cam_center=r['c2w'][:3, -1]).float().contiguous()
        with torch.cuda.device(dev):
            ops.slam_keyframe(dists, conf, loc, recs[i:i + 1], subsamp=sub, mode=OVERLAP_MODE,
                              percentile=overlap_percentile, thr=keyframe_overlap_thr,
                              min_conf_keyframe=min_conf_keyframe, is_first=False)
    host = _to_out(recs, "cpu")
    _wait_scores()
    scores = host.numpy().view(ops.SLAM_RECORD)[:, 0]['score']
    assert not np.isnan(scores).any()
    return [bool(choose_keyframe_from_overlap(float(v), keyframe_overlap_thr, OVERLAP_MODE)) for v in scores]


@torch.no_grad()
def reconstruct_videos(model, device, image_size, amp, filelists, execution_mode, max_bs, local_context_size=0,
                       keyframe_interval=3, subsample=2, min_conf_keyframe=1.5, keyframe_overlap_thr=0.05,
                       overlap_percentile=85.0, num_refinements_iterations=0, verbose=True) -> List[SceneState]:
    """S independent videos in lockstep (module docstring) -> one SceneState per image list."""
    if execution_mode not in ("vidseq", "vidslam"):
        raise ValueError(f"execution_mode {execution_mode!r}: reconstruct_videos runs 'vidseq' or 'vidslam' "
                         "(engine/scenes.py batches 'linseq')")
    encoder, decoder = model
    if getattr(decoder, "memory_mode", None) != "kv":
        raise NotImplementedError(f"reconstruct_videos batches memories of memory_mode 'kv' only (the decoder's is "
                                  f"{getattr(decoder, 'memory_mode', None)!r}); run must3r_inference_video per video")
    if not filelists:
        return []
    max_bs = None if max_bs == 0 else max_bs
    act = get_pointmaps_activation(decoder, verbose=verbose)
    if verbose:
        print(f'loading images of {len(filelists)} videos')
    time_start = datetime.datetime.now()
    views = [_load(fl, image_size, encoder, verbose, device) for fl in filelists]
    plans = [VideoPlan([v['true_shape'] for v in vs], local_context_size, num_refinements_iterations, max_bs)
             for vs in views]
    if verbose:
        print(f'loaded in {datetime.datetime.now() - time_start}')
        print('running inference')
    time_start = datetime.datetime.now()
    imgs = [[v['img'] for v in vs] for vs in views]
    slam = None
    if execution_mode == "vidslam":
        slam = dict(subsample=subsample, min_conf_keyframe=min_conf_keyframe, keyframe_overlap_thr=keyframe_overlap_thr,
                    overlap_percentile=overlap_percentile)
    with _amp(amp):
        x_out = _run(encoder, decoder, plans, imgs, device, act, max_bs, keyframe_interval, slam)
    _report(verbose, 'inference', time_start, device)
    copies = [_launch_scene_copies(xo, im) for xo, im in zip(x_out, imgs)]
    _sync_host_copies()
    return [_finish_scene(c, [torch.from_numpy(v['true_shape']) for v in vs], list(fl))
            for c, vs, fl in zip(copies, views, filelists)]


def _phase(name):
    """Phase boundary of _run ('encode', 'memory', 'postprocess', 'keyframes', 'compact', 'end'; the phases repeat every
    step): a no-op that tools/bench_reconstruct_videos.py replaces to record a CUDA event."""


def _run(encoder, decoder, plans, imgs, device, act, max_bs, keyframe_interval, slam):
    """The lockstep schedule on the device -> per scene the per-frame results of the last pass (device tensors)."""
    dev = torch.device(device)
    S = len(plans)
    _phase("encode")
    feats = _encode(encoder, plans, imgs, dev, max_bs)
    _phase("memory")
    arena = SessionArena(S, decoder.depth, 2 * decoder.embed_dim, decoder.memory_dtype(), dev)
    if slam is None:
        def is_keyframe(vid):
            return vid % keyframe_interval == 0
        arena.ensure(max(p.max_rows(is_keyframe) for p in plans))
    else:
        searchers = [get_searcher(SEARCHER) for _ in plans]
    results = [{} for _ in plans]
    pending = []                # per step of the last pass, the pointmaps still to postprocess (_postprocess's parts)
    passes = plans[0].passes
    for it in range(passes):
        last = it == passes - 1
        for k in range(max(len(p.steps) for p in plans)):
            calls = plan_step_calls(plans, k)
            _phase("memory")
            if slam is not None:
                need = max(arena.lengths[s] + sum(_tokens(hw) * n for hw, n in sig) for sig, run in calls for s in run)
                arena.ensure(need)
            staged, parts = [], []
            for sig, run in calls:
                xs, ps, ts = _call_inputs(feats, plans, run, lambda p: p.steps[k])
                if it == 0 and k == 0:
                    new, pms = decoder.update_tokens(xs, ps, ts, current_mem=None)
                else:
                    new, pms = decoder.update_tokens(xs, ps, ts, current_mem=arena.memory(run),
                                                     mem_lengths=[arena.lengths[s] for s in run])
                staged.append((run, new))
                for g, pm in enumerate(pms):
                    parts.append(((sig[g][0], g), pm.flatten(0, 1),
                                  [(s, q) for s in run for q in plans[s].steps[k][g][1]]))
            stepping = [s for _, run in calls for s in run]
            decided = {}
            if slam is not None and it == 0:
                _phase("postprocess")
                res = [{} for _ in plans]
                _postprocess(parts, act, res)
                if last:
                    for s in stepping:
                        results[s].update(res[s])
                _phase("keyframes")
                if k == 0:
                    adds = [(s, q) for s in stepping for q in plans[s].step_ids[0]]
                else:
                    members = [(s, plans[s].step_ids[k][0]) for s in sorted(stepping)]
                    flags = _slam_decisions(res, searchers, members, dev, **slam)
                    decided = {m: f for m, f in zip(members, flags)}
                    adds = [m for m, f in decided.items() if f]
                for s, q in adds:
                    slam_update_scene_state(slam["subsample"], slam["min_conf_keyframe"], res[s][q], searchers[s])
            elif last:
                pending.append(parts)
            if slam is None:
                edits = {s: plans[s].step(it, k, is_keyframe) for s in stepping}
            else:
                edits = {s: plans[s].step(it, k, lambda vid, s=s: decided[(s, vid)]) for s in stepping}
            apply_edits(arena, staged, edits, _phase)
    _phase("postprocess")
    for parts in pending:
        _postprocess(parts, act, results)
    _phase("end")
    return [[results[s][q] for q in range(len(p.order))] for s, p in enumerate(plans)]
