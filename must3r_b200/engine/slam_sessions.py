"""Several independent online SLAM sessions (SLAM_MUSt3R) served by one model on one GPU, their frames batched.

A session is one SLAM_MUSt3R: its own memory, keyframes, searcher, agents and trajectory, built with SLAM_MUSt3R's
constructor arguments except `chkpt` and `device`, which the sessions share.  `SLAMSessions.step({sid: (frame, frame_id,
cam_id)})` takes one frame for any subset of the sessions and returns, per session, what SLAM_MUSt3R.__call__ returns.

Batching rule: a frame joins the step's batch when its session's memory is non-empty, its session is past the
initialisation re-runs (`num_init_frames`, after a fresh start or a loaded memory), the decoder keeps its memory as K|V
rows (memory_mode 'kv'), and its preprocessed shape is the batch's shape (the shape most frames of the step share).  The
batch then costs one encoder call over its frames, one decoder call in which each frame attends only to its own
session's memory (MUSt3R.update_tokens with mem_lengths, csrc/model.cu m3r_decoder_forward_ragged), the per-session
pose, searcher query and keyframe kernels (MUSt3R_Agent.launch_tail, each into its row of one batch of records), one
commit (lockstep.commit) that appends the new rows of the sessions whose frame is a keyframe, and one wait for all
records and returned arrays (engine/slam.py's _wait_host_copies); then each frame finishes as in SLAM_MUSt3R.__call__
(MUSt3R_Agent.finish_tail, SLAM_MUSt3R._record_frame).  Every other frame runs alone through SLAM_MUSt3R.__call__ and its
resulting memory is copied into its session's slot.

Memory: per decoder level one arena [S, cap, 2D] (SessionArena of engine/lockstep.py); session s's memory is rows
[0, n_s) of slot s.  The arena grows geometrically, for all sessions with one copy per level, when a session would
overflow.  Each session's `memory` is the reference's 5-tuple whose tensors are views of its slot, so save_memory,
pickling and load_memory work unchanged.
"""
from __future__ import annotations

from collections import Counter
from typing import Dict

import numpy as np
import torch

from .. import ops
from ..model import get_pointmaps_activation, load_model
from . import slam
from .images import preproc_frame
from .inference import _reserve, _to_out, postprocess
from .lockstep import SessionArena, commit, plan_batch, slot_runs
from .slam import SLAM_MUSt3R

KEYFRAME_FIELD = ops.SLAM_RECORD.fields["keyframe"][1] // 4     # int32 index of the keyframe flag in a record


class _Session(SLAM_MUSt3R):
    """One session: SLAM_MUSt3R on a shared model, its memory kept in slot `slot` of the sessions' arena."""

    def __init__(self, model, slot, **kwargs):
        self.slot = slot
        self._shared_model = model
        super().__init__(None, **kwargs)

    def _load_model(self, chkpt, device):
        return self._shared_model

    def runs_alone(self):
        """The frames SLAM_MUSt3R.__call__ handles specially: the first one (no memory) and the initialisation re-runs."""
        return self.memory is None or len(self.all_images) < self.num_init_frames


class SLAMSessions:
    """S SLAM sessions on one model.  `session_args` (optional, one dict per session) overrides `kwargs`, SLAM_MUSt3R's
    constructor arguments without chkpt and device, for that session."""

    def __init__(self, chkpt, num_sessions=1, device='cuda:0', session_args=None, **kwargs):
        if session_args is not None and len(session_args) != num_sessions:
            raise ValueError("session_args needs one dict per session")
        self.device = device
        self.model = load_model(chkpt, device=device)
        _reserve(self.model[1], 0, 1.5)
        dec = self.model[1]
        self.kv = dec.memory_mode == 'kv'
        self.arena = SessionArena(num_sessions, dec.depth, 2 * dec.embed_dim if self.kv else dec.embed_dim,
                                  dec.memory_dtype(), device)
        self.sessions = [_Session(self.model, i, device=device, **{**kwargs, **((session_args or [{}] * num_sessions)[i])})
                         for i in range(num_sessions)]
        self.stats = Counter()

    def __len__(self):
        return len(self.sessions)

    def __getitem__(self, i):
        return self.sessions[i]

    # ---- memory slots ----------------------------------------------------------------------------------------------
    def _repoint(self):
        """After the arena grew: every session's memory tuple onto the new buffers."""
        for s in self.sessions:
            if s.memory is not None and self.arena.lengths[s.slot] > 0 and s.memory[0][0].shape[1] == self.arena.lengths[s.slot]:
                s.memory = (self.arena.views(s.slot),) + tuple(s.memory[1:])

    def _to_slot(self, s):
        """Move session s's memory (as SLAM_MUSt3R left it) into its slot."""
        if s.memory is None or not self.kv:
            return
        vals = s.memory[0]
        if self.arena.holds(s.slot, vals):
            return
        grew = self.arena.ensure(vals[0].shape[1])
        self.arena.store(s.slot, vals)
        s.memory = (self.arena.views(s.slot),) + tuple(s.memory[1:])
        if grew:
            self._repoint()

    # ---- one step ----------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, frames: Dict[int, tuple]):
        """frames: {session id: (frame, frame_id, cam_id)} -> {session id: SLAM_MUSt3R.__call__'s result}."""
        cands, prepped = {}, {}
        for sid, (img, fid, cam) in frames.items():
            s = self.sessions[sid]
            if not self.kv or s.runs_alone() or self.arena.lengths[s.slot] == 0 or not self.arena.holds(s.slot, s.memory[0]):
                cands[sid] = None
                continue
            view, to_orig = preproc_frame(img, fid, res=s.res, device=s.device)
            prepped[sid] = (view, to_orig)
            cands[sid] = tuple(int(v) for v in np.asarray(view['true_shape']).reshape(-1)[:2])
        batch, alone = plan_batch(cands)
        out = {}
        if batch:
            out.update(self._step_batch(batch, frames, prepped))
        for sid in alone:
            s = self.sessions[sid]
            out[sid] = SLAM_MUSt3R.__call__(s, *frames[sid])
            self._to_slot(s)
        self.stats['batched'] += len(batch)
        self.stats['alone'] += len(alone)
        return {sid: out[sid] for sid in frames}

    def _decode(self, batch, prepped):
        """One encoder call over the batch's frames, then one ragged decoder call per run of consecutive slots.
        -> (res {pts3d, pts3d_local, conf} [B,1,H,W,..] in batch order, [(run members, staged rows)])."""
        encoder, decoder = self.model
        views = [prepped[sid][0] for sid in batch]
        imgs = torch.cat([v['img'] for v in views]).to(self.device)
        ts = torch.as_tensor(np.concatenate([np.asarray(v['true_shape']).reshape(-1, 2) for v in views]))
        x, pos = encoder(imgs, ts)
        N = x.shape[1]
        need = max(self.arena.lengths[self.sessions[sid].slot] for sid in batch) + N
        if self.arena.ensure(need):
            self._repoint()
        hw = tuple(int(v) for v in ts[0].tolist())
        act = get_pointmaps_activation(decoder, verbose=False)
        pms, staged, i0 = [], [], 0
        for run in slot_runs([self.sessions[sid].slot for sid in batch]):      # batch is in slot order
            i1 = i0 + len(run)
            shape = ts[i0:i1].view(i1 - i0, 1, 2)
            shape._m3r_hw = hw
            lengths = [self.arena.lengths[sl] for sl in run]
            new_tokens, pm = decoder.update_tokens(x[i0:i1, None], pos[i0:i1, None], shape,
                                                   current_mem=self.arena.memory(run), mem_lengths=lengths)
            staged.append((batch[i0:i1], new_tokens))
            pms.append(pm)
            i0 = i1
        pm = torch.cat(pms) if len(pms) > 1 else pms[0]
        return postprocess(pm, pointmaps_activation=act), staged

    def _commit(self, staged, recs, index):
        """Each run's new rows of the sessions whose record says keyframe, behind their memory."""
        flags = recs.view(torch.int32)[:, KEYFRAME_FIELD]
        for members, new_tokens in staged:
            i0 = index[members[0]]
            assert [index[m] for m in members] == list(range(i0, i0 + len(members)))
            slots = [self.sessions[m].slot for m in members]
            commit(self.arena, new_tokens, slots, [self.arena.lengths[s] for s in slots], keep=flags[i0:],
                   keep_stride=flags.stride(0))

    def _step_batch(self, batch, frames, prepped):
        dev = torch.device(self.device)
        # commit and records want the batch in slot order (each decoder run is a contiguous range of it)
        batch = sorted(batch, key=lambda sid: self.sessions[sid].slot)
        res, staged = self._decode(batch, prepped)
        index = {sid: i for i, sid in enumerate(batch)}
        recs = torch.empty((len(batch), ops.SLAM_RECORD.itemsize), dtype=torch.uint8, device=dev)
        preds, tails = [], []
        for i, sid in enumerate(batch):
            s = self.sessions[sid]
            pred = {k: res[k][i:i + 1] for k in ('pts3d', 'pts3d_local', 'conf')}
            tails.append(s.agents[frames[sid][2]].launch_tail(
                prepped[sid][0], pred, False, overlap_mode=s.overlap_mode, overlap_tree=s.overlap_tree,
                kf_x_subsamp=s.kf_x_subsamp, keyframe_overlap_thr=s.keyframe_overlap_thr,
                min_conf_keyframe=s.min_conf_keyframe, overlap_percentile=s.overlap_percentile, rec=recs[i:i + 1]))
            preds.append(pred)
        self._commit(staged, recs, index)
        host_recs = _to_out(recs, 'cpu')
        slam._wait_host_copies()
        records = host_recs.numpy().view(ops.SLAM_RECORD)[:, 0]
        new_rows = {sid: t for members, tok in staged for sid, t in zip(members, [tok] * len(members))}
        out = {}
        for i, sid in enumerate(batch):
            s = self.sessions[sid]
            _, fid, cam = frames[sid]
            view, to_orig = prepped[sid]
            frame_out = s.agents[cam].finish_tail(preds[i], tails[i], records[i], to_orig)
            if s.rerender:
                s.all_images.append(view)
            if frame_out[-1]:
                self._append(s, new_rows[sid][0].shape[1])
            out[sid] = s._record_frame(view, preds[i], fid, frame_out)
        return out

    def _append(self, s, n_new):
        """Host bookkeeping of a committed keyframe: n_new rows behind session s's memory, labelled as its next image."""
        vals, labels, nimgs, _, _ = s.memory
        n = self.arena.lengths[s.slot] + n_new
        self.arena.lengths[s.slot] = n
        labels = torch.cat([labels, torch.full((1, n_new), nimgs, dtype=labels.dtype, device=labels.device)], 1)
        s.memory = (self.arena.views(s.slot), labels, nimgs + 1, nimgs + 1, n)
