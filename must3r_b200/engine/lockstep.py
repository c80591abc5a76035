"""The memories of scenes batched through one decoder call (engine/scenes.py, videos.py, slam_sessions.py,
slam_cameras.py): one arena slot per scene (SessionArena: slot s of a [S, cap, width] buffer per level, base row s * cap),
the calls that scenes share (plan_batch, slot_runs, lockstep_calls), and the edits of their rows (StepEdit, apply_edits,
commit, commit_ordered, compact).  This module is the only Python caller of the m3r_mem_* entry points, and it splits
every edit at their launch limits.
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
from collections import Counter
from typing import Dict, List, NamedTuple, Optional, Sequence

import torch

from .. import _lib
from ..model import common as cm
from .inference import ENCODE_AHEAD_BATCH, stack_views

MAX_COMMIT = 64             # M3R_MAX_COMMIT: scenes (frames of m3r_mem_commit_ordered) per m3r_mem_* launch
MAX_COMPACT_RUNS = 128      # M3R_MAX_COMPACT_RUNS: runs per m3r_mem_compact_rows launch


class SessionArena:
    """Per level one [S, cap, width] buffer; slot s holds session s's memory rows [0, lengths[s]).  `ensure(rows)` grows
    every level geometrically (by `growth`, at least to `rows`) with one copy of the used rows for all sessions."""

    def __init__(self, S, depth, width, dtype, device, growth=1.5, min_cap=0):
        self.S, self.depth, self.width, self.dtype, self.device = S, depth, width, dtype, torch.device(device)
        self.growth, self.min_cap = growth, min_cap
        self.cap = 0
        self.bufs: List[torch.Tensor] = []
        self.lengths = [0] * S
        self.keep_all = torch.ones(1, dtype=torch.int32, device=self.device)    # commit's flag when every slot writes

    def ensure(self, rows):
        """Room for `rows` rows in every slot; True if the buffers were reallocated (views handed out before stay valid,
        on the old buffers)."""
        if rows <= self.cap:
            return False
        cap = max(rows, int(math.ceil(self.cap * self.growth)), self.min_cap)
        used = max(self.lengths)
        new = [torch.empty((self.S, cap, self.width), dtype=self.dtype, device=self.device) for _ in range(self.depth)]
        for n, o in zip(new, self.bufs):
            if used:
                n[:, :used].copy_(o[:, :used])
        self.bufs, self.cap = new, cap
        return True

    def views(self, s, rows=None):
        rows = self.lengths[s] if rows is None else rows
        return [b[s:s + 1, :rows] for b in self.bufs]

    def memory(self, run):
        """The decoder's memory argument for a call over the consecutive slots `run` (pass mem_lengths with it)."""
        return [b[run[0]:run[-1] + 1] for b in self.bufs], None, 0, 0, 0

    def holds(self, s, mem_vals):
        """True if mem_vals are already the views of slot s (nothing to copy)."""
        return (len(self.bufs) == len(mem_vals) and mem_vals[0].shape[1] == self.lengths[s]
                and all(m.data_ptr() == b[s].data_ptr() for m, b in zip(mem_vals, self.bufs)))

    def store(self, s, mem_vals):
        """Copy a [1, n, width] memory (list per level) into slot s."""
        n = mem_vals[0].shape[1]
        self.ensure(n)
        for b, m in zip(self.bufs, mem_vals):
            b[s, :n].copy_(m[0])
        self.lengths[s] = n


def plan_batch(cands: Dict[int, Optional[tuple]]):
    """The batching rule.  cands: session id -> its frame's preprocessed (H, W), or None when the frame must run alone
    (empty memory, an initialisation re-run, a memory_mode other than 'kv').  -> (batched ids, alone ids), both in the
    order given.  The batch takes the shape most frames share (the first such shape on a tie).  A batch of one frame
    still takes the batched path: its memory stays in its slot, where the single-session path would copy it there."""
    shapes = Counter(sh for sh in cands.values() if sh is not None)
    if not shapes:
        return [], list(cands)
    best = max(shapes.values())
    shape = next(sh for sh in cands.values() if sh is not None and shapes[sh] == best)
    batch = [sid for sid, sh in cands.items() if sh == shape]
    return batch, [sid for sid in cands if sid not in batch]


def slot_runs(slots: Sequence[int]):
    """Sorted slot indices -> runs of consecutive slots (one decoder call each: its scenes must be evenly strided)."""
    runs = []
    for s in slots:
        if runs and s == runs[-1][-1] + 1:
            runs[-1].append(s)
        else:
            runs.append([s])
    return runs


def _tokens(hw):
    return (hw[0] // 16) * (hw[1] // 16)


def _groups(shapes, positions, max_bs):
    """stack_views' grouping of the views at `positions` (by shape, lexicographic, cut at max_bs) -> [((H, W), [pos])]."""
    if not positions:
        return []
    ts = torch.tensor([shapes[p] for p in positions], dtype=torch.int32).view(-1, 2)
    _, idx_st = stack_views(ts, [], max_bs=max_bs)
    return [(shapes[positions[idx[0]]], [positions[i] for i in idx]) for idx in idx_st]


def signature(groups):
    """What scenes must share to run a step or render chunk in one call: the shape and view count of every group."""
    return tuple((hw, len(pos)) for hw, pos in groups)


def lockstep_calls(items):
    """items [(slot, signature)] in slot order -> [(signature, [slots])]: the scenes of the most common signature first
    (plan_batch; the first such signature on a tie), each cut into runs of consecutive slots; then the rest likewise."""
    cands = dict(items)
    calls = []
    while cands:
        batch, rest = plan_batch(cands)
        calls += [(cands[batch[0]], run) for run in slot_runs(batch)]
        cands = {s: cands[s] for s in rest}
    return calls


def _host_shape(hw, B, n):
    ts = torch.tensor(hw, dtype=torch.int32).view(1, 1, 2).expand(B, n, 2)
    ts._m3r_hw = tuple(hw)          # the decoder reads (H, W) from here: no device read
    return ts


def _encode(encoder, plans, imgs, device, max_bs):
    """Every view of every scene (plan.shapes, in plan.order), grouped by shape -> feats[s][position] = (x [N, D],
    pos [N, 2])."""
    S = len(plans)
    bs = ENCODE_AHEAD_BATCH if max_bs is None else min(ENCODE_AHEAD_BATCH, max_bs * S)
    by_shape = {}
    for s, p in enumerate(plans):
        for q, hw in enumerate(p.shapes):
            by_shape.setdefault(hw, []).append((s, q))
    feats = [[None] * len(p.order) for p in plans]
    for hw, members in by_shape.items():
        for lo in range(0, len(members), bs):
            chunk = members[lo:lo + bs]
            ts = torch.tensor([hw] * len(chunk), dtype=torch.int32)       # host: the encoder reads it there
            xs, ps = encoder(torch.stack([imgs[s][q] for s, q in chunk]).to(device), ts)
            for j, (s, q) in enumerate(chunk):
                feats[s][q] = (xs[j], ps[j])
    return feats


def _call_inputs(feats, plans, run, groups_of):
    """Stacked decoder inputs of one call: per group x [B, n, N, D], pos [B, n, N, 2], true_shape [B, n, 2]."""
    xs, ps, ts = [], [], []
    for g, (hw, _) in enumerate(groups_of(plans[run[0]])):
        members = [groups_of(plans[s])[g][1] for s in run]
        xs.append(torch.stack([torch.stack([feats[s][q][0] for q in pos]) for s, pos in zip(run, members)]))
        ps.append(torch.stack([torch.stack([feats[s][q][1] for q in pos]) for s, pos in zip(run, members)]))
        ts.append(_host_shape(hw, len(run), len(members[0])))
    return xs, ps, ts


class StepEdit(NamedTuple):
    """One scene's memory edit after one step, in rows of its slot.  runs: the compaction [(src_row, dst_row, rows)],
    applied first; write: (staged_row, dst_row, rows), the step's new rows that stay, or None; length: rows afterwards."""
    runs: list
    write: Optional[tuple]
    length: int


def _ptrs(tensors):
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def commit(arena, staged, slots, dst_rows, row0=0, rows=None, keep=None, keep_stride=0):
    """m3r_mem_commit_rows, MAX_COMMIT scenes per launch: staged rows [row0, row0 + rows) of scene b (staged: list[depth]
    of [B, Nt, width]; rows defaults to the rest) to rows dst_rows[b].. of slot slots[b].  keep: None (all write) or an
    int32 device tensor whose element b * keep_stride is scene b's flag (0: it writes nothing)."""
    Nt = staged[0].shape[1]
    rows = Nt - row0 if rows is None else rows
    if keep is None:
        keep, keep_stride = arena.keep_all, 0
    lib, bufs, stream = _lib.lib(), _ptrs(arena.bufs), cm.stream_ptr(arena.device)
    for lo in range(0, len(slots), MAX_COMMIT):
        hi = min(lo + MAX_COMMIT, len(slots))
        src = (C.c_void_p * arena.depth)(*[t.data_ptr() + lo * t.stride(0) * t.element_size() for t in staged])
        dst = (C.c_int64 * (hi - lo))(*[slots[b] * arena.cap + dst_rows[b] for b in range(lo, hi)])
        _lib.check(lib.m3r_mem_commit_rows(bufs, src, arena.depth, hi - lo, row0, rows, Nt, arena.width, dst,
                                           C.c_void_p(keep.data_ptr() + 4 * lo * keep_stride), keep_stride, stream),
                   "mem_commit_rows")


def commit_ordered(arena, staged, keep, keep_stride):
    """m3r_mem_commit_ordered into slot 0: the new rows of the frames whose flag (keep, as in commit) is set, behind its
    memory in frame order.  staged: list[depth] of [F, Nt, width], F <= MAX_COMMIT."""
    F, Nt = staged[0].shape[:2]
    _lib.check(_lib.lib().m3r_mem_commit_ordered(_ptrs(arena.bufs), _ptrs(staged), arena.depth, F, Nt, arena.width,
                                                 arena.lengths[0], C.c_void_p(keep.data_ptr()), keep_stride,
                                                 cm.stream_ptr(arena.device)), "mem_commit_ordered")


def compact(arena, runs_of):
    """m3r_mem_compact_rows of {slot: runs}, in launches of at most MAX_COMMIT scenes and MAX_COMPACT_RUNS runs (a scene
    whose runs do not fit goes on in the next launch: applied in order, runs compose)."""
    launches, cur, n = [], [], 0
    for slot in sorted(runs_of):
        runs = list(runs_of[slot])
        while runs:
            if n == MAX_COMPACT_RUNS or len(cur) == MAX_COMMIT:
                launches.append(cur)
                cur, n = [], 0
            take, runs = runs[:MAX_COMPACT_RUNS - n], runs[MAX_COMPACT_RUNS - n:]
            cur.append((slot, take))
            n += len(take)
    if cur:
        launches.append(cur)
    lib, bufs, stream = _lib.lib(), _ptrs(arena.bufs), cm.stream_ptr(arena.device)
    for members in launches:
        B = len(members)
        off, flat = [0], []
        for _, rs in members:
            flat += [v for r in rs for v in r]
            off.append(off[-1] + len(rs))
        _lib.check(lib.m3r_mem_compact_rows(bufs, arena.depth, B, arena.width, arena.cap,
                                            (C.c_int64 * B)(*[s * arena.cap for s, _ in members]),
                                            (C.c_int32 * (B + 1))(*off), (C.c_int32 * len(flat))(*flat), stream),
                   "mem_compact_rows")


def apply_edits(arena, staged_calls, edits, phase=lambda name: None):
    """The edits {slot: StepEdit} of one step whose calls staged_calls [(run, staged rows)] touched disjoint slots: the
    compaction of every scene, then the staged rows that stay, one commit per group of adjacent scenes of a call that
    write the same staged rows, then the lengths.  phase('compact') and phase('memory') mark the two device stretches."""
    runs_of = {s: e.runs for s, e in edits.items() if e.runs}
    if runs_of:
        phase("compact")
        compact(arena, runs_of)
    phase("memory")
    for run, new in staged_calls:
        writes = [edits[s].write for s in run]
        for part, group in itertools.groupby(range(len(run)), key=lambda i: writes[i] and (writes[i][0], writes[i][2])):
            g = list(group)
            if part:                    # (staged_row, rows) shared by adjacent scenes of the call
                commit(arena, [t[g[0]:g[-1] + 1] for t in new], [run[i] for i in g], [writes[i][1] for i in g], *part)
    for s, e in edits.items():
        arena.lengths[s] = e.length
