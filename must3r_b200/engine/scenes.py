"""Several offline reconstructions (must3r_inference's linseq schedule) stepped in lockstep on one model and one GPU.

`reconstruct_scenes(model, device, image_size, amp, filelists, ...)` returns, for every image list, the SceneState that
`must3r_inference(model, None, device, image_size, amp, filelist, min(num_mem_images, len(filelist)), max_bs, ...,
is_sequence=True)` returns for that list alone, but the scenes share their calls:

  * Each scene keeps its own schedule (ScenePlan): linspace keyframes, view order, file names, memory batches
    (demo._mem_batches) and views to render (demo._to_render), its steps' views grouped by shape and cut at `max_bs` as
    inference_multi_ar does (stack_views).
  * The views of all scenes are encoded up front, grouped by shape, up to ENCODE_AHEAD_BATCH views per call.
  * The memories live in one SessionArena (engine/slam_sessions.py), one slot per scene, sized once for the schedule.
  * Step k of every scene that has one runs in the same decoder calls: the scenes whose step views have the same shapes
    share a call (plan_batch's rule, then one call per run of consecutive slots, slot_runs).  A step is one
    MUSt3R.update_tokens call (the first one without a memory; every later one with the scenes' memory lengths, so each
    scene attends only to its own rows) followed by one m3r_mem_commit_rows that writes the new rows into the slots.
  * A refinement pass re-runs every step against the full memories and overwrites each step's rows in place, except those
    of the reference view (label 0: the first view of the first step), as inference_multi_ar's refresh branch does.
  * The render pass runs in chunks of up to `max_bs` views per scene (MUSt3R.render_tokens, m3r_decoder_render_ragged);
    chunk c of the scenes with the same view count and shape shares a call.
  * postprocess(compute_cam=True) runs once per image shape over every pointmap of that shape; then every scene's results
    are copied to the host in one batch of asynchronous copies followed by one wait.

`max_bs` keeps its per-scene meaning (views of one scene per call), so a decoder call over S scenes holds up to
S * max_bs views, and an encoder call up to min(ENCODE_AHEAD_BATCH, S * max_bs).

Differences from must3r_inference: only memory_mode 'kv' is supported, there is no retrieval, and a scene with fewer
images than init_num_images builds its memory from the images it has (must3r_inference refuses it: the reference's
memory-batch loop never ends).
"""
from __future__ import annotations

import ctypes as C
import datetime
from typing import List, Sequence

import torch

from .. import _lib
from ..model import get_pointmaps_activation
from ..model import common as cm
from .demo import (SceneState, _amp, _finish_scene, _launch_scene_copies, _linspace_keyframes, _load, _mem_batches,
                   _report, _to_render)
from .inference import ENCODE_AHEAD_BATCH, _sync_host_copies, postprocess, stack_views
from .slam_sessions import SessionArena, plan_batch, slot_runs

MAX_COMMIT = 64         # M3R_MAX_COMMIT: scenes per m3r_mem_commit_rows launch


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


class ScenePlan:
    """One scene's schedule, in must3r_inference's terms.  Positions index the scene's views in `order` (keyframes first).
    steps[k]: the groups [((H, W), [positions])] of memory step k; step_start[k]: the memory row where step k's rows begin;
    render: the render chunks [((H, W), [positions])]; x_out holds the memory-step results of first_positions (with
    render_once) followed by the render results of render_positions."""

    def __init__(self, filelist: Sequence[str], shapes, num_mem_images, init_num_images=2, batch_num_views=1,
                 render_once=False, max_bs=None):
        nimgs = len(filelist)
        if nimgs == 0:
            raise ValueError("a scene needs at least one image")
        nmi = min(num_mem_images, nimgs)
        init = min(init_num_images, nimgs)
        self.keyframes = _linspace_keyframes(nimgs, nmi)
        self.order = self.keyframes + sorted(set(range(nimgs)).difference(self.keyframes))
        self.filenames = [filelist[i] for i in self.order]
        self.shapes = [tuple(int(v) for v in shapes[i]) for i in self.order]
        self.mem_batches = _mem_batches(nimgs, init, batch_num_views, max(nmi, init), nmi)
        self.to_render = _to_render(render_once, nmi, nimgs)
        self.steps, self.step_start, lo = [], [], 0
        rows = 0
        for n in self.mem_batches:
            groups = _groups(self.shapes, list(range(lo, lo + n)), max_bs)
            self.steps.append(groups)
            self.step_start.append(rows)
            rows += sum(_tokens(hw) * len(pos) for hw, pos in groups)
            lo += n
        self.mem_rows = rows
        self.first_positions = list(range(lo)) if self.to_render is not None else []
        self.render_positions = list(range(nimgs)) if self.to_render is None else list(self.to_render)
        self.render = _groups(self.shapes, self.render_positions, max_bs)

    def refresh_row0(self, step):
        """First staged row a refinement re-run of `step` writes back: the reference view's rows (label 0, the first view
        of step 0's first group) are never overwritten."""
        return _tokens(self.steps[0][0][0]) if step == 0 else 0


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


def plan_memory_calls(plans: List[ScenePlan], num_refinements_iterations=0):
    """The lockstep memory schedule -> [(pass, step, signature, [slots])], in execution order."""
    out = []
    for it in range(num_refinements_iterations + 1):
        for step in range(max(len(p.steps) for p in plans)):
            items = [(s, signature(p.steps[step])) for s, p in enumerate(plans) if step < len(p.steps)]
            out += [(it, step, sig, run) for sig, run in lockstep_calls(items)]
    return out


def plan_render_calls(plans: List[ScenePlan]):
    """The lockstep render schedule -> [(chunk, signature, [slots])], in execution order."""
    out = []
    for c in range(max(len(p.render) for p in plans)):
        items = [(s, signature([p.render[c]])) for s, p in enumerate(plans) if c < len(p.render)]
        out += [(c, sig, run) for sig, run in lockstep_calls(items)]
    return out


def arena_rows(plans: List[ScenePlan]):
    """Rows per slot of the scenes' arena: the largest memory of the schedule (refinement passes stage their rows apart)."""
    return max(p.mem_rows for p in plans)


def _host_shape(hw, B, n):
    ts = torch.tensor(hw, dtype=torch.int32).view(1, 1, 2).expand(B, n, 2)
    ts._m3r_hw = tuple(hw)          # the decoder reads (H, W) from here: no device read
    return ts


def _commit_rows(arena, staged, slots, row0, rows, dst_rows, keep, stream):
    """m3r_mem_commit_rows of staged rows [row0, row0 + rows) of each scene to its slot at dst_rows[b]."""
    lib = _lib.lib()
    depth = arena.depth
    bufs = (C.c_void_p * depth)(*[b.data_ptr() for b in arena.bufs])
    Nt = staged[0].shape[1]
    for lo in range(0, len(slots), MAX_COMMIT):
        hi = min(lo + MAX_COMMIT, len(slots))
        src = (C.c_void_p * depth)(*[t[lo].data_ptr() for t in staged])
        dst = (C.c_int64 * (hi - lo))(*[slots[b] * arena.cap + dst_rows[b] for b in range(lo, hi)])
        _lib.check(lib.m3r_mem_commit_rows(bufs, src, depth, hi - lo, row0, rows, Nt, arena.width, dst,
                                           C.c_void_p(keep.data_ptr()), 0, stream), "mem_commit_rows")


def _encode(encoder, plans, imgs, device, max_bs):
    """Every view of every scene, grouped by shape -> feats[s][position] = (x [N, D], pos [N, 2])."""
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


@torch.no_grad()
def reconstruct_scenes(model, device, image_size, amp, filelists, num_mem_images, max_bs, init_num_images=2,
                       batch_num_views=1, render_once=False, num_refinements_iterations=0, verbose=True) -> List[SceneState]:
    """S independent reconstructions in lockstep (module docstring) -> one SceneState per image list."""
    encoder, decoder = model
    if getattr(decoder, "memory_mode", None) != "kv":
        raise NotImplementedError(f"reconstruct_scenes batches memories of memory_mode 'kv' only (the decoder's is "
                                  f"{getattr(decoder, 'memory_mode', None)!r}); run must3r_inference per scene")
    if not filelists:
        return []
    max_bs = None if max_bs == 0 else max_bs
    act = get_pointmaps_activation(decoder, verbose=verbose)
    if verbose:
        print(f'loading images of {len(filelists)} scenes')
    time_start = datetime.datetime.now()
    views = [_load(fl, image_size, encoder, verbose, device) for fl in filelists]
    plans = [ScenePlan(fl, [v['true_shape'] for v in vs], num_mem_images, init_num_images, batch_num_views, render_once,
                       max_bs) for fl, vs in zip(filelists, views)]
    if verbose:
        print(f'loaded in {datetime.datetime.now() - time_start}')
        print('running inference')
    time_start = datetime.datetime.now()
    imgs = [[vs[i]['img'] for i in p.order] for p, vs in zip(plans, views)]
    with _amp(amp):
        x_out = _run(encoder, decoder, plans, imgs, device, act, max_bs, num_refinements_iterations)
    _report(verbose, 'inference', time_start, device)
    copies = [_launch_scene_copies(xo, im) for xo, im in zip(x_out, imgs)]
    _sync_host_copies()
    return [_finish_scene(c, [torch.from_numpy(vs[i]['true_shape']) for i in p.order], p.filenames)
            for c, p, vs in zip(copies, plans, views)]


def _phase(name):
    """Phase boundary of _run ('encode', 'memory', 'render', 'postprocess', 'end'): a no-op that
    tools/bench_reconstruct_scenes.py replaces to record a CUDA event."""


def _run(encoder, decoder, plans, imgs, device, act, max_bs, num_refinements_iterations):
    """The lockstep schedule on the device -> per scene the x_out list of must3r_inference (device tensors)."""
    dev = torch.device(device)
    S = len(plans)
    _phase("encode")
    feats = _encode(encoder, plans, imgs, dev, max_bs)
    _phase("memory")
    arena = SessionArena(S, decoder.depth, 2 * decoder.embed_dim, decoder.memory_dtype(), dev)
    arena.ensure(arena_rows(plans))
    keep = torch.ones(1, dtype=torch.int32, device=dev)
    stream = cm.stream_ptr(dev)
    pending = []          # (H, W), raw pointmaps [rows, H, W, 7], [(slot, position)] per row, 0: memory step / 1: render

    for it, step, sig, run in plan_memory_calls(plans, num_refinements_iterations):
        xs, ps, ts = _call_inputs(feats, plans, run, lambda p: p.steps[step])
        if it == 0 and step == 0:
            new, pms = decoder.update_tokens(xs, ps, ts, current_mem=None)
        else:
            mem = ([b[run[0]:run[-1] + 1] for b in arena.bufs], None, 0, 0, 0)
            new, pms = decoder.update_tokens(xs, ps, ts, current_mem=mem, mem_lengths=[arena.lengths[s] for s in run])
        Nt = new[0].shape[1]
        row0 = 0 if it == 0 else plans[run[0]].refresh_row0(step)
        _commit_rows(arena, new, run, row0, Nt - row0, [plans[s].step_start[step] + row0 for s in run], keep, stream)
        if it == 0:
            for s in run:
                assert arena.lengths[s] == plans[s].step_start[step]
                arena.lengths[s] += Nt
        if it == num_refinements_iterations and plans[run[0]].first_positions:       # render_once: returned as they are
            for g, pm in enumerate(pms):
                members = [(s, q) for s in run for q in plans[s].steps[step][g][1]]
                pending.append((sig[g][0], pm.flatten(0, 1), members, 0))

    _phase("render")
    if any(p.render for p in plans):
        for c, sig, run in plan_render_calls(plans):
            (xs,), (ps,), (ts,) = _call_inputs(feats, plans, run, lambda p: [p.render[c]])
            mem = ([b[run[0]:run[-1] + 1] for b in arena.bufs], None, 0, 0, 0)
            pm = decoder.render_tokens(xs, ps, ts, mem, [arena.lengths[s] for s in run])
            pending.append((sig[0][0], pm.flatten(0, 1), [(s, q) for s in run for q in plans[s].render[c][1]], 1))

    _phase("postprocess")
    results = [({}, {}) for _ in plans]     # per scene: memory-step results, render results, by position
    by_shape = {}
    for hw, pm, members, kind in pending:
        by_shape.setdefault(hw, []).append((pm, members, kind))
    for parts in by_shape.values():
        pm = torch.cat([p for p, _, _ in parts]) if len(parts) > 1 else parts[0][0]
        res = postprocess(pm, pointmaps_activation=act, compute_cam=True)
        k = 0
        for _, members, kind in parts:
            for s, q in members:
                results[s][kind][q] = {key: v[k] for key, v in res.items()}
                k += 1
    _phase("end")
    return [[results[s][0][q] for q in p.first_positions] + [results[s][1][q] for q in p.render_positions]
            for s, p in enumerate(plans)]
