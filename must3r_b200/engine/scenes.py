"""Several offline reconstructions (must3r_inference's linseq schedule) stepped in lockstep on one model and one GPU.

`reconstruct_scenes(model, device, image_size, amp, filelists, ...)` returns, for every image list, the SceneState that
`must3r_inference(model, None, device, image_size, amp, filelist, min(num_mem_images, len(filelist)), max_bs, ...,
is_sequence=True)` returns for that list alone, but the scenes share their calls:

  * Each scene keeps its own schedule (ScenePlan): linspace keyframes, view order, file names, memory batches
    (demo._mem_batches) and views to render (demo._to_render), its steps' views grouped by shape and cut at `max_bs` as
    inference_multi_ar does (stack_views).
  * The views of all scenes are encoded up front, grouped by shape, up to ENCODE_AHEAD_BATCH views per call.
  * The memories live in one SessionArena (engine/lockstep.py), one slot per scene, sized once for the schedule.
  * Step k of every scene that has one runs in the same decoder calls: the scenes whose step views have the same shapes
    share a call (lockstep_calls).  A step is its MUSt3R.update_tokens calls (the first step's without a memory; every
    later one with the scenes' memory lengths, so each scene attends only to its own rows), then the commit of every
    scene's new rows into its slot (ScenePlan.step's edit, lockstep.apply_edits).
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

import datetime
import itertools
from typing import List, Sequence

import torch

from ..model import get_pointmaps_activation
from .demo import (SceneState, _amp, _finish_scene, _launch_scene_copies, _linspace_keyframes, _load, _mem_batches,
                   _report, _to_render)
from .inference import _sync_host_copies, postprocess
from .lockstep import (SessionArena, StepEdit, _call_inputs, _encode, _groups, _tokens, apply_edits, lockstep_calls,
                       signature)


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

    def step(self, it, k) -> StepEdit:
        """The memory edit after step k of pass `it`: pass 0 writes the step's rows behind the memory, a refinement pass
        overwrites them in place from refresh_row0(k) on."""
        rows = sum(_tokens(hw) * len(pos) for hw, pos in self.steps[k])
        row0 = self.refresh_row0(k) if it else 0
        length = self.mem_rows if it else self.step_start[k] + rows
        return StepEdit([], (row0, self.step_start[k] + row0, rows - row0), length)


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
    pending = []          # (H, W), raw pointmaps [rows, H, W, 7], [(slot, position)] per row, 0: memory step / 1: render

    for (it, step), calls in itertools.groupby(plan_memory_calls(plans, num_refinements_iterations), lambda c: c[:2]):
        staged = []       # the calls of a step touch disjoint slots: their rows are committed after the last one
        for _, _, sig, run in calls:
            xs, ps, ts = _call_inputs(feats, plans, run, lambda p: p.steps[step])
            if it == 0 and step == 0:
                new, pms = decoder.update_tokens(xs, ps, ts, current_mem=None)
            else:
                new, pms = decoder.update_tokens(xs, ps, ts, current_mem=arena.memory(run),
                                                 mem_lengths=[arena.lengths[s] for s in run])
            staged.append((run, new))
            if it == num_refinements_iterations and plans[run[0]].first_positions:   # render_once: returned as they are
                for g, pm in enumerate(pms):
                    members = [(s, q) for s in run for q in plans[s].steps[step][g][1]]
                    pending.append((sig[g][0], pm.flatten(0, 1), members, 0))
        apply_edits(arena, staged, {s: plans[s].step(it, step) for run, _ in staged for s in run})

    _phase("render")
    if any(p.render for p in plans):
        for c, sig, run in plan_render_calls(plans):
            (xs,), (ps,), (ts,) = _call_inputs(feats, plans, run, lambda p: [p.render[c]])
            pm = decoder.render_tokens(xs, ps, ts, arena.memory(run), [arena.lengths[s] for s in run])
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
