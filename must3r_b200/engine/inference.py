"""Engine API of the reference (must3r/engine/inference.py) re-stated for must3r_b200.

Same entry points, argument meaning and observable results: ``postprocess``, ``stack_views``,
``encoder_multi_ar``, ``inference_multi_ar_batch``, ``inference_multi_ar``, ``inference_video_multi_ar``,
``inference_encoder``, ``inference``, ``get_Nmem``, ``unstack_pointmaps``, ``concat_preds``.  The functions
are model-agnostic (they only call ``encoder(imgs, true_shape)`` / ``decoder(x, pos, true_shape, mem,
render=...)``), so the CPU test-suite drives them with the oracle model and the GPU suite with the CUDA
model.  ``compute_cam=True`` (Weiszfeld focal + weighted Procrustes, SURVEY.md §8f rank 3) is outside the hot path and
runs as a few torch ops (``engine/camera.py``).
"""
from __future__ import annotations

import itertools
import math
from collections import deque
from contextlib import nullcontext

import numpy as np
import torch

from ..model.common import ActivationType
from .camera import camera_from_pointmaps


# --------------------------------------------------------------------------------------------- host copies
_PENDING_HOST_COPIES = []       # read-back streams with device->host copies not yet waited for
_D2H_STREAMS = {}               # device index -> side stream used only for result read-back


def _d2h_stream(device):
    st = _D2H_STREAMS.get(device.index)
    if st is None:
        st = _D2H_STREAMS[device.index] = torch.cuda.Stream(device=device)
    return st


def _to_out(v, outdevice):
    """`.to(outdevice)` of the reference (engine/inference.py:196), except that device->host results go through pinned
    staging buffers and an asynchronous copy on a dedicated read-back stream, so the D2H traffic overlaps the next
    decoder steps instead of stalling the launch thread or the compute stream.  `_sync_host_copies()` is called before
    results are handed to any callback or returned."""
    if v.is_cuda and str(outdevice) == "cpu":
        dst = torch.empty(v.shape, dtype=v.dtype, pin_memory=True)
        cur = torch.cuda.current_stream(v.device)
        st = _d2h_stream(v.device)
        st.wait_stream(cur)
        with torch.cuda.stream(st):
            dst.copy_(v, non_blocking=True)
        v.record_stream(st)
        _PENDING_HOST_COPIES.append(st)
        return dst
    return v.to(outdevice)


def _with_host_shape(true_shape_group, device):
    """true_shape [n,2] of one aspect-ratio group -> [1,n,2] for the decoder.  The decoder only ever reads true_shape on
    the host (must3r/model/blocks/head.py:31-32), so a host tensor (the usual case: it comes from the image loader) is
    passed through as is - moving it to the GPU, as the reference engine does, costs a blocking pageable H2D copy per
    decoder call - and its (H, W) is attached as `_m3r_hw` so the CUDA decoder does no device->host read either."""
    if true_shape_group.is_cuda:
        return true_shape_group.unsqueeze(0).to(device)
    out = true_shape_group.unsqueeze(0)
    rows = true_shape_group.reshape(-1, 2)
    assert bool((rows == rows[:1]).all()), 'true_shape must be all identical'
    try:
        out._m3r_hw = tuple(int(v) for v in rows[0].tolist())
    except Exception:  # noqa: BLE001  (tensor subclasses that refuse attributes)
        pass
    return out


def _sync_host_copies():
    if _PENDING_HOST_COPIES:
        for st in set(_PENDING_HOST_COPIES):
            st.synchronize()
        _PENDING_HOST_COPIES.clear()


# --------------------------------------------------------------------------------------------- postprocess
def _act(xyz, activation):
    if isinstance(activation, str):
        activation = ActivationType(activation)
    if getattr(activation, "value", activation) == "norm_exp":
        d = xyz.norm(dim=-1, keepdim=True)
        return xyz / d.clip(min=1e-8) * torch.expm1(d)          # must3r/tools/geometry.py:14-18
    if getattr(activation, "value", activation) == "linear":
        return xyz
    raise ValueError(f"Unknown activation: {activation}")


def postprocess(pointmaps, pointmaps_activation=ActivationType.NORM_EXP, compute_cam=False):
    """engine/inference.py:16-48.  7-channel CUDA pointmaps with the NORM_EXP activation take the fused
    kernel (m3r_postprocess); everything else is evaluated with torch in fp32, like the reference."""
    pm = pointmaps.float()
    act_name = getattr(pointmaps_activation, "value", pointmaps_activation)
    if pm.is_cuda and pm.shape[-1] == 7 and act_name == "norm_exp":
        from .. import ops
        pts, loc, conf = ops.postprocess_raw(pm)
        out = {"pts3d": pts, "pts3d_local": loc, "conf": conf}
        return camera_from_pointmaps(out) if compute_cam else out
    out = {"pts3d": _act(pm[..., :3], pointmaps_activation)}
    ch = pm.shape[-1]
    if ch >= 6:
        out["pts3d_local"] = _act(pm[..., 3:6], pointmaps_activation)
    if ch in (4, 7):
        out["conf"] = 1.0 + pm[..., -1].exp()
    if compute_cam:
        if "pts3d_local" not in out or "conf" not in out:
            raise KeyError("compute_cam needs pts3d_local and conf (7-channel pointmaps, engine/inference.py:29-41)")
        camera_from_pointmaps(out)
    return out


# --------------------------------------------------------------------------------------------- view grouping
def _chunks(seq, size):
    return [seq[i:i + size] for i in range(0, len(seq), size)]


def _split_entries(entries, max_bs):
    out = []
    for e in entries:
        out.extend(_chunks(e, max_bs) if isinstance(e, list) else list(torch.split(e, max_bs)))
    return out


def stack_views(true_shape, values, max_bs=None):
    """Group views by identical true_shape (engine/inference.py:65-136).

    Returns ``(true_shape_stacks, index_stacks, *value_stacks)``: groups follow the lexicographic order of the
    unique shapes (torch.unique), views keep their order inside a group; inside a group, views for which any
    value is None (features to be recomputed) are moved to an extra group appended at the end; groups are then
    cut in chunks of ``max_bs``; a group holding None values collapses to a single None."""
    uniq, inverse = torch.unique(true_shape, dim=0, return_inverse=True)
    n_groups = uniq.shape[0]
    members = [[i for i in range(true_shape.shape[0]) if int(inverse[i]) == g] for g in range(n_groups)]
    # peel off the views with missing values
    extra = []
    for g in range(n_groups):
        missing = [any(v[i] is None for v in values) for i in members[g]]
        if any(missing) and not all(missing):
            extra.append([i for i, m in zip(members[g], missing) if m])
            members[g] = [i for i, m in zip(members[g], missing) if not m]
    members += extra

    shape_stacks = [torch.stack([true_shape[i] for i in grp], dim=0) for grp in members]
    index_stacks = [list(grp) for grp in members]
    value_stacks = []
    for v in values:
        per_group = []
        for grp in members:
            items = [v[i] for i in grp]
            per_group.append(items if any(it is None for it in items) else torch.stack(items, dim=0))
        value_stacks.append(per_group)

    if max_bs is not None:
        shape_stacks = _split_entries(shape_stacks, max_bs)
        index_stacks = [c for grp in index_stacks for c in _chunks(grp, max_bs)]
        value_stacks = [_split_entries(vs, max_bs) for vs in value_stacks]
    value_stacks = [[None if isinstance(e, list) and any(it is None for it in e) else e for e in vs]
                    for vs in value_stacks]
    return (shape_stacks, index_stacks, *value_stacks)


def get_Nmem(mem):
    """engine/inference.py:530-535"""
    return 0 if mem is None else mem[1].shape[1]


def unstack_pointmaps(index_stacks_i, pointmaps_0_i):
    """Scatter per-group dicts of stacked tensors back to per-view dicts (engine/inference.py:538-552)."""
    n = max(max(idx) for idx in index_stacks_i) + 1
    out = [None] * n
    for stack, idx in zip(pointmaps_0_i, index_stacks_i):
        for j, view in enumerate(idx):
            out[view] = {k: v[j] for k, v in stack.items()}
    return out


# --------------------------------------------------------------------------------------------- encoder / decoder steps
@torch.no_grad()
def encoder_multi_ar(encoder, imgs, true_shape, verbose=False, max_bs=None, device=None, preserve_gpu_mem=False):
    """Encode a list of views of mixed aspect ratios (engine/inference.py:139-165) -> per-view (x, pos) lists."""
    n = true_shape.shape[0]
    device = device or true_shape.device
    outdevice = "cpu" if preserve_gpu_mem else device
    shape_stacks, index_stacks, img_stacks = stack_views(true_shape, [imgs], max_bs=max_bs)
    x, pos = [None] * n, [None] * n
    for im, ts, idx in zip(img_stacks, shape_stacks, index_stacks):
        xs, ps = encoder(im.to(device), ts.to(device))
        for j, view in enumerate(idx):
            x[view] = _to_out(xs[j], outdevice)
            pos[view] = _to_out(ps[j], outdevice)
    _sync_host_copies()
    return x, pos


@torch.no_grad()
def inference_multi_ar_batch(encoder, decoder, imgs, true_shape, mem=None, verbose=False,
                             encoder_precomputed_features=None, preserve_gpu_mem=False,
                             post_process_function=lambda x: {'pts3d': x}, device=None, render=False,
                             viser_server=None):
    """One decoder call over already-stacked aspect-ratio groups (engine/inference.py:168-202).  With preserve_gpu_mem
    the results are host tensors and, like the reference's `.to('cpu')`, complete when the call returns."""
    out = _multi_ar_batch(encoder, decoder, imgs, true_shape, mem, verbose, encoder_precomputed_features, preserve_gpu_mem,
                          post_process_function, device, render, viser_server)
    _sync_host_copies()
    return out


def _multi_ar_batch(encoder, decoder, imgs, true_shape, mem=None, verbose=False,
                    encoder_precomputed_features=None, preserve_gpu_mem=False,
                    post_process_function=lambda x: {'pts3d': x}, device=None, render=False,
                    viser_server=None):
    """inference_multi_ar_batch without the final wait for the asynchronous device->host copies: the schedulers below keep
    enqueueing decoder steps while results stream back and call _sync_host_copies() before handing anything out."""
    device = device or true_shape.device
    outdevice = "cpu" if preserve_gpu_mem else device
    if encoder_precomputed_features is None:
        feats = [encoder(im.to(device), ts.to(device)) for im, ts in zip(imgs, true_shape)]
        x, pos = [f[0] for f in feats], [f[1] for f in feats]
    else:
        x, pos = encoder_precomputed_features
    x = [v.unsqueeze(0).to(device) for v in x]           # B = 1 scene
    pos = [v.unsqueeze(0).to(device) for v in pos]
    ts = [_with_host_shape(v, device) for v in true_shape]
    mem, pms = decoder(x, pos, ts, mem, render=render)
    results = []
    for pm in pms:
        pm = pm.squeeze(0)
        if post_process_function is not None:
            pm = {k: _to_out(v, outdevice) for k, v in post_process_function(pm).items()}
        else:
            pm = _to_out(pm, outdevice)
        results.append(pm)
    return mem, results


# --------------------------------------------------------------------------------------------- memory edits by label
# The engine edits the memory between decoder calls (eviction of frames that left the window, refresh of keyframes).
# The reference does it with boolean masks computed on the device (engine/inference.py:205-228): every mask indexing is a
# host sync plus a copy of the whole memory, per level.  The label of every token is known on the host (the decoder
# hands them out deterministically, decoder.py:242-247), so a host-side copy of the label row ("shadow") rides along on
# the label tensor; with it the edits become slice operations: no sync, and dropping the most recent frame - what a
# non-keyframe step of the streaming schedule does - is a zero-copy prefix view.  Without a shadow (a memory of unknown
# provenance, or scenes with different label rows) the reference's device path runs.
def _host_labels(mem_labels):
    """-> numpy int64 row of the labels, or None.  (Kept on the tensor as a CPU torch tensor: that survives pickling and
    `torch.load(weights_only=True)` of a saved memory, slam/model.py:431-440; a numpy attribute would not.)"""
    sh = getattr(mem_labels, "_m3r_labels_host", None)
    if sh is None or mem_labels.dim() != 2 or mem_labels.shape[0] != 1 or sh.shape[0] != mem_labels.shape[1]:
        return None
    return sh.numpy()


def _set_host_labels(mem_labels, shadow):
    try:
        if shadow is not None and not torch.is_tensor(shadow):
            shadow = torch.from_numpy(np.ascontiguousarray(shadow, dtype=np.int64))
        mem_labels._m3r_labels_host = shadow
    except Exception:  # noqa: BLE001  (tensor subclasses that refuse attributes)
        pass
    return mem_labels


def _runs(mask):
    """[(start, stop)] of the True runs of a 1-D bool array."""
    if mask.size == 0:
        return []
    edges = np.flatnonzero(np.diff(np.concatenate(([False], mask, [False])).astype(np.int8)))
    return list(zip(edges[0::2].tolist(), edges[1::2].tolist()))


def _shadow_after_call(mem_before, new_mem, idx_st, x_st):
    """Attach the host label row to the memory a decoder update call returned: previous row + for every aspect-ratio
    group, in call order, the labels mem_nimgs + k repeated over the view's N tokens (decoder.py:237-247)."""
    prev = np.zeros((0,), dtype=np.int64) if mem_before is None else _host_labels(mem_before[1])
    if prev is None or new_mem[1].dim() != 2 or new_mem[1].shape[0] != 1:
        return new_mem
    first = 0 if mem_before is None else int(mem_before[2])
    parts, off = [prev], 0
    for ids, xg in zip(idx_st, x_st):
        nv, N = len(ids), int(xg.shape[-2])
        parts.append(np.repeat(np.arange(first + off, first + off + nv, dtype=np.int64), N))
        off += nv
    sh = np.concatenate(parts)
    if sh.shape[0] == new_mem[1].shape[1]:
        _set_host_labels(new_mem[1], sh)
    return new_mem


def _arena_of(mem_values):
    """The growable backing store of a memory produced by the CUDA decoder (model/decoder.py MemArena), or None."""
    a = getattr(mem_values[0], "_m3r_arena", None) if len(mem_values) else None
    if a is None:
        return None
    from ..model.decoder import MemArena
    a = MemArena.of(mem_values)
    return a if (a is not None and a.tail == mem_values[0].shape[1]) else None      # only the latest version may be edited in place


def _release_tail(mem):
    """The engine discards the memory a decoder call returned and keeps `mem` (refinement passes): give the rows appended
    behind `mem` back, so that the next call on `mem` appends in place again."""
    if mem is None:
        return
    a = getattr(mem[0][0], "_m3r_arena", None)
    if a is not None:
        from ..model.decoder import MemArena
        if MemArena.of(mem[0]) is a and a.tail >= mem[0][0].shape[1]:
            a.tail = mem[0][0].shape[1]


def _reserve(decoder, n_tokens=0, growth=0.0):
    fn = getattr(decoder, "reserve_memory", None)
    if fn is not None:
        fn(n_tokens, growth)


def _remove_from_mem(mem_values, mem_labels, idx):
    """Drop every token labelled idx (engine/inference.py:205-213)."""
    sh = _host_labels(mem_labels)
    if sh is None:
        keep = mem_labels != idx
        B, _, D = mem_values[0].shape
        return [v[keep].view(B, -1, D) for v in mem_values], mem_labels[keep].view(B, -1)
    keep = sh != idx
    runs = _runs(keep)
    if len(runs) == 1 and runs[0] == (0, sh.shape[0]):
        return mem_values, mem_labels
    arena = _arena_of(mem_values)
    if len(runs) <= 1 and (not runs or runs[0][0] == 0):
        stop = runs[0][1] if runs else 0                       # the dropped tokens are the tail: prefix views, no copy
        if arena is not None:
            arena.tail = stop                                  # ... and the next decoder call appends right behind them
            values = arena.views(stop)
        else:
            values = [v[:, :stop] for v in mem_values]
        labels = mem_labels[:, :stop]
    elif arena is not None:
        # compaction inside the growable buffers: only the rows behind the hole move (through a scratch copy: source and
        # destination overlap), the memory keeps its storage and the next decoder call appends in place
        pos = 0
        for a, b in runs:
            if a != pos:
                for buf in arena.bufs:
                    buf[:, pos:pos + (b - a)] = buf[:, a:b].clone()
            pos += b - a
        arena.tail = pos
        values = arena.views(pos)
        labels = torch.cat([mem_labels[:, a:b] for a, b in runs], dim=1)
    else:
        values = [torch.cat([v[:, a:b] for a, b in runs], dim=1) for v in mem_values]
        labels = torch.cat([mem_labels[:, a:b] for a, b in runs], dim=1)
    return values, _set_host_labels(labels, sh[keep])


def _restore_label_in_mem(mem_labels, old_idx_to_restore, new_idx_to_remove):
    """engine/inference.py:216-219"""
    sh = _host_labels(mem_labels)
    mem_labels[mem_labels == new_idx_to_remove] = old_idx_to_restore
    if sh is not None:
        sh = sh.copy()
        sh[sh == new_idx_to_remove] = old_idx_to_restore
        _set_host_labels(mem_labels, sh)
    return mem_labels


def _update_in_mem(old_values, new_values, old_labels, new_labels, old_idx, new_idx):
    """Overwrite the tokens labelled old_idx with those labelled new_idx (engine/inference.py:222-228)."""
    osh, nsh = _host_labels(old_labels), _host_labels(new_labels)
    if osh is not None and nsh is not None:
        dst, src = _runs(osh == old_idx), _runs(nsh == new_idx)
        if len(dst) == 1 and len(src) == 1 and dst[0][1] - dst[0][0] == src[0][1] - src[0][0]:
            (a, b), (c, d) = dst[0], src[0]
            for k in range(len(old_values)):
                old_values[k][:, a:b] = new_values[k][:, c:d]
            return old_values
    dst, src = old_labels == old_idx, new_labels == new_idx
    for k in range(len(old_values)):
        old_values[k][dst] = new_values[k][src]
    return old_values


def _refresh_in_mem(mem_values, mem_labels, old_idx, new_idx):
    """Keyframe refresh of a refinement pass (engine/inference.py:315-339): the rows labelled old_idx take the values of the
    rows labelled new_idx, which then disappear.  On one GPU both sets live in the same memory.  With a memory sharded over
    several GPUs (engine/context_parallel.py) the fresh rows may have been stored by another rank: that rank keeps them
    under the keyframe's label, and the rank holding the stale rows forgets them - the union of the shards is the same set."""
    sh = _host_labels(mem_labels)
    if sh is not None:
        n_dst, n_src = int((sh == old_idx).sum()), int((sh == new_idx).sum())
    else:
        n_dst, n_src = int((mem_labels == old_idx).sum()), int((mem_labels == new_idx).sum())
    if n_dst == n_src:
        if n_dst:
            mem_values = _update_in_mem(mem_values, mem_values, mem_labels, mem_labels, old_idx, new_idx)
        return _remove_from_mem(mem_values, mem_labels, new_idx)
    if n_src == 0:
        return _remove_from_mem(mem_values, mem_labels, old_idx)
    if n_dst == 0:
        return mem_values, _restore_label_in_mem(mem_labels, old_idx, new_idx)
    raise RuntimeError(f"inconsistent memory shards: {n_dst} rows labelled {old_idx}, {n_src} labelled {new_idx}")


def _compact_storage(mem):
    """Memory tensors handed back to the caller own exactly their rows (a prefix view would drag the evicted frames'
    storage along, e.g. into a pickle, slam/model.py:431-440)."""
    vals = [v.clone() if v.untyped_storage().nbytes() > v.numel() * v.element_size() else v for v in mem[0]]
    lab = mem[1]
    if lab.untyped_storage().nbytes() > lab.numel() * lab.element_size():
        lab = _set_host_labels(lab.clone(), getattr(lab, "_m3r_labels_host", None))
    return [vals, lab] + list(mem[2:])


def _fresh_labels(new_mem, n_before, mem_before=None, n_new_views=None):
    """Labels given to the views of the last decoder call.  The reference reads them back from the label tensor
    (`sorted(torch.unique(new_mem[1][:, Nmem_before:]))`, engine/inference.py:290,426 - a device sync per step); the decoder
    assigns them deterministically as mem_nimgs + arange(n) (decoder.py:242-247,332-336), so they are computed on the host
    when the call's view count is known."""
    if n_new_views is not None:
        first = 0 if mem_before is None else int(mem_before[2])
        return list(range(first, first + n_new_views))
    return [int(v) for v in sorted(torch.unique(new_mem[1][:, n_before:]))]


def _ensure_features(encoder, x, pos, imgs, true_shape, lo, hi, max_bs, device):
    xi, pi = x[lo:hi], pos[lo:hi]
    if None in xi or None in pi:
        xi, pi = encoder_multi_ar(encoder, imgs[lo:hi], true_shape[lo:hi], verbose=False, max_bs=max_bs, device=device)
        x[lo:hi], pos[lo:hi] = xi, pi
    return xi, pi


# --------------------------------------------------------------------------------------------- missing encoder features
# When the caller leaves the encoding to the engine (encoder_precomputed_features=None: what the reference's demo does,
# must3r/demo/inference.py:198), the reference encodes each step's views right before the decoder call
# (engine/inference.py:270-276,400-406): one ViT-L pass per view, M = 768 rows, far below the GEMMs' efficient size.  With the
# CUDA encoder the missing views are encoded UP FRONT, in large same-shape batches, then the decoder chain runs: measured on
# C3 63.3 ms vs 88.7 ms for per-step encoding.  (Encoding on a side stream NEXT to the latency-bound chain - SM-capped
# persistent GEMMs, chain on a high-priority stream - was measured too and lost: 70.5 .. 93.9 ms, the chain's one-wave kernels
# wait for SMs.)  Same kernels, same per-view features (rows are independent).
ENCODE_AHEAD_BATCH = 50


def _encode_missing_upfront(encoder, imgs, true_shape, x, pos, device, max_bs=None):
    """Fill x / pos for every view whose features are missing, in batches of views with one true_shape (CUDA encoder only)."""
    if not str(device).startswith("cuda") or not getattr(encoder, "batches_well", False):
        return
    missing = [i for i in range(len(x)) if x[i] is None or pos[i] is None]
    if len(missing) < 2:
        return
    bs = min(ENCODE_AHEAD_BATCH, max_bs) if max_bs else ENCODE_AHEAD_BATCH
    groups = {}
    for i in missing:
        groups.setdefault(tuple(int(v) for v in true_shape[i].tolist()), []).append(i)
    for ids in groups.values():
        for lo in range(0, len(ids), bs):
            b = ids[lo:lo + bs]
            xs, ps = encoder(torch.stack([imgs[i] for i in b]).to(device), torch.stack([true_shape[i] for i in b]).to(device))
            for j, v in enumerate(b):
                x[v], pos[v] = xs[j], ps[j]


def _default_is_keyframe(id, res, scene_state):
    return id % 3 == 0


def _default_scene_state_update(res, scene_state):
    return scene_state


# --------------------------------------------------------------------------------------------- video / rolling window
@torch.no_grad()
def inference_video_multi_ar(encoder, decoder, imgs, true_shape, mem_batches, verbose=False, max_bs=None,
                             encoder_precomputed_features=None, preserve_gpu_mem=False,
                             post_process_function=lambda x: {'pts3d': x}, device=None, return_mem=False,
                             viser_server=None, num_refinements_iterations=0, local_context_size=25,
                             is_keyframe_function=None, scene_state=None, scene_state_update_function=None):
    """Streaming schedule with keyframes and a rolling window of recent frames (engine/inference.py:231-366).
    Default callbacks as in the reference: keyframe iff id % 3 == 0 (:236), scene state passed through (:237)."""
    is_keyframe_function = is_keyframe_function or _default_is_keyframe
    scene_state_update_function = scene_state_update_function or _default_scene_state_update
    true_shape = torch.stack(true_shape, dim=0)
    n = true_shape.shape[0]
    device = device or true_shape.device
    x, pos = ([None] * n, [None] * n) if encoder_precomputed_features is None else encoder_precomputed_features
    bounds = [0] + np.cumsum(mem_batches).tolist()
    first_pass = [None] * bounds[-1]
    mem = None
    label_of, keyframes = {}, set()
    custom_callbacks = (viser_server is not None or is_keyframe_function is not _default_is_keyframe
                        or scene_state_update_function is not _default_scene_state_update)
    window = deque()
    _reserve(decoder, 0, 1.5)                  # CUDA decoder: memory buffers grow geometrically, updates append in place
    _encode_missing_upfront(encoder, imgs, true_shape, x, pos, device, max_bs)
    for _ in range(num_refinements_iterations + 1):
        window = deque()
        for step in range(len(bounds) - 1):
            lo, hi = bounds[step], bounds[step + 1]
            ts_i, imgs_i, ids_i = true_shape[lo:hi], imgs[lo:hi], list(range(lo, hi))
            x_i, pos_i = _ensure_features(encoder, x, pos, imgs, true_shape, lo, hi, max_bs, device)
            ts_st, idx_st, x_st, pos_st, img_st = stack_views(ts_i, [x_i, pos_i, imgs_i], max_bs=max_bs)
            n_before = get_Nmem(mem)
            mem_prev = mem
            new_mem, res = _multi_ar_batch(encoder, decoder, img_st, ts_st, mem, verbose=verbose,
                                                    encoder_precomputed_features=(x_st, pos_st),
                                                    preserve_gpu_mem=preserve_gpu_mem,
                                                    post_process_function=post_process_function, device=device,
                                                    viser_server=viser_server)
            res = unstack_pointmaps(idx_st, res)
            first_pass[lo:hi] = res
            mem = list(_shadow_after_call(mem_prev, new_mem, idx_st, x_st))
            new_labels = _fresh_labels(mem, n_before, mem_prev, hi - lo)
            if custom_callbacks:
                _sync_host_copies()        # user callbacks may read the (host) results
            flags = []
            if not label_of:                       # initialisation: every view is a keyframe
                for j, vid in enumerate(ids_i):
                    label_of[vid] = new_labels[j]
                    window.append(vid)
                    keyframes.add(vid)
                    flags.append(True)
                    scene_state = scene_state_update_function(res[j], scene_state)
            else:
                for j, vid in enumerate(ids_i):
                    seen = vid in label_of
                    is_kf = (vid in keyframes) if seen else is_keyframe_function(vid, res[j], scene_state)
                    window.append(vid)
                    flags.append(is_kf)
                    if is_kf and seen:             # refinement pass: refresh the stored tokens of this keyframe
                        old = label_of[vid]
                        if old != 0:               # the reference image is never refreshed
                            mem[0], mem[1] = _refresh_in_mem(mem[0], mem[1], old, new_labels[j])
                        else:
                            mem[0], mem[1] = _remove_from_mem(mem[0], mem[1], new_labels[j])
                    elif seen:                     # known non-keyframe: keep its tokens under the old label
                        mem[1] = _restore_label_in_mem(mem[1], label_of[vid], new_labels[j])
                    else:
                        label_of[vid] = new_labels[j]
                        if is_kf:
                            keyframes.add(vid)
                            scene_state = scene_state_update_function(res[j], scene_state)
            if viser_server is not None:
                viser_server.set_views([torch.tensor(v) for v in ids_i], imgs_i, res, flags)
            while len(window) > local_context_size:      # evict frames that left the local window
                gone = window.popleft()
                if gone not in keyframes:
                    mem[0], mem[1] = _remove_from_mem(mem[0], mem[1], label_of[gone])
            mem[2] = len(label_of)
        assert mem is not None
        while window:                                   # between passes only keyframes stay
            gone = window.popleft()
            if gone not in keyframes:
                mem[0], mem[1] = _remove_from_mem(mem[0], mem[1], label_of[gone])
    _reserve(decoder)
    _sync_host_copies()
    return (_compact_storage(mem), first_pass) if return_mem else first_pass


# --------------------------------------------------------------------------------------------- offline keyframes + render
@torch.no_grad()
def inference_multi_ar(encoder, decoder, imgs, img_ids, true_shape, mem_batches, verbose=False, max_bs=None,
                       to_render=None, encoder_precomputed_features=None, precomputed_mem=None, preserve_gpu_mem=False,
                       post_process_function=lambda x: {'pts3d': x}, device=None, return_mem=False, viser_server=None,
                       num_refinements_iterations=0):
    """Build the memory from the first sum(mem_batches) views, optionally refine it, then render
    (engine/inference.py:369-527)."""
    true_shape = torch.stack(true_shape, dim=0)
    n = true_shape.shape[0]
    device = device or true_shape.device
    x, pos = ([None] * n, [None] * n) if encoder_precomputed_features is None else encoder_precomputed_features
    if precomputed_mem is None:
        mem = None
        bounds = [0] + np.cumsum(mem_batches).tolist()
        first_pass = [None] * bounds[-1]
        label_of = {}
        # CUDA decoder: size the memory buffers once for the whole schedule, every update then appends in place
        known = [v for v in x[:bounds[-1]] if v is not None]
        _encode_missing_upfront(encoder, imgs, true_shape, x, pos, device, max_bs)
        known = [v for v in x[:bounds[-1]] if v is not None]
        if len(known) == bounds[-1]:
            # (a refinement pass re-runs every step against the full memory: keep room for the largest step's rows, which
            # the engine hands back after copying the refreshed ones - _release_tail)
            steps = [sum(int(v.shape[-2]) for v in known[bounds[k]:bounds[k + 1]]) for k in range(len(bounds) - 1)]
            _reserve(decoder, sum(steps) + (max(steps) if num_refinements_iterations > 0 else 0), 0.0)
        else:
            _reserve(decoder, 0, 1.5)
        for _ in range(num_refinements_iterations + 1):
            for step in range(len(bounds) - 1):
                lo, hi = bounds[step], bounds[step + 1]
                ts_i, imgs_i, ids_i = true_shape[lo:hi], imgs[lo:hi], img_ids[lo:hi]
                x_i, pos_i = _ensure_features(encoder, x, pos, imgs, true_shape, lo, hi, max_bs, device)
                ts_st, idx_st, x_st, pos_st, img_st = stack_views(ts_i, [x_i, pos_i, imgs_i], max_bs=max_bs)
                refresh = all(int(v) in label_of for v in ids_i)     # all views already stored: refinement step
                new_mem, res = _multi_ar_batch(encoder, decoder, img_st, ts_st, mem, verbose=verbose,
                                                        encoder_precomputed_features=(x_st, pos_st),
                                                        preserve_gpu_mem=preserve_gpu_mem,
                                                        post_process_function=post_process_function, device=device,
                                                        viser_server=viser_server)
                new_labels = _fresh_labels(new_mem, get_Nmem(mem), mem, hi - lo)
                new_mem = _shadow_after_call(mem, new_mem, idx_st, x_st)
                if refresh:
                    assert mem is not None
                    for j, vid in enumerate(ids_i):
                        old = label_of[int(vid)]
                        if old == 0:
                            continue                                  # reference image: left as is
                        _update_in_mem(mem[0], new_mem[0], mem[1], new_mem[1], old, new_labels[j])
                    del new_mem
                    _release_tail(mem)
                else:
                    mem = new_mem
                    for j, vid in enumerate(ids_i):
                        label_of[int(vid)] = int(new_labels[j])
                res = unstack_pointmaps(idx_st, res)
                first_pass[lo:hi] = res
                if viser_server is not None:
                    _sync_host_copies()
                    viser_server.set_views(ids_i, imgs_i, res, [True] * len(imgs_i))
        _reserve(decoder)
    else:
        first_pass, mem = None, precomputed_mem
        _encode_missing_upfront(encoder, imgs, true_shape, x, pos, device, max_bs)

    if to_render is not None:
        x, pos = [x[v] for v in to_render], [pos[v] for v in to_render]
        true_shape = true_shape[to_render].contiguous()
        imgs, img_ids = [imgs[v] for v in to_render], [img_ids[v] for v in to_render]
        n = len(x)
    assert mem is not None
    if n == 0:
        _sync_host_copies()
        return (mem, first_pass, []) if return_mem else (first_pass, [])

    ts_st, idx_st, x_st, pos_st, img_st, id_st = stack_views(true_shape, [x, pos, imgs, img_ids], max_bs=max_bs)
    rendered = []
    for xs, ps, ts, ims, ids in zip(x_st, pos_st, ts_st, img_st, id_st):
        feats = None if (xs is None or ps is None) else ([xs], [ps])
        _, out = _multi_ar_batch(encoder, decoder, [ims], [ts], mem, verbose=verbose,
                                          encoder_precomputed_features=feats, preserve_gpu_mem=preserve_gpu_mem,
                                          post_process_function=post_process_function, device=device, render=True,
                                          viser_server=viser_server)
        rendered.append(out[0])
        if viser_server is not None:
            _sync_host_copies()
            tmp = unstack_pointmaps([torch.arange(ids.shape[0])], out)
            for i in range(ids.shape[0]):
                viser_server.set_views([ids[i]], [ims[i]], [tmp[i]])
    pointmaps = unstack_pointmaps(idx_st, rendered)
    _sync_host_copies()
    return (mem, first_pass, pointmaps) if return_mem else (first_pass, pointmaps)


def groupby_consecutive(data):
    """Runs of consecutive integers as (first, last) pairs (engine/inference.py:555-567)."""
    if not data:
        return []
    data = sorted(data)
    runs = []
    for _, grp in itertools.groupby(enumerate(data), lambda t: t[1] - t[0]):
        grp = [v for _, v in grp]
        runs.append((grp[0], grp[-1]))
    return runs


# --------------------------------------------------------------------------------------------- batched tensor path
def inference_encoder(encoder, imgs, true_shape_view, max_bs=None, requires_grad=False):
    """imgs [B,nimgs,3,H,W] -> x [B,nimgs,N,D], pos [B,nimgs,N,2], optionally in slices of max_bs
    (engine/inference.py:570-592)."""
    with (nullcontext() if requires_grad else torch.no_grad()):
        B, n = imgs.shape[:2]
        flat = imgs.reshape(B * n, *imgs.shape[2:])
        if max_bs is None or B * n <= max_bs:
            x, pos = encoder(flat, true_shape_view)
        else:
            parts = [encoder(a, b) for a, b in zip(torch.split(flat, max_bs), torch.split(true_shape_view, max_bs))]
            x = torch.cat([p[0] for p in parts])
            pos = torch.cat([p[1] for p in parts])
        return x.view(B, n, *x.shape[1:]), pos.view(B, n, *pos.shape[1:])


def inference(encoder, decoder, imgs, true_shape, mem_batches, verbose=False, max_bs=None, train_decoder_skip=0,
              to_render=None, encoder_requires_grad=False):
    """Batched tensor path used by eval / training (engine/inference.py:595-688): B scenes x nimgs views,
    memory updates in steps of mem_batches, then render (all views or `to_render`), in slices of max_bs."""
    B, n = imgs.shape[:2]
    x, pos = inference_encoder(encoder, imgs, true_shape.view(B * n, 2), max_bs, encoder_requires_grad)
    N, D = x.shape[2:]
    bounds = [0] + np.cumsum(mem_batches).tolist()
    mem, outshape, first_pass = None, None, []
    for step in range(len(bounds) - 1):
        sl = slice(bounds[step], bounds[step + 1])
        ctx = torch.no_grad() if step < train_decoder_skip else nullcontext()
        with ctx:
            mem, pm = decoder(x[:, sl].contiguous(), pos[:, sl].contiguous(), true_shape[:, sl].contiguous(), mem,
                              render=False)
        outshape = outshape or pm.shape
        if step >= train_decoder_skip:
            first_pass.append(pm)
    if first_pass:
        pointmaps_0 = torch.cat(first_pass, dim=1)
    else:
        pointmaps_0 = torch.empty((B, 0, *outshape[2:]), dtype=x.dtype, device=x.device)
    if to_render is not None:
        x, pos = x[:, to_render].contiguous(), pos[:, to_render].contiguous()
        true_shape = true_shape[:, to_render].contiguous()
        n = x.shape[1]
    assert mem is not None
    mem_vals, mem_labels, mem_nimgs, mem_pi, mem_pt = mem
    if n == 0:
        return pointmaps_0, torch.empty((B, 0, *pointmaps_0.shape[2:]), dtype=x.dtype, device=x.device)
    if max_bs is None or B * n <= max_bs:
        _, pointmaps = decoder(x, pos, true_shape, mem, render=True)
        return pointmaps_0, pointmaps
    # chunked render: every (scene, view) pair becomes its own "scene" carrying a copy of its memory
    Nmem, Dmem = mem_vals[0].shape[1:]
    rep_vals = [m.unsqueeze(1).expand(B, n, Nmem, Dmem).reshape(B * n, Nmem, Dmem) for m in mem_vals]
    rep_labels = mem_labels.unsqueeze(1).expand(B, n, Nmem).reshape(B * n, Nmem)
    xv, pv, tv = x.reshape(B * n, N, D), pos.reshape(B * n, N, 2), true_shape.reshape(B * n, 2)
    outs = []
    for lo in range(0, B * n, max_bs):
        sl = slice(lo, lo + max_bs)
        _, pm = decoder(xv[sl].unsqueeze(1), pv[sl].unsqueeze(1), tv[sl].unsqueeze(1),
                        ([m[sl] for m in rep_vals], rep_labels[sl], mem_nimgs, mem_pi, mem_pt), render=True)
        outs.append(pm.squeeze(1))
    pointmaps = torch.cat(outs)
    return pointmaps_0, pointmaps.view(B, n, *pointmaps.shape[1:])


def concat_preds(out0, out):
    """engine/inference.py:691-695"""
    for k in out.keys():
        if k in out0:
            out[k] = torch.cat([out0[k], out[k]], dim=1)
    return out
