"""The lockstep video schedule (must3r_b200/engine/videos.py) without a GPU: VideoPlan's memory layout and edits replayed
against inference_video_multi_ar behind the CPU oracle decoder, the lockstep calls of videos of different lengths and
shapes, the split of compaction runs over launches, and the command line of `python -m must3r_b200.reconstruct_videos`."""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import tiny_oracle
from must3r_b200 import engine, reconstruct, reconstruct_videos as cli, synthetic as syn
from must3r_b200.engine import videos
from must3r_b200.engine.videos import VideoPlan, plan_step_calls
from oracle import must3r_oracle as orc

SHAPES = [(32, 48), (48, 32), (32, 32)]         # 6, 6 and 4 tokens per view with the tiny oracle's 16-pixel patches


class Recorder:
    """The oracle decoder, recording per call the memory it was given (label row, level-0 rows) and the rows it added."""

    def __init__(self, dec):
        self.dec, self.calls = dec, []

    def __call__(self, x, pos, true_shape, mem, render=False):
        new_mem, pms = self.dec(x, pos, true_shape, mem, render=render)
        n0 = 0 if mem is None else mem[0][0].shape[1]
        before = None if mem is None else (mem[1][0].clone(), mem[0][0][0].clone())
        self.calls.append((before, new_mem[0][0][0, n0:].clone()))
        return new_mem, pms

    def __getattr__(self, name):
        return getattr(self.dec, name)


@pytest.fixture(scope="module")
def oracle():
    return tiny_oracle(7)


def frames(n, seed):
    rng = np.random.default_rng(seed)
    shapes = [SHAPES[0] if i < 2 else SHAPES[int(rng.integers(3))] for i in range(n)]
    imgs, tss = [], []
    for i, (H, W) in enumerate(shapes):
        im, ts = syn.synthetic_views(1, H, W, seed=seed * 100 + i)
        imgs.append(im[0])
        tss.append(ts[0])
    return imgs, tss, shapes, [bool(v) for v in rng.integers(0, 2, n)]


@pytest.mark.parametrize("n", [1, 2, 3, 12])
@pytest.mark.parametrize("refinements", [0, 1])
@pytest.mark.parametrize("context", [0, 1, 3, 25])
def test_layout_and_edits_replay_the_engine(oracle, n, refinements, context):
    """For random keyframe decisions and shapes: before every step, VideoPlan's label row equals the label row of the
    memory inference_video_multi_ar hands the decoder, and its edits (compaction runs applied one after another as
    clones, then the write of the staged rows that stay) applied to the rows each call added rebuild that memory's
    level-0 rows bit for bit.  After the last pass, its final label row is the engine's returned memory's."""
    enc, dec = oracle
    for seed in range(2):
        imgs, tss, shapes, pattern = frames(n, 1000 * n + 10 * context + seed)
        rec = Recorder(dec)
        mem, _ = engine.inference_video_multi_ar(
            enc, rec, imgs, tss, videos._mem_batches(n, 2, 1, n, n), max_bs=1, post_process_function=orc.postprocess,
            device="cpu", return_mem=True, local_context_size=context, num_refinements_iterations=refinements,
            is_keyframe_function=lambda vid, res, state: pattern[vid])
        plan = VideoPlan(shapes, context, refinements, max_bs=1)
        width = rec.calls[0][1].shape[-1]
        buf = torch.full((sum(v[1].shape[0] for v in rec.calls), width), float("nan"))
        schedule = [(it, k) for it in range(refinements + 1) for k in range(len(plan.steps))]
        assert len(schedule) == len(rec.calls)
        for (it, k), (before, staged) in zip(schedule, rec.calls):
            if before is None:
                assert plan.length == 0
            else:
                labels, values = before
                assert np.array_equal(plan.label_row(), labels.numpy()), (it, k)
                assert torch.equal(buf[:plan.length], values), (it, k)
            edit = plan.step(it, k, lambda vid: pattern[vid])
            for src, dst, rows in edit.runs:
                assert dst < src
                buf[dst:dst + rows] = buf[src:src + rows].clone()
            if edit.write is not None:
                row0, dst, rows = edit.write
                buf[dst:dst + rows] = staged[row0:row0 + rows]
            assert edit.length == plan.length
        assert np.array_equal(plan.final_label_row(), mem[1][0].numpy())
        want = [v for v in range(min(2, n))] + [v for v in range(2, n) if pattern[v]]
        assert plan.keyframes == want


def test_edits_of_a_steady_window():
    """One shape, local_context_size 2, keyframes 0, 1, 3: frame 2 leaves the window at step 3 (frame 4), its rows close
    up with one run; at local_context_size 0 a non-keyframe is never written."""
    N = 6
    p = VideoPlan([SHAPES[0]] * 6, 2)
    kf = {2: False, 3: True, 4: False, 5: False}.__getitem__
    assert p.step(0, 0).write == (0, 0, 2 * N)
    e = p.step(0, 1, kf)                                     # frame 2: window [0, 1, 2] -> 0, 1 leave (keyframes)
    assert e.runs == [] and e.write == (0, 2 * N, N) and e.length == 3 * N
    e = p.step(0, 2, kf)                                     # frame 3: window [2, 3]
    assert e.runs == [] and e.write == (0, 3 * N, N) and e.length == 4 * N
    e = p.step(0, 3, kf)                                     # frame 4: 2 leaves, 3 moves down over it, 4 behind
    assert e.runs == [(3 * N, 2 * N, N)] and e.write == (0, 3 * N, N) and e.length == 4 * N
    assert p.label_row().tolist() == sum([[v] * N for v in (0, 1, 3, 4)], [])
    q = VideoPlan([SHAPES[0]] * 4, 0)
    q.step(0, 0)
    e = q.step(0, 1, lambda v: False)
    assert e == videos.StepEdit([], None, 2 * N)


def test_lockstep_calls_of_videos():
    """Videos of 12, 3, 5 (a portrait frame at step 2) and 1 frames: step 0 shares one call (two landscape init views,
    cut at max_bs 1 into two groups), later steps share by shape and consecutive slots, and shorter videos drop out."""
    L, P = SHAPES[0], SHAPES[1]
    plans = [VideoPlan([L] * 12), VideoPlan([L] * 3), VideoPlan([L, L, L, P, L]), VideoPlan([L])]
    plans = [VideoPlan(p.shapes, 0, 0, max_bs=1) for p in plans]
    assert plan_step_calls(plans, 0) == [(((L, 1), (L, 1)), [0, 1, 2]), (((L, 1),), [3])]
    assert plan_step_calls(plans, 1) == [(((L, 1),), [0, 1, 2])]
    assert plan_step_calls(plans, 2) == [(((L, 1),), [0]), (((P, 1),), [2])]
    assert plan_step_calls(plans, 3) == [(((L, 1),), [0]), (((L, 1),), [2])]     # same signature, slots apart
    assert plan_step_calls(plans, 4) == [(((L, 1),), [0])]
    assert [len(p.steps) for p in plans] == [11, 2, 4, 1]
    # max_bs None: the init views in one group
    assert plan_step_calls([VideoPlan([L] * 4), VideoPlan([L] * 2)], 0) == [(((L, 2),), [0, 1])]


def test_compaction_runs_split_over_launches(monkeypatch):
    """More runs than one launch takes: every scene's runs go out in order, a scene cut at a launch boundary goes on in
    the next launch, and each launch's base rows are its slots' (ascending)."""
    calls = []

    class Lib:
        def m3r_mem_compact_rows(self, bufs, depth, B, width, cap, base, off, runs, stream):
            off = list(off)
            flat = list(runs[:3 * off[-1]])
            calls.append((list(base[:B]), [[tuple(flat[3 * k:3 * k + 3]) for k in range(off[b], off[b + 1])]
                                           for b in range(B)]))
            return 0
    monkeypatch.setattr(videos._lib, "lib", lambda: Lib())

    class Arena:
        depth, width, cap = 2, 64, 10000
        bufs = [torch.zeros(1), torch.zeros(1)]
    runs_of = {s: [(100 * k + 50, 100 * k, 10) for k in range(n)] for s, n in ((0, 5), (3, 200), (7, 60))}
    videos._compact_rows(Arena(), runs_of, C.c_void_p(0))
    assert [len(sum(r, [])) for _, r in calls] == [128, 128, 9]
    got = {}
    for base, per_scene in calls:
        assert base == sorted(base)
        for b, rs in zip(base, per_scene):
            got.setdefault(b // Arena.cap, []).extend(rs)
    assert got == runs_of


def test_cli_parsing_and_rejections(capsys):
    args = cli.parse_args(["--scenes", "a", "b", "--output", "o", "--execution_mode", "vidslam", "--amp", "bf16"])
    assert args.scenes == ["a", "b"] and args.execution_mode == "vidslam" and args.amp == "bf16"
    assert args.local_context_size == 0 and args.keyframe_interval == 3 and args.subsample == 2
    assert cli.parse_args(["--scenes", "a", "--output", "o", "--execution_mode", "vidseq"]).execution_mode == "vidseq"
    for bad, msg in ((["--execution_mode", "linseq"], "must3r_b200.reconstruct_scenes"),
                     ([], "must3r_b200.reconstruct_scenes"),                    # reconstruct's default mode is linseq
                     (["--execution_mode", "vidseq", "--retrieval", "r.pth"], "--retrieval"),
                     (["--execution_mode", "vidseq", "--memory_mode", "norm_y"], "memory_mode")):
        with pytest.raises(SystemExit):
            cli.parse_args(["--scenes", "a", "--output", "o"] + bad)
        assert msg in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli.parse_args(["--output", "o", "--execution_mode", "vidseq"])          # --scenes is required
    with pytest.raises(SystemExit):
        cli.parse_args(["--scenes", "a", "--image_dir", "x", "--output", "o", "--execution_mode", "vidseq"])
    shared = {a.dest for a in reconstruct.get_args_parser()._actions} - {"image_dir"}
    assert shared == {a.dest for a in cli.get_args_parser()._actions} - {"scenes"}
