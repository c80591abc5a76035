"""The lockstep schedule of several offline reconstructions (must3r_b200/engine/scenes.py) and the command line of
`python -m must3r_b200.reconstruct_scenes`, without a GPU."""
import pytest

from must3r_b200 import reconstruct, reconstruct_scenes as cli
from must3r_b200.engine import demo
from must3r_b200.engine.scenes import (ScenePlan, arena_rows, lockstep_calls, plan_memory_calls, plan_render_calls,
                                       signature)

L, P = (288, 384), (384, 288)          # landscape, portrait (H, W)
NL, NP = 18 * 24, 24 * 18              # tokens per view


def files(n, tag="f"):
    return [f"{tag}{i:02d}.png" for i in range(n)]


def test_plan_follows_must3r_inference():
    """Keyframes, order, file names, memory batches and views to render are must3r_inference's for the same arguments."""
    p = ScenePlan(files(10), [L] * 10, 4, max_bs=1)
    assert p.keyframes == demo._linspace_keyframes(10, 4) == [0, 3, 6, 9]
    assert p.order == [0, 3, 6, 9, 1, 2, 4, 5, 7, 8]
    assert p.filenames == [files(10)[i] for i in p.order]
    assert p.mem_batches == demo._mem_batches(10, 2, 1, 4, 4) == [2, 1, 1]
    # max_bs = 1 cuts the two init views into two groups, as stack_views does
    assert p.steps == [[(L, [0]), (L, [1])], [(L, [2])], [(L, [3])]]
    assert p.step_start == [0, 2 * NL, 3 * NL] and p.mem_rows == 4 * NL
    assert p.render_positions == list(range(10)) and p.first_positions == []
    assert p.render == [(L, [q]) for q in range(10)]
    once = ScenePlan(files(10), [L] * 10, 4, render_once=True, max_bs=3)
    assert once.first_positions == [0, 1, 2, 3] and once.render_positions == [4, 5, 6, 7, 8, 9]
    assert once.render == [(L, [4, 5, 6]), (L, [7, 8, 9])]
    assert once.steps[0] == [(L, [0, 1])]


def test_one_image_short_and_mixed_scenes():
    one = ScenePlan(files(1), [L], 50, max_bs=1)
    assert one.mem_batches == [1] and one.steps == [[(L, [0])]] and one.render == [(L, [0])] and one.mem_rows == NL
    with pytest.raises(ValueError):                     # must3r_inference's own schedule refuses it
        demo._mem_batches(1, 2, 1, 2, 1)
    short = ScenePlan(files(3), [L] * 3, 50, max_bs=1)
    assert short.keyframes == [0, 1, 2] and short.mem_batches == [2, 1]
    # mixed shapes: a portrait keyframe; the groups follow stack_views' lexicographic shape order
    shapes = [L, L, L, P, L, L]
    mixed = ScenePlan(files(6), shapes, 4, max_bs=None)
    assert mixed.keyframes == [0, 1, 3, 5] and [mixed.shapes[q] for q in range(4)] == [L, L, P, L]
    assert mixed.steps == [[(L, [0, 1])], [(P, [2])], [(L, [3])]]
    assert mixed.render == [(L, [0, 1, 3, 4, 5]), (P, [2])]
    init_mixed = ScenePlan(files(2), [P, L], 2, max_bs=None)
    assert init_mixed.steps == [[(L, [1]), (P, [0])]]      # (288, 384) sorts before (384, 288)
    assert init_mixed.refresh_row0(0) == NL and init_mixed.refresh_row0(1) == 0


def test_lockstep_calls_share_signatures_and_consecutive_slots():
    a, b = ((L, 1),), ((P, 1),)
    assert lockstep_calls([(0, a), (1, a), (2, b), (3, a)]) == [(a, [0, 1]), (a, [3]), (b, [2])]
    assert lockstep_calls([(0, b), (1, a)]) == [(b, [0]), (a, [1])]        # a tie: the first signature first
    assert lockstep_calls([]) == []


def test_schedule_of_three_scenes():
    """Scene 0: 10 landscape views; scene 1: 3 views (shorter than num_mem_images); scene 2: 6 views whose second
    memory step (order [0, 1, 3, 5, 2, 4]) is a portrait view."""
    plans = [ScenePlan(files(10), [L] * 10, 4, max_bs=1), ScenePlan(files(3), [L] * 3, 4, max_bs=1),
             ScenePlan(files(6), [L, L, L, P, L, L], 4, max_bs=1)]
    one_l, one_p = ((L, 1),), ((P, 1),)
    mem = plan_memory_calls(plans)
    assert mem == [(0, 0, ((L, 1), (L, 1)), [0, 1, 2]),
                   (0, 1, one_l, [0, 1]), (0, 1, one_p, [2]),
                   (0, 2, one_l, [0]), (0, 2, one_l, [2])]          # scene 1 has no third step: slots 0 and 2 apart
    ref = plan_memory_calls(plans, num_refinements_iterations=1)
    assert ref[:5] == mem and ref[5:] == [(1,) + c[1:] for c in mem]
    assert [p.mem_rows for p in plans] == [4 * NL, 3 * NL, 3 * NL + NP]
    assert arena_rows(plans) == 4 * NL
    assert plans[2].render == [(L, [0]), (L, [1]), (L, [3]), (L, [4]), (L, [5]), (P, [2])]
    render = plan_render_calls(plans)
    assert render[:3] == [(c, one_l, [0, 1, 2]) for c in range(3)]
    assert render[3:9] == [(3, one_l, [0]), (3, one_l, [2]), (4, one_l, [0]), (4, one_l, [2]), (5, one_l, [0]),
                           (5, one_p, [2])]
    assert render[9:] == [(c, one_l, [0]) for c in range(6, 10)]
    assert signature(plans[2].steps[1]) == one_p


def test_refresh_rows_skip_the_reference_view():
    p = ScenePlan(files(5), [L] * 5, 3, max_bs=None)
    assert p.steps == [[(L, [0, 1])], [(L, [2])]]
    # re-run of the init step: staged rows [NL, 2 NL) over memory rows [NL, 2 NL); later steps whole
    assert p.refresh_row0(0) == NL and p.step_start[0] + p.refresh_row0(0) == NL
    assert p.refresh_row0(1) == 0 and p.step_start[1] == 2 * NL


def test_cli_parsing_and_rejections(capsys):
    args = cli.parse_args(["--scenes", "a", "b", "--output", "o", "--max_bs", "2", "--amp", "bf16"])
    assert args.scenes == ["a", "b"] and args.output == "o" and args.max_bs == 2 and args.amp == "bf16"
    assert args.execution_mode == "linseq" and args.num_mem_imgs == 50
    assert cli.parse_args(["--scenes", "a", "--output", "o", "--amp", "False"]).amp is False
    for bad, msg in ((["--execution_mode", "vidseq"], "must3r_b200.reconstruct"),
                     (["--execution_mode", "vidslam"], "must3r_b200.reconstruct"),
                     (["--retrieval", "r.pth"], "--retrieval"),
                     (["--memory_mode", "norm_y"], "memory_mode")):
        with pytest.raises(SystemExit):
            cli.parse_args(["--scenes", "a", "--output", "o"] + bad)
        assert msg in capsys.readouterr().err
    with pytest.raises(SystemExit):
        cli.parse_args(["--output", "o"])                     # --scenes is required
    with pytest.raises(SystemExit):
        cli.parse_args(["--scenes", "a", "--image_dir", "x", "--output", "o"])
    # reconstruct's own parser keeps its arguments
    r = reconstruct.parse_args(["--image_dir", "d", "--output", "o"])
    assert r.image_dir == "d" and not hasattr(r, "scenes")
    shared = {a.dest for a in reconstruct.get_args_parser()._actions} - {"image_dir"}
    assert shared == {a.dest for a in cli.get_args_parser()._actions} - {"scenes"}
