"""Host bookkeeping of the multi-session SLAM (must3r_b200/engine/slam_sessions.py): the arena's slots and growth, the
batching rule, and the command line's arguments.  No GPU."""
import pytest
import torch

from must3r_b200 import slam as single
from must3r_b200 import slam_sessions as cli
from must3r_b200.engine.slam_sessions import SessionArena, plan_batch, slot_runs


def test_arena_slots_and_growth():
    a = SessionArena(3, depth=2, width=8, dtype=torch.float16, device="cpu", growth=1.5)
    assert a.cap == 0 and a.lengths == [0, 0, 0]
    mem = [torch.arange(5 * 8, dtype=torch.float16).view(1, 5, 8) + l for l in range(2)]
    a.store(1, mem)
    assert a.cap == 5 and a.lengths == [0, 5, 0]
    v = a.views(1)
    assert a.holds(1, v) and not a.holds(0, v) and not a.holds(1, [t[:, :4] for t in v])
    assert all(torch.equal(x, m) for x, m in zip(v, mem))
    assert [t.shape for t in a.views(0)] == [(1, 0, 8)] * 2
    assert not a.ensure(5)
    a.lengths[2] = 3
    a.bufs[0][2, :3] = 7
    old = a.bufs
    assert a.ensure(6)                                   # geometric: 5 * 1.5 -> 8, every level, every slot's rows kept
    assert a.cap == 8 and all(b.shape == (3, 8, 8) for b in a.bufs) and a.bufs[0] is not old[0]
    assert torch.equal(a.views(1)[1], mem[1]) and bool((a.bufs[0][2, :3] == 7).all())
    assert all(torch.equal(x, m) for x, m in zip(v, mem))     # views handed out before stay valid
    assert a.ensure(20) and a.cap == 20                 # at least the rows asked for
    assert not a.holds(1, v)                            # ... but are no longer the slot's


def test_batching_rule():
    sh, other = (224, 224), (160, 224)
    assert plan_batch({0: sh, 1: sh, 2: sh}) == ([0, 1, 2], [])
    assert plan_batch({0: None, 1: sh, 2: sh}) == ([1, 2], [0])             # first frame / init re-run: alone
    assert plan_batch({0: other, 1: sh, 2: sh, 3: None}) == ([1, 2], [0, 3])   # the shape most frames share
    assert plan_batch({0: other, 1: sh}) == ([0], [1])                        # tie: the first shape
    assert plan_batch({2: sh}) == ([2], [])
    assert plan_batch({0: None, 1: None}) == ([], [0, 1])
    assert plan_batch({}) == ([], [])
    assert slot_runs([0, 1, 2]) == [[0, 1, 2]]
    assert slot_runs([0, 2, 3, 5]) == [[0], [2, 3], [5]]


def test_cli_arguments(tmp_path):
    d0, d1 = tmp_path / "a", tmp_path / "b"
    d0.mkdir()
    d1.mkdir()
    args = cli.parse_args(["--chkpt", "c.pth", "--sessions", str(d0), str(d1), "--output", str(tmp_path / "out")])
    assert args.sessions == [str(d0), str(d1)]
    ref = single.get_args_parser().parse_args(["--chkpt", "c.pth"])
    for name in cli.PROCESSING:                           # same names and defaults as python -m must3r_b200.slam
        if name != "output":
            assert getattr(args, name) == getattr(ref, name), name
    assert not hasattr(args, "input") and not hasattr(args, "gui")


@pytest.mark.parametrize("argv,msg", [
    (["--chkpt", "c", "--output", "o"], "--sessions"),
    (["--chkpt", "c", "--sessions", "{d}"], "--output"),
    (["--chkpt", "c", "--sessions", "{d}/missing", "--output", "o"], "no such folder"),
    (["--chkpt", "c", "--sessions", "{d}", "--output", "o", "--device", "cpu"], "CUDA"),
    (["--chkpt", "c", "--sessions", "{d}", "--output", "o", "--skip_every", "0"], "skip_every"),
    (["--chkpt", "c", "--sessions", "{d}", "--output", "o", "--res", "300"], "choice"),
    (["--chkpt", "c", "--sessions", "{d}", "--output", "o", "--input", "{d}"], "unrecognized"),
])
def test_cli_rejections(argv, msg, tmp_path, capsys):
    argv = [a.replace("{d}", str(tmp_path)) for a in argv]
    with pytest.raises(SystemExit):
        cli.parse_args(argv)
    assert msg in capsys.readouterr().err
