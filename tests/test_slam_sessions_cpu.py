"""Host bookkeeping of the multi-session SLAM (must3r_b200/engine/slam_sessions.py): the arena's slots and growth, the
batching rule, the split of a keyframe commit over launches, and the command line's arguments.  No GPU."""
import ctypes as C
from types import SimpleNamespace

import pytest
import torch

from must3r_b200 import ops
from must3r_b200 import slam as single
from must3r_b200 import slam_sessions as cli
from must3r_b200.engine import lockstep
from must3r_b200.engine.lockstep import SessionArena, plan_batch, slot_runs
from must3r_b200.engine.slam_sessions import SLAMSessions


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


def test_keyframe_commit_of_70_sessions_splits_over_launches(monkeypatch):
    """One run of 70 consecutive slots commits in launches of at most 64 sessions: each launch gets its sessions'
    staged blocks, their rows behind each memory, and the keyframe flag of its first session's record."""
    calls = []

    class Lib:
        def m3r_mem_commit_rows(self, arena, staged, depth, B, row0, rows, stride, width, dst, keep, keep_stride, stream):
            assert B <= 64 and (depth, row0, rows, stride, width) == (2, 0, 3, 3, 8)
            calls.append((B, staged[0], list(dst[:B]), keep.value, keep_stride))
            return 0
    monkeypatch.setattr(lockstep._lib, "lib", lambda: Lib())
    monkeypatch.setattr(lockstep.cm, "stream_ptr", lambda device: C.c_void_p(0))
    ss = SLAMSessions.__new__(SLAMSessions)              # only the arena and the slots: no model
    ss.arena = SessionArena(72, depth=2, width=8, dtype=torch.float16, device="cpu")
    ss.arena.ensure(20)
    ss.sessions = [SimpleNamespace(slot=s) for s in range(72)]
    members = list(range(1, 71))
    ss.arena.lengths = [s % 5 for s in range(72)]
    staged = [torch.zeros(70, 3, 8, dtype=torch.float16) for _ in range(2)]
    recs = torch.zeros((70, ops.SLAM_RECORD.itemsize), dtype=torch.uint8)
    ss._commit([(members, staged)], recs, {sid: i for i, sid in enumerate(members)})
    flag = ops.SLAM_RECORD.fields["keyframe"][1]
    assert [c[0] for c in calls] == [64, 6]
    for (B, src, dst, keep, stride), lo in zip(calls, (0, 64)):
        assert src == staged[0][lo].data_ptr()
        assert dst == [s * 20 + s % 5 for s in members[lo:lo + B]]
        assert keep == recs.data_ptr() + lo * ops.SLAM_RECORD.itemsize + flag and stride == ops.SLAM_RECORD.itemsize // 4


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
