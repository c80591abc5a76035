"""Several SLAM sessions on one GPU (must3r_b200/engine/slam_sessions.py): the ragged decoder call and the keyframe
commit (csrc/model.cu), then whole sessions against SLAM_MUSt3R run alone on the same frames and against the reference's
run (tests/golden/slam.npz), and the command line against `python -m must3r_b200.slam` per folder."""
import ast
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from must3r_b200 import _lib
from must3r_b200.engine import slam, slam_sessions
from must3r_b200.engine.images import preproc_frame
from must3r_b200.engine.slam_sessions import SLAMSessions
from must3r_b200.model import common as cm
from must3r_b200.model import load_model

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_slam_cli_golden as mkc  # noqa: E402
import make_slam_golden as mk  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {torch.float16: 3e-3, torch.bfloat16: 2.5e-2}        # tests/test_model_gpu.py
E2E = mk.RUNS["e2e"]


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(HERE, "golden", "slam.npz"))


@pytest.fixture(scope="module")
def chkpt(tmp_path_factory):
    p = str(tmp_path_factory.mktemp("sessions") / "tiny.pth")
    mk.write_checkpoint(p)
    return p


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_ragged_decoder_matches_separate_calls(chkpt, dtype):
    """Four scenes with memories of 1, 3, 2 and 5 views (196 tokens each) in one [4, cap, 2D] arena whose rows past each
    length are NaN: one ragged update_tokens call gives each scene's pointmaps and new rows as its own call does."""
    prev = cm.get_precision()
    cm.set_precision(dtype)
    try:
        enc, dec = load_model(chkpt, device="cuda")
        views = [preproc_frame(im, i, res=224, device="cuda")[0] for i, im in enumerate(mk.frames(15, seed=4))]

        def encode(vs):
            ts = torch.as_tensor(np.concatenate([v["true_shape"] for v in vs]))
            x, pos = enc(torch.cat([v["img"] for v in vs]), ts)
            return x, pos, ts

        n_views, mems, k = [1, 3, 2, 5], [], 0
        for n in n_views:
            x, pos, ts = encode(views[k:k + n])
            mem, _ = dec(x[None], pos[None], ts[None], None)
            mems.append(mem)
            k += n
        lens = [m[0][0].shape[1] for m in mems]
        cap = max(lens) + 50
        arena = [torch.full((4, cap, 2 * dec.embed_dim), float("nan"), dtype=dtype, device="cuda") for _ in range(dec.depth)]
        for b, m in enumerate(mems):
            for l in range(dec.depth):
                arena[l][b, :lens[b]] = m[0][l][0]
        xq, pq, tq = encode(views[k:k + 4])
        new_b, pm_b = dec.update_tokens(xq[:, None], pq[:, None], tq.view(4, 1, 2), current_mem=(arena, None, 0, 0, 0),
                                        mem_lengths=lens)
        for b, m in enumerate(mems):
            new_s, pm_s = dec.update_tokens(xq[b:b + 1, None], pq[b:b + 1, None], tq[b:b + 1].view(1, 1, 2), current_mem=m)
            assert bool(torch.isfinite(pm_b[b]).all())
            assert rel(pm_b[b:b + 1].float(), pm_s.float()) < TOL[dtype], b
            for l in range(dec.depth):
                assert rel(new_b[l][b:b + 1].float(), new_s[l].float()) < TOL[dtype], (b, l)
        with pytest.raises(ValueError):
            dec.update_tokens(xq[:, None], pq[:, None], tq.view(4, 1, 2), current_mem=(arena, None, 0, 0, 0),
                              mem_lengths=lens[:3])
        with pytest.raises(ValueError):
            dec.update_tokens(xq[:, None], pq[:, None], tq.view(4, 1, 2), current_mem=(arena, None, 0, 0, 0),
                              mem_lengths=[0, 0, 0, 0])
    finally:
        cm.set_precision(prev)


def test_ragged_decoder_argument_errors(chkpt):
    enc, dec = load_model(chkpt, device="cuda")
    w = dec._packed(cm.get_precision())
    call = cm.DecoderCall()
    nm = torch.ones(1, dtype=torch.int32, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    lib = _lib.lib()
    for field, value, msg in (("new_only", 0, b"new_only"), ("render", 1, b"new_only"), ("mem_mode", 1, b"kv"),
                              ("Nm", 0, b"Nm")):
        call = cm.DecoderCall()
        call.B, call.G, call.Nm, call.new_only, call.mem_mode = 1, 1, 10, 1, 0
        setattr(call, field, value)
        rc = lib.m3r_decoder_forward_ragged(C.byref(w), C.byref(call), C.c_void_p(nm.data_ptr()), C.c_void_p(ws.data_ptr()),
                                            ws.numel(), cm.stream_ptr(torch.device("cuda")))
        assert rc != 0 and msg in lib.m3r_last_error(), field
    assert lib.m3r_decoder_forward_ragged(C.byref(w), C.byref(call), None, C.c_void_p(ws.data_ptr()), ws.numel(), None) != 0


def commit(arena, staged, dst_rows, keep, stride, keep_byte_offset=0):
    lib = _lib.lib()
    a = (C.c_void_p * len(arena))(*[t.data_ptr() for t in arena])
    s = (C.c_void_p * len(staged))(*[t.data_ptr() for t in staged])
    rows = (C.c_int64 * len(dst_rows))(*dst_rows)
    Nt = staged[0].shape[1]
    return lib.m3r_mem_commit_rows(a, s, len(arena), staged[0].shape[0], 0, Nt, Nt, staged[0].shape[2], rows,
                                   C.c_void_p(keep.data_ptr() + keep_byte_offset), stride,
                                   cm.stream_ptr(torch.device("cuda")))


def test_mem_commit_rows_appends_exactly_the_flagged_rows():
    S, cap, W, B, Nt, depth = 4, 50, 256, 3, 7, 3
    sentinel = 7.0
    arena = [torch.full((S, cap, W), sentinel, dtype=torch.float16, device="cuda") for _ in range(depth)]
    staged = [torch.randn(B, Nt, W, device="cuda").half() for _ in range(depth)]
    keep = torch.tensor([1, -5, 0, 99, 1, 3], dtype=torch.int32, device="cuda")   # stride 2: flags 1, 0, 1
    dst = [0 * cap + 5, 2 * cap + 0, 3 * cap + cap - Nt]
    assert commit(arena, staged, dst, keep, 2) == 0
    torch.cuda.synchronize()
    for l in range(depth):
        want = torch.full((S * cap, W), sentinel, dtype=torch.float16, device="cuda")
        for b in (0, 2):
            want[dst[b]:dst[b] + Nt] = staged[l][b]
        assert torch.equal(arena[l].view(S * cap, W), want), l
    lib = _lib.lib()
    assert commit(arena, staged, dst, keep, 2, keep_byte_offset=2) != 0 and b"aligned" in lib.m3r_last_error()
    assert commit(arena, [t[..., :252] for t in staged], dst, keep, 2) != 0
    assert commit(arena, staged, [0, -1, 2], keep, 2) != 0 and b"dst_row" in lib.m3r_last_error()
    big = [torch.zeros(65, 1, 8, dtype=torch.float16, device="cuda")]
    assert commit(arena[:1], big, list(range(65)), keep, 0) != 0


# ------------------------------------------------------------------------------------------------ whole sessions
def _alone(chkpt, frames, **kw):
    s = slam.SLAM_MUSt3R(chkpt, device="cuda:0", **{**E2E, **kw})
    outs = [s(im, i, 0) for i, im in enumerate(frames)]
    return s, outs


def _stepped(ss, seqs):
    outs = [[] for _ in seqs]
    for k in range(max(len(s) for s in seqs)):
        res = ss.step({i: (seq[k], k, 0) for i, seq in enumerate(seqs) if k < len(seq)})
        for i, o in res.items():
            outs[i].append(o)
    return outs


@pytest.fixture(scope="module")
def three(chkpt, tmp_path_factory):
    """Session 0: the golden e2e sequence; 1: 8 other frames; 2: 10 other frames from a memory saved after 5 frames."""
    d = tmp_path_factory.mktemp("three")
    pre, _ = _alone(chkpt, mk.frames(5, seed=9), keep_memory=True)
    mem = str(d / "pre.pkl")
    pre.save_memory(mem)
    seqs = [mk.frames(), mk.frames(8, seed=5), mk.frames(10, seed=7)]
    args = [{}, {}, dict(load_memory=mem, keep_memory=True)]
    ss = SLAMSessions(chkpt, 3, device="cuda:0", session_args=args, **E2E)
    outs = _stepped(ss, seqs)
    return dict(ss=ss, seqs=seqs, args=args, outs=outs, dir=d)


def test_golden_session_reproduces_the_reference(three, g):
    ss, outs = three["ss"], three["outs"]
    s = ss[0]
    assert s.keyframes == g["e2e_keyframes"].tolist()
    np.testing.assert_allclose(torch.stack(s.all_poses).cpu().numpy(), g["e2e_poses"], atol=3e-2)
    assert ss.stats["batched"] > 0 and ss.stats["alone"] > 0
    s.rerender_all_frames(maxbs=5)
    np.testing.assert_allclose(torch.stack(s.all_poses).cpu().numpy(), g["e2e_rerender_poses"], atol=3e-2)


@pytest.mark.parametrize("i", [0, 1, 2])
def test_sessions_match_slam_run_alone(three, chkpt, i, tmp_path):
    s, outs = three["ss"][i], three["outs"][i]
    a, aouts = _alone(chkpt, three["seqs"][i], **three["args"][i])
    assert s.keyframes == a.keyframes
    assert [o[-1] for o in outs] == [o[-1] for o in aouts]
    assert len(s.all_poses) == len(a.all_poses) and s.all_timestamps == a.all_timestamps
    for o, ao in zip(outs, aouts):
        np.testing.assert_allclose(o[5].cpu().numpy(), ao[5].cpu().numpy(), atol=3e-2)      # w2c of every frame
    if i != 0:                                   # session 0 was rerendered by the test above
        np.testing.assert_allclose(torch.stack(s.all_poses).cpu().numpy(), torch.stack(a.all_poses).cpu().numpy(),
                                   atol=3e-2)
        for o, ao in zip(outs, aouts):
            assert o[0].shape == ao[0].shape and o[1].shape == ao[1].shape and o[6].tolist() == ao[6].tolist()
            np.testing.assert_allclose(float(o[4]), float(ao[4]), rtol=3e-2)
        p, q = str(tmp_path / "s.npz"), str(tmp_path / "a.npz")
        s.write_all_poses(p, filtering_mode="laplacian-conf")
        a.write_all_poses(q, filtering_mode="laplacian-conf")
        zs, za = np.load(p, allow_pickle=True), np.load(q, allow_pickle=True)
        np.testing.assert_allclose(zs["poses"], za["poses"], atol=3e-2)
        assert np.array_equal(zs["timestamps"], za["timestamps"])
        np.testing.assert_allclose(zs["confs"], za["confs"], rtol=1e-2)


def test_saved_session_memory_continues_like_the_live_memory(three, chkpt):
    """Session 1's memory, saved and loaded into SLAM_MUSt3R, continues as the same memory built by SLAM_MUSt3R alone."""
    d = three["dir"]
    p = str(d / "s1.pkl")
    three["ss"][1].save_memory(p)
    a, _ = _alone(chkpt, three["seqs"][1])
    q = str(d / "a1.pkl")
    a.save_memory(q)
    more = mk.frames(5, seed=13)
    b1 = slam.SLAM_MUSt3R(chkpt, device="cuda:0", load_memory=p, **E2E)
    b2 = slam.SLAM_MUSt3R(chkpt, device="cuda:0", load_memory=q, **E2E)
    assert b1.memory[0][0].shape == b2.memory[0][0].shape and b1.memory[2:] == b2.memory[2:]
    for k, im in enumerate(more):
        o1, o2 = b1(im, 100 + k, 0), b2(im, 100 + k, 0)
        assert o1[-1] == o2[-1]
        assert rel(torch.as_tensor(o1[0]), torch.as_tensor(o2[0])) < 2e-2
    assert b1.keyframes == b2.keyframes


def test_step_without_keyframe_syncs_only_at_the_shared_wait(chkpt, monkeypatch, g):
    frames = mk.frames()
    ss = SLAMSessions(chkpt, 2, device="cuda:0", **E2E)
    _stepped(ss, [frames[:4], frames[:4]])
    waits = []
    dec, wait = SLAMSessions._decode, slam._wait_host_copies

    def decode_then_strict(self, *a, **k):
        out = dec(self, *a, **k)
        torch.cuda.set_sync_debug_mode("error")
        return out

    def named_wait():
        torch.cuda.set_sync_debug_mode(0)
        waits.append(1)
        wait()
        torch.cuda.set_sync_debug_mode("error")

    monkeypatch.setattr(SLAMSessions, "_decode", decode_then_strict)
    monkeypatch.setattr(slam, "_wait_host_copies", named_wait)
    try:
        out = ss.step({0: (frames[4], 4, 0), 1: (frames[4], 4, 0)})
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not out[0][-1] and not out[1][-1] and not g["e2e_keyframe"][5]
    assert waits == [1]


# ------------------------------------------------------------------------------------------------ command line
def test_cli_matches_the_single_session_command(chkpt, tmp_path):
    d = str(tmp_path)
    mkc.write_folders(os.path.join(d, "frames"))
    folders = [os.path.join(d, "frames", n) for n in ("seq", "cam0", "cam1")]
    common = ["--chkpt", chkpt, "--device", "cuda:0", "--image_string", mkc.IMAGE_STRING, "--res", "224"]

    def sh(mod, argv):
        r = subprocess.run([sys.executable, "-m", mod] + argv, cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        return r.stdout

    out = sh("must3r_b200.slam_sessions", common + ["--sessions"] + folders + ["--output", os.path.join(d, "multi")])
    kf_multi = [ast.literal_eval(x.split("keyframes: ")[1]) for x in out.splitlines() if x.startswith("session ")]
    for i, f in enumerate(folders):
        one = sh("must3r_b200.slam", common + ["--input", f, "--output", os.path.join(d, f"one{i}")])
        kf_one = ast.literal_eval([x for x in one.splitlines() if " keyframes: [" in x][-1].split("keyframes: ")[1])
        assert kf_multi[i] == kf_one, i
        zm = np.load(os.path.join(d, "multi", f"session_{i}", "all_poses.npz"), allow_pickle=True)
        zo = np.load(os.path.join(d, f"one{i}", "all_poses.npz"), allow_pickle=True)
        assert np.array_equal(zm["timestamps"], zo["timestamps"])
        assert np.array_equal(zm["imgHWs"], zo["imgHWs"])
        np.testing.assert_allclose(zm["poses"], zo["poses"], atol=3e-2)
        np.testing.assert_allclose(zm["confs"], zo["confs"], rtol=1e-2)
        assert os.path.exists(os.path.join(d, "multi", f"session_{i}", "memory.pkl"))
