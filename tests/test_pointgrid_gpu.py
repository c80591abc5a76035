"""The grid index of the keyframe point map (must3r_b200/engine/keyframes.py PointGrid, csrc/pointgrid.cu) against the
brute-force scan `nn_min_dist`, bucket by bucket: the index must give bitwise the same distances."""
import os
import pickle
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from must3r_b200 import ops  # noqa: E402
from must3r_b200.engine import keyframes as kf  # noqa: E402
import test_pointgrid_cpu as model  # noqa: E402

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def room(n, seed, size=(4.0, 3.0, 2.5)):
    """Surface points of a room-sized box."""
    g = _gen(seed)
    s = torch.tensor(size)
    p = torch.rand(n, 3, generator=g) * s
    ax = torch.randint(0, 3, (n,), generator=g)
    wall = torch.where(torch.rand(n, generator=g) < 0.5, torch.zeros(n), s[ax])
    p[torch.arange(n), ax] = wall
    return p


def brute(pts, pb, q, qb, nb):
    out = torch.empty(q.shape[0], dtype=torch.float32, device=q.device)
    for b in range(nb):
        sel = qb == b
        if sel.any():
            out[sel] = kf.nn_min_dist(q[sel], pts[pb == b])
    return out


def check(pts, q, nb=1, seed=0, grid=None):
    g = _gen(seed)
    pb = torch.randint(0, nb, (pts.shape[0],), generator=g, dtype=torch.int32)
    qb = torch.randint(0, nb, (q.shape[0],), generator=g, dtype=torch.int32)
    pts, q, pb, qb = pts.float().cuda(), q.float().cuda(), pb.cuda(), qb.cuda()
    grid = grid or kf.PointGrid(nb)
    grid.add(pts, pb)
    got = grid.query(q, qb)
    want = brute(pts, pb, q, qb, nb)
    bad = (got.view(torch.int32) != want.view(torch.int32)).nonzero()
    assert bad.numel() == 0, (bad[:5].tolist(), got[bad[:5, 0]].tolist(), want[bad[:5, 0]].tolist())
    return grid


@pytest.mark.parametrize("nb", [1, 8, 32])
def test_uniform_and_surface_maps(nb):
    g = _gen(1)
    check(torch.rand(20000, 3, generator=g) * 10 - 5, torch.rand(5000, 3, generator=g) * 12 - 6, nb)
    walls = room(60000, 2)
    near = room(8000, 3) + torch.randn(8000, 3, generator=g) * 0.02
    far = torch.rand(500, 3, generator=g) * 200 - 100        # far from the map: found at coarse block levels
    check(walls, torch.cat([near, far]), nb, seed=1)


def test_clusters_duplicates_and_overflow():
    g = _gen(4)
    centres = torch.randn(20, 3, generator=g) * 3
    clusters = (centres[torch.randint(0, 20, (30000,), generator=g)] + torch.randn(30000, 3, generator=g) * 0.01)
    dup = clusters[:5000].clone()
    odd = torch.tensor([[1e9, 0, 0], [0, -3e8, 2], [1e38, 1e38, 0], [float("nan"), 0, 0], [float("inf"), 1, 1],
                        [0, -float("inf"), 0], [-2e4, 1.0, 1.0]])
    pts = torch.cat([clusters, dup, odd])
    q = torch.cat([clusters[::13] + torch.randn(2308, 3, generator=g) * 0.005, odd, odd + 1.0,
                   torch.tensor([[float("nan"), 1, 1], [5e5, 5e5, 5e5]]), torch.rand(300, 3, generator=g) * 1e7])
    check(pts, q, 1)
    check(pts, q, 4, seed=5)
    check(odd, q, 2, seed=6)                                 # a map of nothing but overflow points


def test_cell_faces_and_single_point():
    ax = torch.arange(-6, 7, dtype=torch.float32) * 0.125
    lattice = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).reshape(-1, 3)
    q = torch.cat([lattice + 0.0625, lattice, lattice + torch.tensor([0.125, 0, 0])])
    check(torch.cat([lattice, lattice]), q, 3)
    check(torch.tensor([[0.3, -0.2, 1.0]]), torch.tensor([[0.3, -0.2, 1.0], [5.0, 5.0, 5.0], [-1e6, 0, 0]]), 1)


def test_keys_match_the_model():
    g = _gen(9)
    pts = torch.cat([torch.randn(5000, 3, generator=g) * 3, torch.tensor([[1e9, 0, 0], [float("nan"), 0, 0], [0, float("inf"), 0],
                                                                          [-1.0, -0.5, 0.25], [0.999, 1.0, 1.001]])])
    b = torch.randint(0, 511, (pts.shape[0],), generator=g, dtype=torch.int32)
    for h in (0.01, 0.25, 3.0):
        inv = float(model.F(1.0 / float(model.F(h))))
        got = ops.pointgrid_keys(pts.cuda(), b.cuda(), inv).cpu().numpy()
        assert (got == model.keys(pts.numpy(), b.numpy().astype("int64"), inv)).all(), h


def test_empty_map_and_empty_buckets():
    q = torch.randn(1000, 3, generator=_gen(7)).cuda()
    assert torch.isinf(kf.PointGrid(4).query(q, torch.zeros(1000, dtype=torch.int32, device="cuda"))).all()
    grid = kf.PointGrid(4)
    grid.add(room(5000, 8).cuda(), torch.zeros(5000, dtype=torch.int32, device="cuda"))
    qb = torch.arange(1000, device="cuda", dtype=torch.int32) % 4
    d = grid.query(q, qb)
    assert torch.isinf(d[qb != 0]).all() and torch.isfinite(d[qb == 0]).all()
    assert torch.isinf(kf.DeviceNN().query(q)).all()


def test_incremental_adds_match_one_build():
    frames = [room(12000, 20 + i) + 0.3 * i for i in range(5)]
    cam = torch.tensor([1.0, 1.5, 1.2]).cuda()
    q = room(6000, 30).cuda() + 0.01
    for method in ("kdtree-scipy", "quadrant_x2-kdtree-scipy", "quadrant_x4-kdtree-scipy"):
        inc, one = kf.get_searcher(method), kf.get_searcher(method)
        for f in frames:
            inc.add_pts(f.cuda(), cam_center=cam)
            inc.query(q, cam_center=cam)                     # rebuilt after every add
        one.add_pts(torch.cat(frames).cuda(), cam_center=cam)
        a, b = inc.query(q, cam_center=cam), one.query(q, cam_center=cam)
        assert torch.equal(a, b), method
        if "quadrant" in method:                             # the searcher's quadrants are the buckets
            ids = one._ids(q, cam).int()
            pid = one._ids(torch.cat(frames).cuda(), cam).int()
            assert torch.equal(a, brute(torch.cat(frames).cuda(), pid, q, ids, one.grid.nb))
        else:
            assert torch.equal(a, kf.nn_min_dist(q, torch.cat(frames).cuda()))


def test_pickle_round_trip():
    cam = torch.tensor([0.5, 0.5, 0.5]).cuda()
    s = kf.get_searcher("quadrant_x2-kdtree-scipy")
    s.add_pts(room(20000, 40).cuda(), cam_center=cam)
    q = room(3000, 41).cuda() + 0.02
    want = s.query(q, cam_center=cam)
    blob = pickle.dumps(s)
    t = pickle.loads(blob)
    assert t.grid._grid is None and not t.grid.pts.is_cuda
    assert torch.equal(t.query(q, cam_center=cam), want)
    t.add_pts(room(100, 42).cuda(), cam_center=cam)          # keeps growing after a load
    assert len(t.grid) == 20100


def test_non_default_stream():
    pts, q = room(40000, 50).cuda(), (room(10000, 51) + 0.03).cuda()
    want = kf.nn_min_dist(q, pts)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        grid = kf.PointGrid(1)
        grid.add(pts)
        got = grid.query(q)
    s.synchronize()
    assert torch.equal(got, want)


def test_device_nn_selects_by_map_size():
    q = (room(4000, 60) + 0.02).cuda()
    nn = kf.DeviceNN()
    for i in range(4):                                       # crosses BRUTE_MAX_POINTS on the way
        nn.add_pts(room(kf.DeviceNN.BRUTE_MAX_POINTS // 2 + 1, 61 + i).cuda())
        assert nn.uses_brute_force() == (len(nn.grid) <= kf.DeviceNN.BRUTE_MAX_POINTS)
        assert torch.equal(nn.query(q), kf.nn_min_dist(q, nn.grid.pts))
        assert torch.equal(nn.query(q), nn.grid.query(q))
    assert not nn.uses_brute_force()
    small = pickle.loads(pickle.dumps(kf.DeviceNN()))
    small.add_pts(room(100, 70).cuda())
    small = pickle.loads(pickle.dumps(small))
    assert small.uses_brute_force() and torch.equal(small.query(q), kf.nn_min_dist(q, room(100, 70).cuda()))


def test_bucket_ids_are_checked_before_narrowing():
    grid = kf.PointGrid(8)
    pts = room(100, 80).cuda()
    bad = torch.zeros(100, dtype=torch.int64, device="cuda")
    bad[3] = -(1 << 40)                                      # wraps to 0 as int32
    with pytest.raises(ValueError):
        grid.add(pts, bad)
    with pytest.raises(ValueError):
        grid.add(pts, bad.abs())
    grid.add(pts, torch.zeros(100, dtype=torch.int64, device="cuda"))
    qb = torch.tensor([0, -(1 << 40), 1 << 33, 8, 7], device="cuda")
    d = grid.query(pts[:5], qb)
    assert d[0] == 0 and torch.isnan(d[1:4]).all() and torch.isinf(d[4])
