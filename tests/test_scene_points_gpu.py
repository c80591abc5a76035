"""m3r_scene_points (csrc/scene.cu, ops.scene_points) against torch boolean masking: points and colours bitwise, in
numpy's order (view after view, raster order), for every threshold of one launch.  Outputs go into sentinel-filled
buffers; nothing past the points may be written."""
import numpy as np
import pytest
import torch

from must3r_b200 import ops

pytestmark = pytest.mark.gpu
SENTINEL = -12345.0


def _views(shapes, seed=0, conf_fn=None):
    gen = torch.Generator().manual_seed(seed)
    pts, conf, imgs, c2w = [], [], [], []
    for i, (H, W) in enumerate(shapes):
        pts.append((torch.randn(H, W, 3, generator=gen) * 3).cuda())
        c = 1 + 4 * torch.rand(H, W, generator=gen)
        if conf_fn is not None:
            c = conf_fn(i, c)
        conf.append(c.cuda())
        imgs.append((torch.rand(3, H, W, generator=gen) * 2.4 - 1.2).cuda())      # ImgNorm range and beyond: clipping
        ang = 0.3 * i
        m = torch.eye(4)
        m[:3, :3] = torch.tensor([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]])
        m[:3, 3] = torch.randn(3, generator=gen)
        c2w.append(m.cuda())
    return pts, conf, imgs, c2w


def _want(pts, conf, imgs, thr, c2w=None):
    outs = []
    for t in thr:
        p, c = [], []
        for v in range(len(conf)):
            m = conf[v] >= t
            q = pts[v]
            if c2w is not None:
                q = q.double() @ c2w[v][:3, :3].double().T + c2w[v][:3, 3].double()
            p.append(q[m])
            c.append(imgs[v].permute(1, 2, 0).mul(0.5).add(0.5).clamp(0, 1)[m])
        outs.append((torch.cat(p), torch.cat(c)))
    return outs


def _run(pts, conf, imgs, thr, c2w=None, extra=1000):
    cap = sum(int(c.numel()) for c in conf) * len(thr) + extra
    pb = torch.full((cap, 3), SENTINEL, device="cuda")
    cb = torch.full((cap, 3), SENTINEL, device="cuda")
    p, c, counts = ops.scene_points(pts, conf, imgs, thr, c2w=c2w, out=(pb, cb))
    n = sum(counts)
    assert p.shape[0] == n and (n == 0 or p.data_ptr() == pb.data_ptr())    # an empty tensor has no data pointer
    assert bool((pb[n:] == SENTINEL).all()) and bool((cb[n:] == SENTINEL).all()), "written past the point cloud"
    return p, c, counts


def _check(pts, conf, imgs, thr, c2w=None):
    p, c, counts = _run(pts, conf, imgs, thr, c2w)
    want = _want(pts, conf, imgs, thr, c2w)
    off = 0
    for t, (wp, wc) in enumerate(want):
        assert counts[t] == wp.shape[0], (t, counts[t], wp.shape[0])
        gp, gc = p[off:off + counts[t]], c[off:off + counts[t]]
        assert torch.equal(gc, wc), t
        if c2w is None:
            assert torch.equal(gp, wp), t
        else:
            # fp32 R x + t with two fmas and an add against a float64 evaluation: each coordinate within 4 ulp of the
            # terms' magnitude, |R||x| + |t| (< 1e-6 relative to it)
            mag = pts_mag(wp, c2w)
            assert bool(((gp.double() - wp).abs() <= 4 * 2.0 ** -23 * mag).all()), t
        off += counts[t]
    return counts


def pts_mag(wp, c2w):
    big = max(float(m[:3, :3].abs().sum(1).max()) for m in c2w) + 1
    return (wp.abs().max(dim=1, keepdim=True).values + max(float(m[:3, 3].abs().max()) for m in c2w)) * big


@pytest.mark.parametrize("T", [1, 8])
def test_one_view(T):
    pts, conf, imgs, _ = _views([(384, 512)])
    _check(pts, conf, imgs, np.linspace(1.2, 4.8, T).tolist())


@pytest.mark.parametrize("T", [1, 8])
def test_200_mixed_views(T):
    shapes = [(384, 512) if i % 3 else (512, 384) for i in range(200)]
    pts, conf, imgs, _ = _views(shapes, seed=1)
    counts = _check(pts, conf, imgs, [6.0, 5.0, 4.0, 3.0, 2.5, 2.0, 1.5, 1.05][:T])
    assert counts[0] == sum(int((c >= 6.0).sum()) for c in conf)


def test_square_224_and_ragged_sizes():
    pts, conf, imgs, _ = _views([(224, 224), (37, 53), (1, 1), (16, 1025), (224, 224)], seed=2)
    _check(pts, conf, imgs, [1.5, 3.0, 4.5])


def test_thresholds_tied_to_conf_values():
    pts, conf, imgs, _ = _views([(288, 384), (384, 288)], seed=3)
    vals = torch.cat([c.reshape(-1) for c in conf])
    thr = [float(vals[k]) for k in (0, 1000, 77777, vals.numel() - 1)]
    conf[1].view(-1)[::7] = thr[1]                  # many exact ties
    counts = _check(pts, conf, imgs, thr)
    assert counts[1] >= conf[1].numel() // 7      # every tie is kept (>=)


def test_nan_and_inf_conf():
    def poison(i, c):
        c.view(-1)[::5] = float("nan")
        c.view(-1)[1::11] = float("inf")
        c.view(-1)[2::13] = -float("inf")
        return c
    pts, conf, imgs, _ = _views([(224, 224), (384, 512)], seed=4, conf_fn=poison)
    counts = _check(pts, conf, imgs, [1.05, 3.0, float("inf"), -float("inf")])
    nan = sum(int(torch.isnan(c).sum()) for c in conf)
    assert counts[3] == sum(int(c.numel()) for c in conf) - nan      # -inf keeps everything but NaN


def test_view_with_no_selected_point():
    def low(i, c):
        return torch.full_like(c, 1.01) if i == 1 else c
    pts, conf, imgs, _ = _views([(224, 224), (384, 512), (224, 224)], seed=5, conf_fn=low)
    _check(pts, conf, imgs, [1.5, 2.0])
    _, _, counts = _run(pts, conf, imgs, [100.0])
    assert counts == [0]


def test_local_pointmaps_transform():
    pts, conf, imgs, c2w = _views([(384, 512), (512, 384), (224, 224)], seed=6)
    _check(pts, conf, imgs, [1.05, 2.5, 4.0], c2w=c2w)


def test_argument_errors():
    pts, conf, imgs, _ = _views([(32, 32)])
    with pytest.raises(ValueError):
        ops.scene_points(pts, conf, imgs, [1.0] * 9)
    with pytest.raises(ValueError):
        ops.scene_points(pts, conf, imgs, [])
    with pytest.raises(ValueError):
        ops.scene_points(pts, conf, [imgs[0].half()], [1.0])
    with pytest.raises(ValueError):
        ops.scene_points(pts, conf, imgs, [1.0], out=(torch.empty(1, 3, device="cuda"), torch.empty(1, 3, device="cuda")))
