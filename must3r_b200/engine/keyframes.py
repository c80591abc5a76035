"""Keyframe selection of the SLAM front end on the GPU (SURVEY.md §8f rank 3): the overlap score of
must3r/slam/model.py:62-91 (`get_overlap_score`), the decision of :123-128 (`choose_keyframe_from_overlap`) and the
nearest-neighbour searchers of must3r/slam/nns.py (`get_searcher`, `KDTree_scipy`, `QuandrantSearcher`), with the same names,
arguments and results - but the point database stays on the device and the per-frame query runs on an exact grid index
(`PointGrid`, `m3r_pointgrid_query`) instead of a scipy KD-tree on the CPU (`.cpu().numpy()` of every prediction +
`KDTree.query`).  The brute-force scan `nn_min_dist` (`m3r_nn_min_dist`) stays as the reference the index is tested against.
Results are torch tensors on the query's device; the score itself is a Python float (the caller branches on it).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .. import _lib, ops


def nn_min_dist(queries: torch.Tensor, db: torch.Tensor) -> torch.Tensor:
    """[Q,3], [P,3] fp32 CUDA -> [Q] distance to the nearest database point (inf if P == 0)."""
    if not queries.is_cuda:
        raise RuntimeError("must3r_b200 keyframe search needs CUDA tensors (no CPU fallback)")
    q = queries.reshape(-1, 3).float().contiguous()
    d = db.reshape(-1, 3).float().contiguous()
    out = torch.empty((q.shape[0],), dtype=torch.float32, device=q.device)
    with torch.cuda.device(q.device):
        _lib.check(_lib.lib().m3r_nn_min_dist(C.c_void_p(q.data_ptr()), q.shape[0], C.c_void_p(d.data_ptr()) if d.numel() else None,
                                              d.shape[0], C.c_void_p(out.data_ptr()),
                                              C.c_void_p(torch.cuda.current_stream(q.device).cuda_stream)), "nn_min_dist")
    return out


def get_quadrant_id(rays: torch.Tensor, quadrant_divider: int = 4, eps: float = 1e-5) -> torch.Tensor:
    """must3r/slam/tools.py:9-31: viewing-direction quadrant of every ray (spherical coordinates, quantised)."""
    rays = rays / rays.norm(dim=-1, keepdim=True).clip(eps)
    thetas = (torch.acos(rays[:, -1]) / math.pi).clip(eps, 1 - eps)
    phis = (torch.atan2(rays[:, 1], rays[:, 0]) / math.pi).clip(-1 + eps, 1 - eps)
    theta_idx = torch.floor(thetas * quadrant_divider).long()
    phis_idx = torch.floor(phis * quadrant_divider).long() + quadrant_divider
    return theta_idx + phis_idx * quadrant_divider


class PointGrid:
    """Exact nearest-neighbour index over a growing point map [P,3] fp32 whose points each carry a bucket id in [0, nb):
    `query` returns, per query point, the distance to the nearest map point of the query's bucket (inf if there is none,
    NaN for a bucket id outside [0, nb), e.g. the quadrant of a NaN point), bitwise equal to `nn_min_dist` over that bucket's points (csrc/pointgrid.cu).  The map stays on the device; the grid
    (points sorted by bucket and cell, plus the table of occupied cells) is rebuilt at the first query after `add`.

    Pickles as CPU tensors of the points and buckets; the grid is rebuilt on the query's device on first use."""

    MAX_BUCKETS = 512
    TARGET = 4.0                 # points per occupied cell the cell size aims at

    def __init__(self, nb=1):
        if not 1 <= nb <= self.MAX_BUCKETS:
            raise ValueError(f"PointGrid: {nb} buckets (1..{self.MAX_BUCKETS})")
        self.nb = nb
        self.pts, self.buckets = None, None
        self._grid = None

    def __len__(self):
        return 0 if self.pts is None else self.pts.shape[0]

    def add(self, pts, buckets=None):
        p = pts.reshape(-1, 3).float()
        if p.shape[0] == 0:
            return
        if buckets is None:
            b = torch.zeros(p.shape[0], dtype=torch.int32, device=p.device)
        else:
            b = buckets.reshape(-1)
            if b.shape[0] != p.shape[0]:
                raise ValueError(f"PointGrid.add: {b.shape[0]} bucket ids for {p.shape[0]} points")
            if int(b.min()) < 0 or int(b.max()) >= self.nb:      # on the caller's ids, before narrowing to int32
                raise ValueError(f"PointGrid.add: bucket ids outside [0, {self.nb})")
            b = b.int()
        if self.pts is not None:
            p, b = torch.cat([self.pts.to(p.device), p]), torch.cat([self.buckets.to(p.device), b])
        self.pts, self.buckets = p.contiguous(), b.contiguous()
        self._grid = None

    def __getstate__(self):
        return {"nb": self.nb, "pts": None if self.pts is None else self.pts.cpu(),
                "buckets": None if self.buckets is None else self.buckets.cpu()}

    def __setstate__(self, state):
        self.nb, self.pts, self.buckets = state["nb"], state["pts"], state["buckets"]
        self._grid = None

    def _initial_cell_size(self, pts):
        """Cell side for ~TARGET points per cell if the points covered the surface of their bounding box."""
        fin = pts[torch.isfinite(pts).all(dim=1)]
        if fin.shape[0] == 0:
            return 1.0
        ext = (fin.amax(dim=0) - fin.amin(dim=0)).double().tolist()
        area = 2.0 * (ext[0] * ext[1] + ext[1] * ext[2] + ext[2] * ext[0])
        if area > 0:
            return math.sqrt(area * self.TARGET / fin.shape[0])
        return max(ext) * self.TARGET / fin.shape[0] if max(ext) > 0 else 1.0

    def _build(self, device):
        pts = self.pts.to(device).contiguous()
        buckets = self.buckets.to(device).contiguous()
        self.pts, self.buckets = pts, buckets
        # The cell size is a deterministic function of the map: start from the bounding-box estimate, then rescale (as for
        # a surface, by the square root) until the occupied cells hold 2..8 points on average, at most twice.
        h = self._initial_cell_size(pts)
        low54 = (1 << 54) - 1
        for it in range(3):
            h32 = float(np.float32(min(max(h, 1e-30), 1e30)))
            inv = float(np.float32(1.0 / h32))
            keys = ops.pointgrid_keys(pts, buckets, inv)
            skeys, perm = torch.sort(keys, stable=True)
            cell_keys, counts = torch.unique_consecutive(skeys, return_counts=True)
            real = (cell_keys & low54) != low54                  # the buckets' overflow lists are not cells
            n_cells = int(real.sum())
            mean = int(counts[real].sum()) / max(n_cells, 1)
            if n_cells == 0 or 2.0 <= mean <= 8.0 or it == 2:
                break
            h = h32 * math.sqrt(self.TARGET / mean)
        first = torch.arange(self.nb, device=device, dtype=torch.int64) << 54
        bucket_cells = torch.cat([torch.searchsorted(cell_keys, first),
                                  torch.tensor([cell_keys.shape[0]], device=device)]).int()
        cell_off = torch.cat([torch.zeros(1, dtype=torch.int64, device=device), counts.cumsum(0)]).int()
        self._grid = (pts[perm].contiguous(), cell_keys, cell_off, bucket_cells, h32, inv)

    def query(self, q, qbuckets=None):
        q = q.reshape(-1, 3).float().contiguous()
        if not q.is_cuda:
            raise RuntimeError("must3r_b200 keyframe search needs CUDA tensors (no CPU fallback)")
        qb = None
        if qbuckets is not None:                                 # an id outside [0, nb) becomes -1: its distance is NaN
            qb = qbuckets.reshape(-1)
            qb = torch.where((qb >= 0) & (qb < self.nb), qb, torch.full_like(qb, -1)).int().contiguous()
        with torch.cuda.device(q.device):
            if self.pts is None:
                return torch.full((q.shape[0],), math.inf, dtype=torch.float32, device=q.device)
            if self._grid is None or self._grid[0].device != q.device:
                self._build(q.device)
            spts, cell_keys, cell_off, bucket_cells, h, inv = self._grid
            return ops.pointgrid_query(q, qb, spts, cell_keys, cell_off, bucket_cells, h, inv)


class DeviceNN:
    """must3r/slam/nns.py:40-62 (`KDTree_scipy`): `add_pts` grows the database, `query` returns nearest distances.
    Both ways of answering give bitwise the same distances; which one runs depends only on the map size: the brute-force
    scan `nn_min_dist` up to BRUTE_MAX_POINTS points, where it is as fast as the grid index (tools/bench_pointgrid.py),
    the index above."""

    BRUTE_MAX_POINTS = 65536

    def __init__(self):
        self.grid = PointGrid(1)

    def add_pts(self, pts, **kw):
        self.grid.add(pts)

    def uses_brute_force(self):
        return len(self.grid) <= self.BRUTE_MAX_POINTS

    def query(self, pts, **kw):
        if self.uses_brute_force() and self.grid.pts is not None:
            if self.grid.pts.device != pts.device:
                self.grid.pts = self.grid.pts.to(pts.device)
            return nn_min_dist(pts, self.grid.pts)
        return self.grid.query(pts)


class QuadrantSearcher:
    """must3r/slam/nns.py:65-95 (`QuandrantSearcher`): one database per viewing-direction quadrant; a query point only
    sees database points observed from a similar direction.  All quadrants share one grid index (the quadrant is the
    point's bucket), so a query is one launch whatever quadrants its points fall in."""

    def __init__(self, method="quadrant_x4-kdtree-scipy"):
        self.quadrant_divider = int(method.split('quadrant_x')[-1].split('-')[0])
        self.grid = PointGrid(2 * self.quadrant_divider ** 2)

    def _ids(self, pts, cam_center):
        return get_quadrant_id(pts.reshape(-1, 3).float() - cam_center.reshape(1, 3).to(pts.device).float(), self.quadrant_divider)

    def add_pts(self, pts, cam_center, **kw):
        pts = pts.reshape(-1, 3)
        self.grid.add(pts, self._ids(pts, cam_center))

    def query(self, pts, cam_center, **kw):
        pts = pts.reshape(-1, 3)
        return self.grid.query(pts, self._ids(pts, cam_center))


QuandrantSearcher = QuadrantSearcher          # the reference's spelling (nns.py:65)


def get_searcher(method, isquadrant=False):
    """must3r/slam/nns.py:9-19"""
    if 'quadrant_x' in method and not isquadrant:
        return QuadrantSearcher(method)
    if "kdtree-scipy" in method:
        return DeviceNN()
    if method == 'none':
        return None
    raise ValueError(f"Unknown searcher method {method}")


def get_overlap_score(res, overlap_tree, cam_center, mode='nn', kf_x_subsamp=None, min_conf_keyframe=1.5, percentile=70,
                      eps=1e-9):
    """must3r/slam/model.py:62-91: how much of the new frame is NOT yet covered by the keyframes' points = the `percentile`
    of the distances from its confident points to their nearest stored neighbour (optionally / depth), or a confidence
    statistic."""
    if mode == 'meanconf':
        return res['conf'].mean()
    if mode == 'medianconf':
        return res['conf'].median()
    if 'nn' not in mode:
        raise ValueError(f"Unknown overlap score method {mode}")
    pts3d = res['pts3d'][0, 0, ::kf_x_subsamp, ::kf_x_subsamp] if kf_x_subsamp else res['pts3d']
    msk = res['conf'][0, 0, ::kf_x_subsamp, ::kf_x_subsamp] if kf_x_subsamp else res['conf']
    msk = msk > min_conf_keyframe
    if int(msk.sum()) == 0:
        return 0.
    dists = overlap_tree.query(pts3d[msk], cam_center=cam_center)
    if 'norm' in mode:
        depths = res['pts3d_local'][0, 0, ::kf_x_subsamp, ::kf_x_subsamp, -1]
        dists = dists / (depths[msk].float() + eps)
    dists = torch.where(torch.isposinf(dists), torch.full_like(dists, torch.finfo(dists.dtype).max), dists)
    return float(torch.quantile(dists.double(), percentile / 100.0, interpolation='linear'))      # np.percentile's default


def choose_keyframe_from_overlap(overlap_score, thr, overlap_mode):
    """must3r/slam/model.py:123-128"""
    return overlap_score > thr if 'nn' in overlap_mode else overlap_score < thr
