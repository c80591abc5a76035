"""NumPy model of the grid index of must3r_b200/csrc/pointgrid.cu (key packing, cell coordinates, per-cell lower bound,
ring-stop rule over levels of blocks, overflow lists), checked against its own brute-force scan (bitwise) and against
scipy's KDTree on adversarial point sets.  The model uses the kernel's constants and float32 arithmetic; the GPU tests
(test_pointgrid_gpu.py) hold the kernel itself to the brute-force scan."""
import numpy as np
import pytest
from scipy.spatial import KDTree

F = np.float32
AXIS_BITS = 18
BIAS = 1 << (AXIS_BITS - 1)
OVF = (1 << (3 * AXIS_BITS)) - 1
RING = 2
SLACK = F(0.0625)
SHRINK = F(0.99998)


def cell_coords(p, inv_h):
    with np.errstate(over="ignore", invalid="ignore"):
        v = (p.astype(F) * F(inv_h)).astype(F)
        ok = np.all((v >= -BIAS) & (v < BIAS - 1), axis=-1)
    c = np.floor(np.where(ok[..., None], v, 0)).astype(np.int64)
    return c, ok


def morton(u):
    """Interleave the bits of biased coordinates u [..., 3] (x highest): bit i of x, y, z -> bits 3i+2, 3i+1, 3i."""
    u = np.asarray(u, dtype=np.int64)
    k = np.zeros(u.shape[:-1], dtype=np.int64)
    for i in range(AXIS_BITS):
        for a in range(3):
            k |= ((u[..., a] >> i) & 1) << (3 * i + 2 - a)
    return k


def unmorton(k):
    u = np.zeros(np.shape(k) + (3,), dtype=np.int64)
    for i in range(AXIS_BITS):
        for a in range(3):
            u[..., a] |= ((k >> (3 * i + 2 - a)) & 1) << i
    return u


def pack(b, c):
    return (np.asarray(b, dtype=np.int64) << (3 * AXIS_BITS)) | morton(c + BIAS)


def keys(p, b, inv_h):
    c, ok = cell_coords(p, inv_h)
    return np.where(ok, pack(b, c), (np.asarray(b, dtype=np.int64) << (3 * AXIS_BITS)) | OVF)


def unpack(k):
    return unmorton(k & OVF) - BIAS


def sqdist(q, pts):
    with np.errstate(over="ignore", invalid="ignore"):
        d = (q[None, :] - pts).astype(F)
        return (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(F)


def fmin(best, d2):
    d2 = d2[~np.isnan(d2)]                                   # fminf drops NaN
    return F(min(best, d2.min())) if d2.size else best


def box_lb2(q, lo, hi, h):
    """Lower bound of the squared distance from q to the cells [lo, hi) per axis (unbiased cell coordinates)."""
    with np.errstate(over="ignore", invalid="ignore"):
        a = ((lo.astype(F) - SLACK) * F(h)).astype(F)
        b = ((hi.astype(F) + SLACK) * F(h)).astype(F)
        g = np.maximum(F(0), np.maximum(a - q[None, :], q[None, :] - b)).astype(F)
        return ((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1] + g[:, 2] * g[:, 2]) * SHRINK).astype(F)


def lb2(q, cells, h):
    return box_lb2(q, cells, cells + 1, h)


def ring(r):
    o = np.stack(np.meshgrid(*[np.arange(-r, r + 1)] * 3, indexing="ij"), -1).reshape(-1, 3)
    return o[np.abs(o).max(1) == r]


RINGS = [ring(r) for r in range(RING + 1)]


class GridModel:
    def __init__(self, pts, buckets, nb, h):
        self.h, self.inv = F(h), F(1.0 / np.float64(F(h)))
        k = keys(pts, buckets, self.inv)
        order = np.argsort(k, kind="stable")
        self.pts, sk = pts[order].astype(F), k[order]
        self.cell_keys, start = np.unique(sk, return_index=True)
        self.cell_off = np.append(start, len(sk))
        self.bucket_cells = np.append(np.searchsorted(self.cell_keys, np.arange(nb, dtype=np.int64) << (3 * AXIS_BITS)),
                                      len(self.cell_keys))
        self.levels = []                                     # deepest level each grid query reached

    def _scan(self, q, c, best):
        return fmin(best, sqdist(q, self.pts[self.cell_off[c]:self.cell_off[c + 1]]))

    def _visit(self, q, c0, c1, best):
        """Cells c0..c1 in order: skip those whose lower bound is not below the best so far."""
        if c1 <= c0:
            return best
        lbs = lb2(q, unpack(self.cell_keys[c0:c1]), self.h)
        for j in np.nonzero(lbs < best)[0]:
            if lbs[j] < best:
                best = self._scan(q, c0 + j, best)
        return best

    def query(self, q, b):
        q = q.astype(F)
        best = F(np.inf)
        base = b << (3 * AXIS_BITS)
        lo, hi = self.bucket_cells[b], self.bucket_cells[b + 1]
        if lo < hi and self.cell_keys[hi - 1] == base | OVF:
            hi -= 1
            best = self._scan(q, hi, best)
        if lo < hi and np.isfinite(q).all():
            c, ok = cell_coords(q, self.inv)
            if not ok:
                return F(np.sqrt(self._visit(q, lo, hi, best)))
            done = False
            for L in range(AXIS_BITS + 1):
                n = 1 << (AXIS_BITS - L)
                for r in range(RING + 1):
                    blk = ((c + BIAS) >> L)[None, :] + RINGS[r]
                    blk = blk[np.all((blk >= 0) & (blk < n), axis=1)]
                    if L > 0:                                # children all visited by the previous level's rings
                        prev = (c + BIAS) >> (L - 1)
                        blk = blk[~np.all((2 * blk >= prev - RING) & (2 * blk + 1 <= prev + RING), axis=1)]
                    lbs = box_lb2(q, (blk << L) - BIAS, ((blk + 1) << L) - BIAS, self.h)
                    for j in np.nonzero(lbs < best)[0]:
                        if lbs[j] < best:
                            first = base | (morton(blk[j]) << (3 * L))
                            c0 = lo + np.searchsorted(self.cell_keys[lo:hi], first)
                            c1 = lo + np.searchsorted(self.cell_keys[lo:hi], first + (1 << (3 * L)))
                            best = self._visit(q, c0, c1, best)
                    bound = F(F((r << L) - 0.125) * self.h)
                    done = r >= 1 and best < F(bound * bound * SHRINK)
                    if done:
                        break
                if done:
                    break
            self.levels.append(L)
        return F(np.sqrt(best))


def brute(q, pts):
    return F(np.sqrt(fmin(F(np.inf), sqdist(q.astype(F), pts.astype(F))))) if len(pts) else F(np.inf)


def check(pts, queries, h, nb=1, seed=0):
    rng = np.random.default_rng(seed)
    pts, queries = pts.astype(F), queries.astype(F)
    pb = rng.integers(0, nb, len(pts)).astype(np.int64)
    qb = rng.integers(0, nb, len(queries)).astype(np.int64)
    m = GridModel(pts, pb, nb, h)
    got = np.array([m.query(q, b) for q, b in zip(queries, qb)], dtype=F)
    want = np.array([brute(q, pts[pb == b]) for q, b in zip(queries, qb)], dtype=F)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), np.nonzero(got.view(np.int32) != want.view(np.int32))
    for b in range(nb):                                      # the brute force itself against scipy, on the finite points
        fin = pts[(pb == b) & np.isfinite(pts).all(1)].astype(np.float64)
        sel = (qb == b) & np.isfinite(queries).all(1) & np.isfinite(want)
        if sel.any() and len(fin):
            ref, _ = KDTree(fin).query(queries[sel].astype(np.float64), k=1)
            close = ref < 1e18
            np.testing.assert_allclose(want[sel][close], ref[close], rtol=2e-6, atol=1e-6 * float(np.abs(fin).max()) + 1e-30)
    return m


def surface(n, seed):
    """Points on the walls of a 4 x 3 x 2.5 box."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(0, 1, (n, 3)) * np.array([4.0, 3.0, 2.5])
    ax = rng.integers(0, 3, n)
    p[np.arange(n), ax] = np.where(rng.random(n) < 0.5, 0.0, np.array([4.0, 3.0, 2.5])[ax])
    return p


def test_key_packing():
    c = np.array([[-BIAS, -BIAS, -BIAS], [BIAS - 2, BIAS - 2, BIAS - 2], [0, -1, 5], [3, 0, -7]])
    for b in (0, 1, 511):
        k = pack(b, c)
        assert (k >= 0).all() and (k >> (3 * AXIS_BITS) == b).all()
        assert np.array_equal(unpack(k), c)
        assert (k < (b << (3 * AXIS_BITS)) | OVF).all()                  # the overflow list sorts after every cell
    assert ((511 << (3 * AXIS_BITS)) | OVF) < 2 ** 63
    assert pack(1, c).min() > ((0 << (3 * AXIS_BITS)) | OVF)              # buckets never interleave
    u = np.random.default_rng(0).integers(0, (1 << AXIS_BITS) - 1, (500, 3))
    for L in (1, 4, 9):                       # an aligned block of 2^L cells per side is one contiguous key range
        k = morton(u)
        assert np.array_equal(k >> (3 * L), morton(u >> L))
    _, ok = cell_coords(np.array([[0, 0, BIAS - 1.0], [np.nan, 0, 0], [np.inf, 0, 0], [0, -BIAS, 0], [0, 0, BIAS - 1.5]]), 1.0)
    assert ok.tolist() == [False, False, False, True, True]


def test_lower_bounds_hold_on_cell_faces():
    """Every point's rounded squared distance is above its cell's lower bound and above the stop bound of every ring
    (of every block level) that does not contain its cell - on points and queries placed exactly on cell faces, far out
    and near the key range's edge."""
    rng = np.random.default_rng(1)
    for h in (F(0.1), F(0.37), F(1.0), F(3.0e4)):
        inv = F(1.0 / np.float64(h))
        base = np.concatenate([rng.integers(-20, 20, (300, 3)) * h, rng.integers(-BIAS + 2, BIAS - 3, (100, 3)) * h])
        jitter = np.concatenate([np.zeros((200, 3)), rng.uniform(-1, 1, (200, 3)) * h * 1e-6])
        pts = (base + jitter).astype(F)
        c, ok = cell_coords(pts, inv)
        for q in pts[rng.choice(len(pts), 40)]:
            cq, okq = cell_coords(q, inv)
            d2 = sqdist(q, pts[ok])
            lb = lb2(q, c[ok], h)
            assert ((lb < d2) | (lb == 0)).all()             # a zero bound only prunes once the best is already 0
            if okq:
                for L in (0, 1, 3, 8):
                    cheb = np.abs(((c[ok] + BIAS) >> L) - ((cq + BIAS) >> L)[None]).max(1)
                    for r in range(1, RING + 1):
                        bound = F(F((r << L) - 0.125) * h)
                        assert (d2[cheb > r] > F(bound * bound * SHRINK)).all()


@pytest.mark.parametrize("nb", [1, 8])
def test_model_matches_brute_force_on_surfaces(nb):
    pts = surface(3000, 2)
    q = np.concatenate([surface(150, 3) + np.random.default_rng(4).normal(0, 0.02, (150, 3)),
                        np.random.default_rng(5).uniform(-2, 6, (50, 3))])
    for h in (0.02, 0.1, 0.5):                               # dense cells, ~4 per cell, and queries that need the fallback
        check(pts, q, h, nb)


def test_faces_duplicates_and_single_point():
    h = F(0.25)
    g = np.stack(np.meshgrid(*[np.arange(-3, 4) * 0.25] * 3, indexing="ij"), -1).reshape(-1, 3)
    pts = np.concatenate([g, g, g[:50]])                     # every point on a cell corner, each at least twice
    q = np.concatenate([g[::7] + 0.125, g[::5], g[::3] + np.array([0.25, 0, 0])])
    check(pts, q, h, nb=3)
    check(np.array([[0.3, -0.2, 1.0]]), np.array([[0.3, -0.2, 1.0], [5.0, 5.0, 5.0], [-1e6, 0, 0]]), 0.1)


def test_outliers_huge_and_non_finite():
    rng = np.random.default_rng(7)
    pts = np.concatenate([surface(800, 8), [[1e9, 0, 0], [0, -3e8, 2], [1e38, 1e38, 0], [np.nan, 0, 0], [np.inf, 1, 1],
                                            [0, -np.inf, 0], [-2e4, 1.0, 1.0]]])
    q = np.concatenate([surface(60, 9), [[1e9, 1, 0], [0, -3e8, 2.5], [1e38, 1e38, 1e30], [np.nan, 0, 0], [np.inf, 0, 0],
                                         [-2e4, 1, 1.5], [5e5, 5e5, 5e5], [3000, 0, 0], [-500, 200, 100]],
                        rng.uniform(-1e7, 1e7, (10, 3))])
    m = check(pts, q, 0.05, nb=1)
    assert (m.cell_keys[-1] & OVF) == OVF                    # the far points went to the overflow list
    assert max(m.levels) >= 10                               # far queries climbed to coarse blocks
    check(pts, q, 0.05, nb=4, seed=3)


def test_empty_buckets_and_empty_map():
    pts = surface(200, 10)
    m = GridModel(pts.astype(F), np.zeros(200, dtype=np.int64), 4, 0.1)
    assert np.isinf(m.query(np.array([1.0, 1.0, 1.0]), 2))
    assert m.query(np.array([1.0, 1.0, 1.0]), 0) == brute(np.array([1.0, 1.0, 1.0]), pts)
    e = GridModel(np.zeros((0, 3), dtype=F), np.zeros(0, dtype=np.int64), 1, 0.1)
    assert np.isinf(e.query(np.array([0.0, 0.0, 0.0]), 0))
