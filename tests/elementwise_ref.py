"""Float64 references of the small kernels of csrc/elementwise.cu where the model starts and ends (the RoPE table, the
stand-alone curope RoPE, the postprocess activation) and of the nearest-neighbour scan m3r_nn_min_dist, the element-wise
allowance of each kernel's fp32 arithmetic, check(), and the input generators that the CPU bound test and the GPU
contract test share.  Every reference is computed in float64 on the inputs' device, in chunks where the shapes need it.

Notation as in gemm_ref.py: U = 2^-24 (fp32 unit roundoff; one ulp of x is at most 2U |x|), u = 2^-11 (fp16) or 2^-8
(bf16).  Every allowance counts the rounding of the stored result twice, so a correctly rounded result sits at half of
it.  The build does not use --use_fast_math, so the CUDA math library's documented maximum errors apply (CUDA C++
Programming Guide, single-precision mathematical functions): powf 4 ulp, sinf / cosf 2 ulp, expf 2 ulp, expm1f 1 ulp;
x / y and sqrtf are correctly rounded (0 ulp), and denormals are kept.  The compiler may contract a * b + c into an fma;
each bound below covers both forms.

RoPE table (m3r_rope_table): tab[t][32a + d] = cos(theta), tab[t][32a + 16 + d] = sin(theta), d < 16, a = 0 (y), 1 (x),
theta = p_a f0 / base^(d/16) in exact arithmetic, with f0 and base their fp32 values.  The kernel computes
fl(p) * fl(f0 / powf(base, d / Q)):
  angle   |dtheta| <= c_theta U |theta|, c_theta = 8 (powf, 4 ulp) + 1 (the division) + 1 (the product)
          + ln(base) where d / Q is rounded (Q not a power of two: a relative error U of the exponent e < 1 moves
          base^e by ln(base) e U).  p is exact below 2^24.
  trig    2 ulp of the result: 4U (|ref| + |dtheta|)
  error bound of a table entry   e_tab = |dtheta| + 4U (|ref| + |dtheta|)               (used by the GEMM, see below)
  allowance                       e_tab + 4U (|ref| + |dtheta|)                         (the trig rounding counted twice)
The real-table GEMM check passes the exact float64 table and e_tab to gemm_ref.reference (rope_tab_err), which adds
|u| e_cos + |w| e_sin to its RoPE term.

Stand-alone RoPE (m3r_rope_2d, curope semantics): Q = D / 4, pairs (u, v) = (tok[a 2Q + d], tok[a 2Q + Q + d]) of the
16-bit or fp32 token values, rotated by the same angle with inv_freq = fwd / base^(d/Q):
  u' = u cos - v sin, v' = v cos + u sin    (two fp32 products and an add, or a product and an fma)
  E0 = |u| e_cos + |v| e_sin                                   trig and angle, e_* = e_tab above for this Q
  E1 = E0 + U (|u| (|cos| + e_cos) + |v| (|sin| + e_sin))       the products (or the product inside the fma)
  E  = E1 + U (|u'| + E1)                                      the add
  allowance = E + 2 u_o (|u'| + E) (+ 2^-24 for fp16: the subnormal floor)   gemm_ref.out_bound, u_o = U for fp32 tokens
Negative fwd and negative positions only change signs; the angle term grows with |theta|, up to a few thousand.

Postprocess (m3r_postprocess): for channels 0:3 and 3:6, exact value X = x expm1(d) / max(d, c) with d = |x| (float64),
c = fl(1e-8); conf = 1 + exp(c6).  The kernel computes d^ = sqrtf(x*x + y*y + z*z), f = expm1f(d^) / fmaxf(d^, c), x f:
  d^      the sum of three non-negative squares: 3 roundings, relative 3U; the square root halves it and rounds once:
          |d^ - d| <= Dd = 2.5U d + 2^-74.  2^-74 = sqrt(3 * 2^-150): squares below 2^-126 are subnormal and round with an
          absolute error of up to 2^-150 each.
  expm1   a relative error Dd / d of the argument reaches expm1 amplified by A = d e^d / (e^d - 1) <= 1 + d (this is the
          term CHAIN_TOL_LOCAL of test_model_gpu.py observes), and expm1f adds 1 ulp: 2U.
  divide  by the same d^ (d > c): its relative error Dd / d cancels against the amplified one, leaving (A - 1) Dd / d
          (0 <= A - 1 <= d); by c (d <= c, or d^ on the other side of c): no cancellation, A Dd / d.  The division
          rounds once: U.
  rel     = 2 (A - [d > c (1 + 4U)]) Dd / d + 2U + 2U,   E = 1.0001 rel |X|   (1.0001: second-order terms)
          Here every rounding is counted twice, like the output rounding, and the library's error bound (expm1f, 2U)
          once: d^ carries five roundings that for d > 1 dominate (a faithful computation reaches 0.7 of Dd on random
          points), and at d < 1 three roundings of up to U each meet.  At d < 1 the allowance stays near 6U |X|,
          below 4 ulp.
  allowance = E + 2U (|X| + E) + 2^-149                     the product x f rounds once; 2^-149: a subnormal product
  conf    E = 4U e^c6 (expf, 2 ulp); allowance E + 2U (|1 + e^c6| + E)
Where the reference's own formula in fp32 (oracle postprocess: x / clip(d, 1e-8) * expm1(d)) gives a non-finite value,
the kernel must give the same class: NaN where it is NaN, the same infinity where it is infinite.  That covers a NaN
component (NaN in all three outputs), an inf component (NaN), d above ln(FLT_MAX) (+-inf, NaN where the component is 0)
and c6 = NaN / +inf (NaN / +inf; c6 = -inf gives 1, finite).  A zero vector must give exactly 0 with the input's sign.

Nearest-neighbour scan (m3r_nn_min_dist): exact value D = min_j |q - p_j| over the non-NaN database points (float64).
The kernel rounds each q - p (U relative), squares and sums with dz*dz and two fmas (three roundings of non-negative
partials): every candidate's squared distance is within 5U (1 + 1e-6) relative of its exact value, plus 3 * 2^-150
absolute where squares are subnormal.  A minimum of values that each err by that much errs by that much, so
  E = 2.5U (1 + 1e-6) D + 2^-74   (the square root halves the relative error),   allowance = E + 2U (D + E)
Exact: an empty database, a database of only NaN / inf points and a NaN query give +inf (fminf drops NaN candidates, the
rule pointgrid.cu documents); an exact duplicate gives exactly 0.

Bitwise kernels (no bound): m3r_im2col16 is F.unfold(img, 16, stride=16).transpose(1, 2), the patch matrix conv2d
multiplies by w.reshape(D, 768), rounded to 16 bit as tensor.to(dtype) rounds; m3r_unpatchify is a pixel shuffle;
m3r_attn_state_fill writes o = 0 and (m, l) = (-inf, 0); m3r_peer_bcast is a byte copy.

The bounds are validated against a plain-torch emulation of the kernels' fp32 arithmetic in
test_elementwise_bound_cpu.py: the faithful emulation stays within half of each allowance and every planted fault
exceeds it."""
import math

import numpy as np
import torch

from gemm_ref import U32, out_bound

C_POW, C_TRIG, C_EXP, C_EXPM1 = 4, 2, 2, 1              # CUDA single-precision maximum errors, in ulp
CLAMP = float(np.float32(1e-8))                           # the fp32 1e-8 of the clamp
LN_FLT_MAX = math.log(float(np.finfo(np.float32).max))    # 88.72...: expf / expm1f overflow above it
CHUNK_ELEMS = 1 << 22                                     # float64 [queries, points, 3] elements per chunk (32 MB)
GRIDS = [(14, 14), (24, 32), (32, 24), (18, 32), (21, 32)]   # 224x224, 512x384, 384x512, 512x288, 512x336
F32 = lambda v: float(np.float32(v))                      # noqa: E731


# ------------------------------------------------------------------------------------------------ RoPE
def c_theta(Q, base):
    """Relative error of the kernel's angle, in units of U (module docstring)."""
    return 2 * C_POW + 2 + (math.log(F32(base)) if Q & (Q - 1) else 0.0)


def rope_trig(pos, Q, base, f0):
    """pos [..., 2] int64 -> exact (cos, sin) [..., 2, Q] float64 of theta = p f0 / base^(d/Q), their error bounds
    e_tab and the table allowance."""
    d = torch.arange(Q, dtype=torch.float64, device=pos.device)
    inv = F32(f0) / F32(base) ** (d / Q)
    th = pos.double()[..., None] * inv                                   # [..., 2, Q]
    dth = c_theta(Q, base) * U32 * th.abs()
    cs, sn = torch.cos(th), torch.sin(th)
    trig = lambda r: 2 * C_TRIG * U32 * (r.abs() + dth)                # noqa: E731
    ec, es = dth + trig(cs), dth + trig(sn)
    return cs, sn, ec, es, ec + trig(cs), es + trig(sn)


def rope_table_ref(pos, base, f0):
    """m3r_rope_table of pos [T, 2] int64: (exact table, entry error bound e_tab, allowance), each [T, 64] float64."""
    cs, sn, ec, es, ac, as_ = rope_trig(pos, 16, base, f0)
    lay = lambda c, s: torch.cat([c[:, 0], s[:, 0], c[:, 1], s[:, 1]], 1)  # noqa: E731
    return lay(cs, sn), lay(ec, es), lay(ac, as_)


def rope_2d_ref(tok, pos, base, fwd):
    """curope rope_2d of tok [B, N, H, D] (16-bit or fp32 values, any strides) by pos [B, N, 2] int64: (exact rotated
    tokens [B, N, H, D] float64, allowance of the result stored in tok's dtype)."""
    B, N, H, D = tok.shape
    Q = D // 4
    cs, sn, ec, es, _, _ = rope_trig(pos, Q, base, fwd)                  # [B, N, 2, Q]
    t = tok.double()
    val, err = torch.empty_like(t), torch.empty_like(t)
    for a in range(2):
        c, s = cs[:, :, None, a], sn[:, :, None, a]                      # [B, N, 1, Q]
        e_c, e_s = ec[:, :, None, a], es[:, :, None, a]
        u, v = t[..., 2 * a * Q:2 * a * Q + Q], t[..., 2 * a * Q + Q:2 * a * Q + 2 * Q]
        for lo, x, y, sg in ((2 * a * Q, u, v, -1.0), (2 * a * Q + Q, v, u, 1.0)):
            r = x * c + sg * y * s
            e1 = x.abs() * e_c + y.abs() * e_s
            e1 = e1 + U32 * (x.abs() * (c.abs() + e_c) + y.abs() * (s.abs() + e_s))
            val[..., lo:lo + Q], err[..., lo:lo + Q] = r, e1 + U32 * (r.abs() + e1)
    return val, out_bound(val, err, tok.dtype)


def grid_pos(gh, gw, dy=0, dx=0):
    """[gh * gw, 2] int64 (y, x) positions of a patch grid in raster order, offset by (dy, dx)."""
    ys, xs = torch.meshgrid(torch.arange(gh), torch.arange(gw), indexing="ij")
    return torch.stack([ys.flatten() + dy, xs.flatten() + dx], 1)


TABLE_CASES = [(f"grid{gh}x{gw}_f{f0:.4g}", grid_pos(gh, gw), 100.0, f0) for gh, gw in GRIDS for f0 in (1.0, 224 / 512)]
TABLE_CASES += [("beyond_2000_3000", grid_pos(24, 32, 2000, 3000), 100.0, 1.0),
                ("beyond_64x64_f0", grid_pos(64, 64, 300, 900), 100.0, 224 / 512),
                ("base10000", grid_pos(14, 14), 10000.0, 1.0)]

RDT = [torch.float32, torch.float16, torch.bfloat16]
ROPE_CASES = []
for i, (dt, D) in enumerate([(dt, D) for dt in RDT for D in (4, 12, 64, 128)]):
    fwd = (1.0, 224 / 512, -1.0, -224 / 512)[i % 4]
    ROPE_CASES.append((f"{str(dt)[6:]}_D{D}_fwd{fwd:.3g}_{('grid', 'negative', 'large')[i % 3]}", dt, 2, 35, 3, D, fwd,
                       ("grid", "negative", "large")[i % 3]))


def rope_inputs(dt, B, N, H, D, kind, seed):
    """Tokens [B, N, H, D] of dtype dt (CPU) and positions [B, N, 2] int64: a raster grid 7 wide, random on
    [-3000, 3000), or random on [0, 5000)."""
    g = torch.Generator().manual_seed(seed)
    tok = (torch.randn(B, N, H, D, generator=g) * 2).to(dt)
    if kind == "grid":
        pos = grid_pos((N + 6) // 7, 7)[:N][None].expand(B, -1, -1)
    elif kind == "negative":
        pos = torch.randint(-3000, 3000, (B, N, 2), generator=g)
    else:
        pos = torch.randint(0, 5000, (B, N, 2), generator=g)
    return tok, pos.contiguous()


# ------------------------------------------------------------------------------------------------ postprocess
def postprocess_ref(pm):
    """m3r_postprocess of pm [P, 7] fp32: {name: (reference, allowance)} for pts3d, pts3d_local [P, 3] and conf [P],
    float64.  The reference is the exact value where the reference's fp32 formula is finite and its non-finite class
    (NaN / +-inf) elsewhere; the allowance is 0 there and at zero vectors (exact classes, see check())."""
    from oracle import must3r_oracle as orc
    cls = orc.postprocess(pm)
    out = {}
    for name, lo in (("pts3d", 0), ("pts3d_local", 3)):
        x = pm[:, lo:lo + 3].double()
        d = x.norm(dim=1, keepdim=True)
        val = x * torch.expm1(d) / d.clamp_min(CLAMP)
        A = torch.where(d > 0, d / -torch.expm1(-d), torch.ones_like(d))  # d e^d / (e^d - 1), stable for large d
        Dd = 2.5 * U32 * d + 2.0 ** -74
        rel = 2 * (A - (d > CLAMP * (1 + 4 * U32)).double()) * Dd / d + 2 * C_EXPM1 * U32 + 2 * U32
        e = 1.0001 * rel * val.abs()
        bnd = e + 2 * U32 * (val.abs() + e) + 2.0 ** -149
        fin = torch.isfinite(cls[name].double())
        out[name] = (torch.where(fin, val, cls[name].double()), torch.where(fin & (d > 0), bnd, torch.zeros_like(bnd)))
    c6 = pm[:, 6].double()
    ex = torch.exp(c6)
    val = 1 + ex
    e = 2 * C_EXP * U32 * ex
    fin = torch.isfinite(cls["conf"].double())
    out["conf"] = (torch.where(fin, val, cls["conf"].double()),
                   torch.where(fin, e + 2 * U32 * (val + e), torch.zeros_like(val)))
    return out


def zero_sign_ok(pm, out, lo):
    """At zero vectors of channels lo:lo+3 the output is exactly 0 with the input's sign."""
    z = (pm[:, lo:lo + 3] == 0).all(1)
    return bool((out[z] == 0).all()) and bool((torch.signbit(out[z]) == torch.signbit(pm[z, lo:lo + 3])).all())


SPECIAL_PM = [  # (x, y, z) of both groups and c6 of the rows that start every postprocess input
    ((0.0, 0.0, 0.0), 0.0), ((-0.0, 0.0, -0.0), -1.0), ((float("nan"), 1.0, 2.0), float("nan")),
    ((1.0, 2.0, float("nan")), float("inf")), ((float("inf"), 0.5, 0.5), float("-inf")),
    ((0.0, float("-inf"), 3.0), 95.0), ((90.0, 0.0, 0.0), -100.0), ((-60.0, 70.0, 0.0), 80.0),
    ((500.0, -600.0, 700.0), 88.0), ((88.0, 0.0, 0.0), -88.0), ((0.0, 50.0, -70.0), 3.0),
    ((1e-20, -1e-20, 1e-20), 0.0), ((1e-30, 0.0, -1e-30), 0.5), ((1e-9, 0.0, 0.0), 1.0),
    ((5e-9, -5e-9, 0.0), -2.0), ((3e-8, 0.0, 4e-8), 2.0), ((1e-5, 2e-5, -2e-5), 0.1), ((0.0, 0.0, 1e-2), -0.1),
]


def pm_inputs(P, seed, device):
    """[P, 7] fp32 head outputs: the SPECIAL_PM rows first, then random directions whose norms are log-uniform on
    [1e-9, 80] (each group on its own), confidence logits on [-20, 20]."""
    g = torch.Generator().manual_seed(seed)
    pm = torch.empty(P, 7)
    for lo in (0, 3):
        v = torch.randn(P, 3, generator=g)
        n = torch.exp(torch.empty(P, 1).uniform_(math.log(1e-9), math.log(80.0), generator=g))
        pm[:, lo:lo + 3] = v / v.norm(dim=1, keepdim=True) * n
    pm[:, 6] = torch.empty(P).uniform_(-20, 20, generator=g)
    for i, (xyz, c6) in enumerate(SPECIAL_PM[:P]):
        j = (i + 5) % len(SPECIAL_PM)
        pm[i, 0:3], pm[i, 3:6], pm[i, 6] = torch.tensor(xyz), torch.tensor(SPECIAL_PM[j][0]), c6
    return pm.to(device)


# ------------------------------------------------------------------------------------------------ nearest neighbour
def nn_ref(q, db):
    """m3r_nn_min_dist of q [Q, 3] and db [P, 3] fp32: (exact minimum distance [Q] float64, allowance; 0 where the
    result is exact: +inf and 0)."""
    Qn, P = q.shape[0], db.shape[0]
    best = torch.full((Qn,), math.inf, dtype=torch.float64, device=q.device)
    if P:
        p64 = db.double()
        step = max(1, CHUNK_ELEMS // (3 * P))
        for i in range(0, Qn, step):
            s = ((q[i:i + step, None, :].double() - p64[None]) ** 2).sum(2)
            best[i:i + step] = torch.nan_to_num(s, nan=math.inf, posinf=math.inf).amin(1)
    D = best.sqrt()
    e = 2.5 * U32 * (1 + 1e-6) * D + 2.0 ** -74
    bnd = e + 2 * U32 * (D + e)
    return D, torch.where(torch.isfinite(D) & (D > 0), bnd, torch.zeros_like(bnd))


NN_P = [0, 1, 1023, 1024, 1025, 4097, 65536]
NN_Q = [1, 255, 256, 257, 3136]                  # 3136: a 224x224 frame subsampled by 4
NN_KINDS = ["cluster", "far", "ties"]


def nn_points(kind, P, Q, seed):
    """(queries [Q, 3], database [P, 3]) fp32 on the CPU.  cluster: eight tight Gaussian clusters, queries near database
    points and anywhere; far: |p| ~ 1e3 with 1e-3 spacing; ties: an integer lattice queried at lattice points (exact
    duplicates) and at midpoints (exact ties).  Every kind has NaN and inf database points and a NaN query."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)                          # noqa: E731
    if kind == "cluster":
        c = r(8, 3) * 4 - 2
        db = c[torch.randint(0, 8, (P,), generator=g)] + torch.randn(P, 3, generator=g) * 0.05
        q = c[torch.randint(0, 8, (Q,), generator=g)] + torch.randn(Q, 3, generator=g) * 0.08
    elif kind == "far":
        db = 1000.0 + torch.randint(-40, 40, (P, 3), generator=g).float() * 1e-3
        q = 1000.0 + torch.randint(-45, 45, (Q, 3), generator=g).float() * 1e-3 + (r(Q, 3) - 0.5) * 1e-3
    else:
        db = torch.randint(-6, 6, (P, 3), generator=g).float()
        q = torch.randint(-6, 6, (Q, 3), generator=g).float() + 0.5 * torch.randint(0, 2, (Q, 3), generator=g).float()
    if P:
        if Q > 1:
            q[1::5] = db[torch.randint(0, P, (len(q[1::5]),), generator=g)]   # exact duplicates
        db[::7, 1] = math.nan
        db[3::11, 2] = math.inf
    if Q > 2:
        q[2, 0] = math.nan
    return q.contiguous(), db.contiguous()


# ------------------------------------------------------------------------------------------------ check
def check(out, val, bnd, what, dims=None) -> float:
    """Fail on the first element of `out` that errs by more than its allowance, naming its index (dims: the names of
    out's dimensions); where the allowance is 0 the result must be exact: the same value, the same infinity, or NaN
    where val is NaN.  Return the worst err / allowance over the other elements."""
    o = out.double()
    exact = bnd == 0
    err = (o - val).abs()
    ratio = torch.where(exact, torch.zeros_like(err), err / torch.where(exact, torch.ones_like(bnd), bnd))
    same = (o == val) | (torch.isnan(o) & torch.isnan(val))
    bad = torch.where(exact, ~same, ~(ratio <= 1))                        # ~(<=): also catches NaN
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        idx = np.unravel_index(i, tuple(out.shape))
        names = dims or [f"dim{k}" for k in range(out.dim())]
        at = ", ".join(f"{n} {int(k)}" for n, k in zip(names, idx))
        kind = "exact" if bool(exact.flatten()[i]) else f"error {float(err.flatten()[i]):.3g} > allowance " \
                                                            f"{float(bnd.flatten()[i]):.3g}"
        raise AssertionError(f"{what}: element ({at}): got {float(o.flatten()[i]):.9g}, reference "
                             f"{float(val.flatten()[i]):.9g}, {kind} ({int(bad.sum())} elements over)")
    return float(ratio.max()) if ratio.numel() else 0.0
