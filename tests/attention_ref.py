"""Float64 reference of m3r_attention, the element-wise error allowance of the kernel's arithmetic, and the problem
generator that the CPU bound test and the GPU contract test share.

reference() takes the arguments of m3r_attn_args (Q, the two key segments with their batch strides, kv_group, the skip
range and scale) on the same 16-bit inputs, computes the softmax in float64 on the inputs' device, and returns, for every
(row, head, column), the output and the quantities the allowance is built from.  bound() turns them into the allowance,
check() compares an output with it element by element.

The allowance, for output column c of one (row, head), with p_j = exp(s_j - max s) the float64 softmax weights of the
attended keys, l = sum_j p_j and ref_c = sum_j p_j v_jc / l (u = 2^-11 fp16, 2^-8 bf16; KAPPA = 6):

  (2u + 2^-21) |ref_c|                            output rounding: round-to-nearest errs by up to u 2^e <= u |x| for
                                                  |x| in [2^e, 2^e+1); the factor 2 keeps a correctly rounded output at
                                                  half the allowance.  2^-21 covers 1/l and the final fp32 products.
+ KAPPA u sqrt(sum_j p_j^2 v_jc^2) / l            P is rounded to the operand type before P V: independent
                                                  round-to-nearest errors, |delta_j| <= u, zero mean.  (Row sums use the
                                                  unrounded P.)  KAPPA u is KAPPA sqrt(3) standard deviations.
+ sum_j p_j eps_j |v_jc - ref_c| / l              fp32 errors that perturb each weight p_j by a relative eps_j, with
                                                  |v_jc - ref_c| <= |v_jc| + |ref_c| (matmul-sized):
      eps_j = 2^-24 (C_S a_j + C_M a_max + C_0),  a_j = scale sum_i |q_i k_ji|, a_max = max_j a_j
      C_S = 140: S = Q K^T on the tensor cores, 4 k16 steps, each adding 16 exact products to the fp32 accumulator
                 with up to 17 truncations of at most 2^-23 of the largest magnitude (<= sum_i |q_i k_ji|): 68 x 2; plus
                 the fp32 scale * log2(e) (1) and the rounding of the fma that forms the exponent (1).
      C_M = 10:  the running max folded into the exponent (m * sl2 rounded: 1), the lazy refresh factor versus the two
                 rounded offsets it bridges (4), the split merge's weights exp2(m_s - m) (2), the fma's second operand
                 (1), rounded up.
      C_0 = 16:  ex2.approx (2 ulp) for P, for the refresh factor and for the merge weights, and the fp32 products by
                 those factors, rounded up.
+ KAPPA 2^-23 sqrt(n_add) (|ref_c| + KAPPA sqrt(sum_j p_j^2 v_jc^2) / l)
                                                  fp32 accumulation of O = P V on the tensor cores (n_add = 17 per k16 step,
                                                  8 steps per 128-key tile): truncation errors of at most 2^-23 of the
                                                  running sum, whose signs follow the random signs of the products; the
                                                  running sum stays within |ref| + KAPPA standard deviations.  It also
                                                  covers the fp32 row sums (fewer, round-to-nearest additions).
+ fp16 only: KAPPA 2^-25 sqrt(sum_j v_jc^2) / l   P below 2^-14 is subnormal in fp16: absolute error <= 2^-25.

The running max the kernel subtracts is never above the true max, so its P is p_j times a factor >= 1: every relative
term above holds, and the subnormal one only shrinks.

lse_allowance() bounds m + log2(l) of an exported state against the float64 log-sum-exp in log2 units: the same eps_j
(weighted by p_j / l), the fp32 row-sum term and the rounding of m itself, converted to log2 units.

All of this is validated against a plain-torch emulation of the kernel's algorithm in test_attention_bound_cpu.py: the
faithful emulation stays within half the allowance and each of eight planted faults exceeds it."""
import math
from dataclasses import dataclass, replace
from typing import Optional

import torch

HD = 64
KAPPA = 6.0
C_S, C_M, C_0 = 140.0, 10.0, 16.0
U = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
LOG2E = 1.4426950408889634
CHUNK_ELEMS = 1 << 26                    # float64 elements per [heads, rows, keys] temporary (512 MB)


# ------------------------------------------------------------------------------------------------ keys of one batch
def skip_range(kw, b):
    """[lo, hi) of the keys query batch b skips (empty when skip_len <= 0)."""
    if kw["skip_len"] <= 0:
        return 0, 0
    lo = kw["skip_lo"] + (b % kw["kv_group"]) * kw["skip_step"]
    return lo, lo + kw["skip_len"]


def keys_of(kw, b):
    """K and V of query batch b over both segments in global key order ([Nk0 + Nk1, H*64] each, input dtype) and the
    mask of the keys it attends."""
    kvb = b // kw["kv_group"]
    ks, vs = [], []
    for s in (0, 1):
        n = kw[f"Nk{s}"]
        if n > 0:
            r0 = kvb * kw[f"kv_bstride{s}"]
            ks.append(kw[f"k{s}"][r0:r0 + n, :kw["H"] * HD])
            vs.append(kw[f"v{s}"][r0:r0 + n, :kw["H"] * HD])
    k, v = torch.cat(ks), torch.cat(vs)
    lo, hi = skip_range(kw, b)
    g = torch.arange(k.shape[0], device=k.device)
    return k, v, ~((g >= lo) & (g < hi))


# ------------------------------------------------------------------------------------------------ reference
@dataclass
class Ref:
    B: int
    H: int
    Nq: int
    out: torch.Tensor        # [B*Nq, H*64] float64 softmax(Q K^T scale) V
    pv2: torch.Tensor        # sqrt(sum_j p_j^2 v_jc^2) / l
    e_v: torch.Tensor        # sum_j p_j eps_j (|v_jc| + |ref_c|) / l
    v2: torch.Tensor         # sqrt(sum_j v_jc^2) / l
    lse2: torch.Tensor       # [B*Nq, H] log2 sum_j exp(s_j): the exported m + log2(l)
    e_l: torch.Tensor        # [B*Nq, H] sum_j p_j eps_j / l
    n_add: torch.Tensor      # [B*Nq, 1] fp32 accumulation steps into O


def reference(q, k0, v0, k1=None, v1=None, *, B, H, Nq, Nk0, kv_bstride0, Nk1=0, kv_bstride1=0, kv_group=1,
              skip_lo=0, skip_step=0, skip_len=0, scale=0.125) -> Ref:
    kw = dict(q=q, k0=k0, v0=v0, k1=k1, v1=v1, B=B, H=H, Nq=Nq, Nk0=Nk0, kv_bstride0=kv_bstride0, Nk1=Nk1,
              kv_bstride1=kv_bstride1, kv_group=kv_group, skip_lo=skip_lo, skip_step=skip_step, skip_len=skip_len)
    dev, D = q.device, H * HD
    scale = float(torch.tensor(scale, dtype=torch.float32))           # the kernel gets the fp32 value
    f64 = dict(device=dev, dtype=torch.float64)
    out, pv2, e_v, v2 = (torch.empty(B * Nq, D, **f64) for _ in range(4))
    lse2, e_l = torch.empty(B * Nq, H, **f64), torch.empty(B * Nq, H, **f64)
    tiles = (Nk0 + 127) // 128 + (Nk1 + 127) // 128
    n_add = torch.full((B * Nq, 1), 17.0 * 8 * tiles + 64, **f64)
    for b in range(B):
        k, v, keep = keys_of(kw, b)
        k = k[keep].double().view(-1, H, HD).transpose(0, 1)          # [H, n, 64]
        v = v[keep].double().view(-1, H, HD).transpose(0, 1)
        n = k.shape[1]
        ka, va, vsq = k.abs(), v.abs(), v * v
        step = max(1, CHUNK_ELEMS // (H * n))
        for r0 in range(0, Nq, step):
            r1 = min(Nq, r0 + step)
            rows = slice(b * Nq + r0, b * Nq + r1)
            qq = q[rows, :D].double().view(-1, H, HD).transpose(0, 1)  # [H, r, 64]
            s = (qq @ k.transpose(1, 2)) * scale
            a = (qq.abs() @ ka.transpose(1, 2)) * scale
            m = s.amax(-1, keepdim=True)
            p = torch.exp(s - m)
            del s
            l = p.sum(-1, keepdim=True)
            o = (p @ v) / l
            pe = p * (2.0 ** -24) * (C_S * a + C_M * a.amax(-1, keepdim=True) + C_0)
            del a
            pes = pe.sum(-1, keepdim=True)
            ev = (pe @ va + o.abs() * pes) / l
            del pe
            pv = torch.sqrt((p * p) @ vsq) / l
            vv = torch.sqrt(vsq.sum(1, keepdim=True)) / l
            put = lambda t: t.transpose(0, 1).reshape(r1 - r0, D)     # noqa: E731
            out[rows], e_v[rows], pv2[rows], v2[rows] = put(o), put(ev), put(pv), put(vv)
            lse2[rows] = ((m + torch.log(l)) * LOG2E)[..., 0].transpose(0, 1)
            e_l[rows] = (pes / l)[..., 0].transpose(0, 1)
    return Ref(B, H, Nq, out, pv2, e_v, v2, lse2, e_l, n_add)


def bound(ref: Ref, dtype) -> torch.Tensor:
    """Element-wise allowance [B*Nq, H*64] for a 16-bit output of m3r_attention (or m3r_attn_merge) in `dtype`."""
    u = U[dtype]
    r = ref.out.abs()
    b = (2 * u + 2.0 ** -21) * r + KAPPA * u * ref.pv2 + ref.e_v
    b = b + KAPPA * 2.0 ** -23 * torch.sqrt(ref.n_add) * (r + KAPPA * ref.pv2)
    if dtype == torch.float16:
        b = b + KAPPA * 2.0 ** -25 * ref.v2
    return b


def lse_allowance(ref: Ref) -> torch.Tensor:
    """[B*Nq, H] allowance of m + log2(l) (log2 units) against ref.lse2."""
    return (ref.e_l + KAPPA * 2.0 ** -23 * torch.sqrt(ref.n_add)) * LOG2E + 2.0 ** -22 * (ref.lse2.abs() + 1)


def check(out, ref: Ref, bnd, what="") -> float:
    """Fail on the first element of `out` ([B*Nq, H*64]) that is not finite or errs by more than its allowance; return
    the worst err / allowance."""
    err = (out.double() - ref.out).abs()
    ratio = err / bnd
    bad = ~(ratio <= 1)                                                  # also catches NaN
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        row, col = divmod(i, ref.H * HD)
        bb, qi = divmod(row, ref.Nq)
        raise AssertionError(
            f"{what}: batch {bb} query {qi} head {col // HD} column {col % HD}: got {float(out[row, col]):.6g}, "
            f"reference {float(ref.out[row, col]):.6g}, error {float(err[row, col]):.3g} > allowance "
            f"{float(bnd[row, col]):.3g} ({int(bad.sum())} elements over)")
    return float(ratio.max())


# ------------------------------------------------------------------------------------------------ planted output faults
def ulp(x):
    """One unit in the last place of 16-bit values x (normal range)."""
    bits = 11 if x.dtype == torch.float16 else 8
    e = torch.floor(torch.log2(x.float().abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e - (bits - 1))


def off_by_4ulp(out, ref, bnd):
    """One element moved by 4 ulp: the one where that is largest against its allowance."""
    out = out.clone()
    i = int((4 * ulp(out).double() / bnd).flatten().argmax())
    r, c = divmod(i, out.shape[1])
    out[r, c] = (out[r, c].float() + 4 * ulp(out[r, c])).to(out.dtype)
    return out


def swap_tile_edge(out):
    """Rows 63 and 64 (either side of the first 64-row query tile edge) swapped."""
    out = out.clone()
    out[[63, 64]] = out[[64, 63]]
    return out


# ------------------------------------------------------------------------------------------------ problems
@dataclass(frozen=True)
class Case:
    """One attention problem.  gap0 / gap1: NaN rows between key batches (kv_bstride = Nk + gap); gap0 = -1 gives
    kv_bstride0 = 0, one memory for every key batch.  layout: "pad" - Q, K|V in separate buffers with a NaN head's worth of
    columns after each operand; "qkv3" - self-attention out of the fused [rows, 3D] q|k|v buffer; "qkv5" - queries and the
    segment-1 keys out of the merged [rows, 5D] q|k|v|k|v buffer (the views' new tokens), segment 0 from a [rows, 2D] K|V
    memory.  scores: "rand"; "grow" - the row max grows by more than 2^8 on every key tile; "uniform" - all keys equal;
    "lastmax" - the last key outscores every other.  splits: forced key splits (None: the library's cost model)."""
    name: str
    B: int
    H: int
    Nq: int
    Nk0: int
    Nk1: int = 0
    kv_group: int = 1
    skip: tuple = (0, 0, 0)
    gap0: int = 0
    gap1: int = 0
    layout: str = "pad"
    scores: str = "rand"
    qscale: float = 1.0
    splits: Optional[int] = None
    scale: float = 0.125

    def small(self):
        """The same key lengths and skip layout with fewer heads, queries and batches (for the CPU emulation)."""
        B, g, Nq = self.B, self.kv_group, min(self.Nq, 70)
        if B > 4:
            g = min(g, 2)
            B = 2 * g
        Nk1 = self.Nk1
        if self.layout == "qkv3":
            return replace(self, B=min(B, 2), kv_group=1, H=1, layout="pad", Nq=Nq)
        if self.layout == "qkv5":
            Nk1 = g * Nq if self.Nk1 == self.kv_group * self.Nq else Nk1
            return replace(self, B=B, kv_group=g, H=1, Nq=Nq, Nk1=Nk1, layout="pad",
                           skip=(self.skip[0], Nq if self.skip[1] else 0, Nq if self.skip[2] else 0))
        return replace(self, B=B, kv_group=g, H=min(self.H, 2), Nq=Nq)


HOSTILE_K = 32.0                 # x the unit mean query direction: outscores every attended key by e^8 or more
HOSTILE_V = 4096.0               # |V| of skipped keys: large, finite in both 16-bit types
SENTINEL_NAN = float("nan")


def make_inputs(c: Case, dtype, device, seed=0):
    """Buffers and views of case c: returns (kw, keep) where kw holds the m3r_attn_args fields (q/k0/v0/k1/v1 as views
    into NaN-padded buffers) and keep the buffers alive."""
    g = torch.Generator().manual_seed(seed)
    B, H, Nq, Nk0, Nk1, G = c.B, c.H, c.Nq, c.Nk0, c.Nk1, c.kv_group
    assert B % G == 0
    Bkv, D, Nk = B // G, H * HD, Nk0 + Nk1
    rn = lambda *s: torch.randn(*s, generator=g)                         # noqa: E731
    dirs = rn(H, HD)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)                         # mean query direction per head
    q = rn(B, Nq, H, HD)
    if c.skip[2] > 0 or c.scores in ("grow", "lastmax"):
        q = q + 3.0 * dirs                                               # q . dir ~ 3: one direction wins everywhere
    q = q * c.qscale
    k, v = rn(Bkv, Nk, H, HD), rn(Bkv, Nk, H, HD)
    gi = torch.arange(Nk, dtype=torch.float32)
    if c.scores == "grow":
        k = k + (gi * (16.0 / 128))[None, :, None, None] * dirs           # +8.7 log2 units of max per tile
    elif c.scores == "uniform":
        k = k[:, :1].expand_as(k).clone()
    elif c.scores == "lastmax":
        k[:, -1] = 24.0 * dirs
    if c.gap0 < 0:
        k[:, :Nk0], v[:, :Nk0] = k[:1, :Nk0].clone(), v[:1, :Nk0].clone()  # one memory shared by every key batch
    kw_skip = dict(skip_lo=c.skip[0], skip_step=c.skip[1], skip_len=c.skip[2], kv_group=G)
    for b in range(B):                                                   # every skipped key is hostile
        lo, hi = skip_range(kw_skip, b)
        lo, hi = max(lo, 0), min(hi, Nk)
        if hi > lo:
            k[b // G, lo:hi] = HOSTILE_K * dirs
            sign = torch.where(torch.rand(hi - lo, H, HD, generator=g) < 0.5, -1.0, 1.0)
            v[b // G, lo:hi] = sign * HOSTILE_V * (0.5 + 0.5 * torch.rand(hi - lo, H, HD, generator=g))
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    nan = lambda *s: torch.full(s, SENTINEL_NAN, dtype=dtype)            # noqa: E731
    keep = []

    def kv_buffer(kk, vv, n, gap, ld_extra):
        """[rows, 2*(D + ld_extra)] K | NaN | V | NaN with `gap` NaN rows after each key batch."""
        bs = n + max(gap, 0)
        nb = kk.shape[0] if gap >= 0 else 1
        w = D + ld_extra
        buf = nan(nb * bs + 64, 2 * w)
        for kb in range(nb):
            buf[kb * bs:kb * bs + n, :D] = kk[kb].reshape(n, D)
            buf[kb * bs:kb * bs + n, w:w + D] = vv[kb].reshape(n, D)
        buf = buf.to(device)
        keep.append(buf)
        return buf[:, :D], buf[:, w:w + D], (bs if gap >= 0 else 0)

    kw = dict(B=B, H=H, Nq=Nq, Nk0=Nk0, Nk1=Nk1, kv_group=G, skip_lo=c.skip[0], skip_step=c.skip[1],
              skip_len=c.skip[2], scale=c.scale, k1=None, v1=None, kv_bstride1=0)
    if c.layout == "qkv3":
        assert Nk1 == 0 and G == 1 and Nk0 == Nq and c.gap0 == 0
        buf = torch.cat([q.reshape(B * Nq, D), k.reshape(B * Nq, D), v.reshape(B * Nq, D)], 1)
        buf = torch.cat([buf, nan(64, 3 * D)]).to(device)
        keep.append(buf)
        kw.update(q=buf[:B * Nq, :D], k0=buf[:, D:2 * D], v0=buf[:, 2 * D:], kv_bstride0=Nq)
        return kw, keep
    if c.layout == "qkv5":
        assert Nk1 == G * Nq and c.gap1 == 0
        filler = torch.randn(B * Nq, 2 * D, generator=g).to(dtype)
        buf = torch.cat([q.reshape(B * Nq, D), filler, k[:, Nk0:].reshape(B * Nq, D), v[:, Nk0:].reshape(B * Nq, D)], 1)
        buf = torch.cat([buf, nan(64, 5 * D)]).to(device)
        keep.append(buf)
        kw.update(q=buf[:B * Nq, :D], k1=buf[:, 3 * D:4 * D], v1=buf[:, 4 * D:], kv_bstride1=Nk1)
        if Nk0 > 0:
            k0, v0, bs0 = kv_buffer(k[:, :Nk0], v[:, :Nk0], Nk0, c.gap0, 0)
        else:
            k0, v0, bs0 = kw["k1"], kw["v1"], 0
        kw.update(k0=k0, v0=v0, kv_bstride0=bs0)
        return kw, keep
    qbuf = torch.cat([q.reshape(B * Nq, D), nan(B * Nq, HD)], 1)
    qbuf = torch.cat([qbuf, nan(64, D + HD)]).to(device)
    keep.append(qbuf)
    kw["q"] = qbuf[:B * Nq, :D]
    if Nk0 > 0:
        kw["k0"], kw["v0"], kw["kv_bstride0"] = kv_buffer(k[:, :Nk0], v[:, :Nk0], Nk0, c.gap0, HD)
    if Nk1 > 0:
        kw["k1"], kw["v1"], kw["kv_bstride1"] = kv_buffer(k[:, Nk0:], v[:, Nk0:], Nk1, c.gap1, HD)
    if Nk0 == 0:                                                         # the ABI wants segment-0 pointers all the same
        kw["k0"], kw["v0"], kw["kv_bstride0"] = kw["k1"], kw["v1"], 0
    return kw, keep


def ref_args(kw):
    """The reference() keyword arguments of a make_inputs() problem."""
    return {k: kw[k] for k in ("k1", "v1", "B", "H", "Nq", "Nk0", "kv_bstride0", "Nk1", "kv_bstride1", "kv_group",
                               "skip_lo", "skip_step", "skip_len", "scale")}


# ------------------------------------------------------------------------------------------------ case matrix
def _cases():
    cs = []
    sp = [None, 1, 2, 3, 7, 32]
    for i, nq in enumerate([1, 63, 64, 65, 127, 128, 129, 193, 257]):
        cs.append(Case(f"nq{nq}", B=3, H=2, Nq=nq, Nk0=300, splits=sp[i % len(sp)]))
    for i, nk in enumerate([1, 2, 127, 128, 129, 255, 256, 257, 1000]):
        for s in ([None, 1, 2, 3, 7, 32] if nk in (257, 1000) else [sp[i % len(sp)]]):
            cs.append(Case(f"nk{nk}_s{s}", B=2, H=2, Nq=100, Nk0=nk, splits=s))
    cs += [
        Case("seg0_empty", B=2, H=2, Nq=130, Nk0=0, Nk1=300, splits=3),
        Case("seg0_in_tile", B=2, H=2, Nq=130, Nk0=200, Nk1=300, splits=3, gap0=7, gap1=5),
        Case("seg0_tile_multiple", B=2, H=2, Nq=130, Nk0=256, Nk1=200, splits=2),
        Case("skip_lo_on_edge", B=2, H=2, Nq=100, Nk0=512, Nk1=384, skip=(256, 0, 100), splits=3),
        Case("skip_hi_on_edge", B=2, H=2, Nq=100, Nk0=512, Nk1=384, skip=(156, 0, 100), splits=2),
        Case("skip_edge_minus1", B=2, H=2, Nq=100, Nk0=512, Nk1=384, skip=(255, 0, 130), splits=7),
        Case("skip_edge_plus1", B=2, H=2, Nq=100, Nk0=512, Nk1=384, skip=(129, 0, 254)),
        Case("skip_whole_tiles", B=2, H=2, Nq=100, Nk0=512, Nk1=384, skip=(128, 0, 256), splits=3),
        Case("skip_straddles_segments", B=2, H=2, Nq=100, Nk0=500, Nk1=384, skip=(450, 0, 200), splits=3),
        Case("skip_in_seg1", B=2, H=2, Nq=100, Nk0=500, Nk1=384, skip=(600, 0, 200), splits=2),
        Case("skip_leaves_last_key", B=2, H=2, Nq=65, Nk0=200, Nk1=100, skip=(0, 0, 299), splits=2),
        Case("skip_leaves_first_key", B=2, H=2, Nq=65, Nk0=200, Nk1=100, skip=(1, 0, 299)),
        Case("skip_group_step", B=4, H=2, Nq=100, Nk0=300, Nk1=600, kv_group=2, skip=(100, 300, 250), splits=3),
        Case("skip_empty_splits7", B=2, H=2, Nq=100, Nk0=1024, skip=(128, 0, 768), splits=7),
        Case("skip_empty_splits32", B=2, H=2, Nq=100, Nk0=1024, skip=(100, 0, 900), splits=32),
        Case("group20", B=20, H=1, Nq=65, Nk0=300, kv_group=20, splits=2),
        Case("bstride0_zero", B=4, H=2, Nq=100, Nk0=300, Nk1=200, kv_group=2, gap0=-1, splits=3),
        Case("bstride_gaps", B=4, H=2, Nq=100, Nk0=300, Nk1=200, kv_group=2, gap0=77, gap1=9),
        Case("heads1", B=2, H=1, Nq=129, Nk0=400, splits=3),
        Case("heads16", B=2, H=16, Nq=129, Nk0=400),
        Case("self_qkv3_h12", B=2, H=12, Nq=200, Nk0=200, layout="qkv3", splits=2),
        Case("update_qkv5", B=2, H=12, Nq=100, Nk0=600, Nk1=200, kv_group=2, skip=(600, 100, 100), gap0=33,
             layout="qkv5", splits=3),
        Case("grow", B=2, H=2, Nq=129, Nk0=1000, scores="grow", splits=1),
        Case("grow_split3", B=2, H=2, Nq=129, Nk0=1000, scores="grow", splits=3),
        Case("qscale40", B=2, H=2, Nq=129, Nk0=500, qscale=40.0),
        Case("uniform", B=2, H=2, Nq=129, Nk0=1000, scores="uniform", splits=3),
        Case("lastmax", B=2, H=2, Nq=129, Nk0=1000, scores="lastmax", splits=7),
        Case("scale0.3", B=2, H=2, Nq=129, Nk0=300, scale=0.3, splits=2),
    ]
    return cs


CASES = _cases()
C3_CASES = [
    Case("c3_render", B=20, H=12, Nq=768, Nk0=15360, kv_group=20),
    Case("c3_update", B=1, H=12, Nq=768, Nk0=18 * 768, Nk1=768, skip=(18 * 768, 768, 768), gap0=768, layout="qkv5"),
    Case("c3_decoder_self", B=2, H=12, Nq=768, Nk0=768, layout="qkv3"),
    Case("c3_encoder_self", B=2, H=16, Nq=768, Nk0=768, layout="qkv3"),
]
