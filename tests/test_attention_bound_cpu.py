"""The allowance of tests/attention_ref.py is neither flaky nor blind: a plain-torch emulation of the attention kernel's
algorithm stays within half of it on the whole case matrix of the GPU contract test (fewer heads and queries, the same
key lengths and skip layouts), and each of eight planted faults exceeds it in at least one case where it applies.

The emulation follows csrc/attention.cu: 128-key tiles in the kernel's visiting order (segment 0, then segment 1,
fully masked tiles never visited), the key range cut into contiguous shares of those tiles, per share an online softmax
in fp32 with the lazy max refresh (threshold 8 in log2 units), exp2 of fma(s, scale log2 e, -m), row sums of the
unrounded P, P rounded to the operand type for P V, the partial (O, m, l) of the shares merged with exp2 weights, and the
output O / l rounded to 16 bit."""
import math

import pytest
import torch

from attention_ref import (C3_CASES, CASES, HD, bound, check, keys_of, make_inputs, off_by_4ulp, ref_args, reference,
                           skip_range, swap_tile_edge)

DT = [torch.float16, torch.bfloat16]
THRESH = 8.0


def kernel_splits(c):
    """The split count the library runs for a forced count (None: one share; the cost model needs the GPU's SM count)."""
    tiles = (c.Nk0 + 127) // 128 + (c.Nk1 + 127) // 128
    sp = min(c.splits or 1, 32, tiles)
    chunk = (tiles + sp - 1) // sp
    return (tiles + chunk - 1) // chunk


def emulate(kw, dtype, splits, mut=None):
    """The kernel's arithmetic for every (batch, head); `mut` plants one fault (see MUTATIONS)."""
    B, H, Nq, Nk0 = kw["B"], kw["H"], kw["Nq"], kw["Nk0"]
    sl2 = torch.tensor(kw["scale"], dtype=torch.float32) * torch.tensor(1.4426950408889634, dtype=torch.float32)
    out = torch.empty(B * Nq, H * HD, dtype=dtype)
    pdt = torch.bfloat16 if mut == "p_bf16" else dtype
    for b in range(B):
        k_all, v_all, _ = keys_of(kw, b)
        lo, hi = skip_range(kw, b)
        if mut == "leak_lo" and hi > lo:
            lo += 1
        if mut == "leak_hi" and hi > lo:
            hi -= 1
        tiles = []                                               # (first global key, valid keys) in visiting order
        for base, n in ((0, Nk0), (Nk0, kw["Nk1"])):
            for t0 in range(0, n, 128):
                nv = min(128, n - t0)
                if not (hi > lo and base + t0 >= lo and base + t0 + nv <= hi):
                    tiles.append((base + t0, nv))
        if mut == "drop_tile":
            del tiles[len(tiles) // 2]
        chunk = (len(tiles) + splits - 1) // splits
        for h in range(H):
            q = kw["q"][b * Nq:(b + 1) * Nq, h * HD:(h + 1) * HD].float()
            k = k_all[:, h * HD:(h + 1) * HD].float()
            v = v_all[:, h * HD:(h + 1) * HD].float()
            parts = []
            for sp in range(splits):
                o = torch.zeros(Nq, HD)
                m_used = torch.full((Nq,), -math.inf)
                l = torch.zeros(Nq)
                for g0, nv in tiles[sp * chunk:(sp + 1) * chunk]:
                    g = g0 + torch.arange(128)
                    kt = torch.zeros(128, HD)
                    vt = torch.zeros(128, HD)
                    kt[:nv], vt[:nv] = k[g0:g0 + nv], v[g0:g0 + nv]
                    s = q @ kt.t()
                    keep = (torch.arange(128) < nv) & ~((g >= lo) & (g < hi))
                    if mut == "drop_key":
                        keep &= g != kw["drop"]
                    s = s.masked_fill(~keep, -math.inf)
                    mx = s.amax(1)
                    fresh = (m_used == -math.inf) | ((mx - m_used) * sl2 > THRESH)
                    fresh &= mx > -math.inf
                    alpha = torch.where(fresh, torch.where(m_used == -math.inf, torch.zeros(()),
                                                           torch.exp2((m_used - mx) * sl2)), torch.ones(()))
                    m_used = torch.where(fresh, mx, m_used)
                    l = l * alpha
                    moff = torch.where(m_used == -math.inf, torch.zeros(()), m_used * sl2)
                    p = torch.exp2((s.double() * float(sl2) - moff.double()[:, None]).float())   # fma: one rounding
                    l = l + p.sum(1)
                    if mut != "alpha_l_only":
                        o = o * alpha[:, None]
                    o = o + p.to(pdt).float() @ vt
                parts.append((o, torch.where(m_used == -math.inf, m_used, m_used * sl2), l))
            ms = torch.stack([m for _, m, _ in parts])
            if mut == "merge_wrong_m" and splits > 1:
                ms = torch.cat([ms[1:2], ms[1:]])                # share 0's partial weighted with share 1's max
            m = ms.amax(0)
            oo, ll = torch.zeros(Nq, HD), torch.zeros(Nq)
            for (o, _, l), mk in zip(parts, ms):
                w = torch.where(mk == -math.inf, torch.zeros(()), torch.exp2(mk - m))
                oo, ll = oo + o * w[:, None], ll + l * w
            inv = torch.where(ll > 0, 1.0 / ll, torch.zeros(()))
            out[b * Nq:(b + 1) * Nq, h * HD:(h + 1) * HD] = (oo * inv[:, None]).to(dtype)
    return out


SMALL = [c.small() for c in CASES + C3_CASES]


@pytest.fixture(scope="module")
def problems():
    cache = {}

    def get(c, dtype):
        if (c, dtype) not in cache:
            kw, keep = make_inputs(c, dtype, "cpu", seed=1)
            r = reference(kw["q"], kw["k0"], kw["v0"], **ref_args(kw))
            cache[(c, dtype)] = (kw, keep, r, bound(r, dtype))
        return cache[(c, dtype)]
    return get


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
def test_faithful_emulation_within_half_the_bound(problems, dtype):
    worst = {}
    for c in SMALL:
        kw, _, r, bnd = problems(c, dtype)
        worst[c.name] = check(emulate(kw, dtype, kernel_splits(c)), r, bnd, c.name)
    print({k: round(v, 3) for k, v in worst.items()})
    assert max(worst.values()) <= 0.5, max(worst.items(), key=lambda kv: kv[1])


def by_name(*names):
    return [c for c in SMALL if c.name in names]


# planted fault -> the cases it applies to; each must be rejected in at least one of them.  leak_lo / leak_hi: the first /
# last skipped key is attended; drop_key_127 / 128: the key either side of a tile edge is lost; alpha_l_only: a max
# refresh rescales l but not O; merge_wrong_m: share 0 is weighted with share 1's max; p_bf16: P rounded to bf16 in an
# fp16 run; ulp4: one output element 4 ulp off; swap_tile_edge: rows 63 and 64 swapped; drop_tile: one 128-key tile of
# the 15360-key render memory is skipped.
MUTATIONS = {
    "leak_lo": by_name("skip_lo_on_edge", "skip_whole_tiles", "skip_edge_minus1"),
    "leak_hi": by_name("skip_hi_on_edge", "skip_whole_tiles", "skip_straddles_segments"),
    "drop_key_127": by_name("nk257_s1", "nk1000_s3"),
    "drop_key_128": by_name("nk257_s1", "nk1000_s3"),
    "alpha_l_only": by_name("grow", "grow_split3"),
    "merge_wrong_m": by_name("nk1000_s3", "lastmax", "grow_split3"),
    "p_bf16": by_name("nk257_s1", "nk1000_s1", "nk1000_sNone", "heads1"),
    "ulp4": by_name("nk1_s1", "nk2_s2", "qscale40", "c3_render"),
    "swap_tile_edge": by_name("nq65", "nq129", "c3_render"),
    "drop_tile": by_name("c3_render"),
}


@pytest.mark.parametrize("dtype", DT, ids=["fp16", "bf16"])
@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_each_fault_is_rejected(problems, dtype, mut):
    if mut == "p_bf16" and dtype == torch.bfloat16:
        pytest.skip("P is already bf16")
    cases = MUTATIONS[mut]
    assert cases, mut
    for c in cases:
        kw, _, r, bnd = problems(c, dtype)
        sp = kernel_splits(c)
        if mut in ("ulp4", "swap_tile_edge"):
            out = emulate(kw, dtype, sp)
            out = off_by_4ulp(out, r, bnd) if mut == "ulp4" else swap_tile_edge(out)
        else:
            if mut.startswith("drop_key"):
                kw = dict(kw, drop=int(mut[-3:]))
            out = emulate(kw, dtype, sp, mut="drop_key" if mut.startswith("drop_key") else mut)
        try:
            check(out, r, bnd, f"{mut} {c.name}")
        except AssertionError as e:
            print(e)
            return
    pytest.fail(f"{mut} passed the allowance in every case it applies to")
