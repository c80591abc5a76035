"""The allowances of tests/elementwise_ref.py are neither flaky nor blind: a plain-torch emulation of the kernels' fp32
arithmetic stays within half of each of them over the case matrix, and each planted fault exceeds one of them in at least
one case where it applies, with a message naming the element.

The emulations follow csrc/elementwise.cu: the RoPE table's powf / division / product / cosf / sinf in fp32, the RoPE
rotation in fp32 products rounded once to the token type, the postprocess expression in kernel order (squares summed,
sqrt, expm1 / max(d, 1e-8), times x; 1 + exp), and the nearest-neighbour scan's rounded differences, fma chain and
sqrt over 1024-point tiles, NaN candidates dropped."""
import math

import pytest
import torch

from elementwise_ref import (NN_KINDS, ROPE_CASES, TABLE_CASES, check, nn_points, nn_ref, pm_inputs, postprocess_ref,
                             rope_2d_ref, rope_inputs, rope_table_ref, zero_sign_ok)
from gemm_ref import off_by_4ulp

F32 = torch.float32


# ------------------------------------------------------------------------------------------------ emulations
def fma(a, b, c):
    """fp32 a * b + c with one rounding (the product is exact in float64)."""
    return (a.double() * b.double() + c.double()).float()


def emulate_inv_freq(Q, base, f0, div=None):
    d = torch.arange(Q, dtype=F32)
    return torch.tensor(f0, dtype=F32) / torch.pow(torch.tensor(base, dtype=F32), d / (div or float(Q)))


def emulate_table(pos, base, f0, mut=None):
    inv = emulate_inv_freq(16, base, 1.0 if mut == "f0_dropped" else f0, div=15.0 if mut == "freq_index" else None)
    ang = pos.to(F32)[:, :, None] * inv                                   # [T, 2, 16]
    c, s = torch.cos(ang), torch.sin(ang)
    if mut == "cos_sin_swapped":
        c, s = s, c
    tab = torch.cat([c[:, 0], s[:, 0], c[:, 1], s[:, 1]], 1)
    if mut == "halves_swapped":                                           # one row whose y and x differ
        r = int(((pos[:, 0] - pos[:, 1]).abs() > 2).nonzero()[0])
        tab[r] = torch.cat([tab[r, 32:], tab[r, :32]])
    if mut == "next_token_row":
        tab[:-1] = tab[1:].clone()
    return tab


def emulate_rope(tok, pos, base, fwd, mut=None):
    B, N, H, D = tok.shape
    Q = D // 4
    ang = pos.to(F32)[..., None] * emulate_inv_freq(Q, base, fwd)        # [B, N, 2, Q]
    c, s = torch.cos(ang)[:, :, None], torch.sin(ang)[:, :, None]        # [B, N, 1, 2, Q]
    t = tok.float()
    out = t.clone()
    for a in range(2):
        u = t[..., 2 * a * Q:2 * a * Q + Q]
        v = t[..., 2 * a * Q + Q - 1:2 * a * Q + 2 * Q - 1] if mut == "partner_q_minus_1" else \
            t[..., 2 * a * Q + Q:2 * a * Q + 2 * Q]
        out[..., 2 * a * Q:2 * a * Q + Q] = u * c[..., a, :] - v * s[..., a, :]
        out[..., 2 * a * Q + Q:2 * a * Q + 2 * Q] = v * c[..., a, :] + u * s[..., a, :]
    if mut == "head_skipped":
        out[:, :, 1] = t[:, :, 1]
    if mut == "bf16_output":
        return out.to(torch.bfloat16).to(tok.dtype)
    return out.to(tok.dtype)


def emulate_postprocess(pm, mut=None):
    outs = []
    for lo in (0, 3):
        x = pm[:, lo:lo + 3]
        d = torch.sqrt(x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1] + x[:, 2] * x[:, 2])
        num = torch.exp(d) - 1 if mut == "exp_minus_1" else torch.expm1(d)
        den = d if mut == "clamp_removed" else d.clamp_min(1e-8)
        outs.append(x * (num / den)[:, None])
    ex = torch.exp(pm[:, 6])
    conf = ex if mut == "exp_for_1_plus_exp" else 1 + ex
    if mut == "groups_swapped":
        outs.reverse()
    return outs[0], outs[1], conf


def emulate_nn(q, db, mut=None):
    P = db.shape[0]
    if mut == "last_tile_dropped":
        P -= P % 1024
    best = torch.full((q.shape[0],), math.inf)
    for i in range(0, q.shape[0], 256):
        qq = q[i:i + 256, None, :]
        dx, dy, dz = (qq[..., k] - db[None, :P, k] for k in range(3))
        s = fma(dx, dx, fma(dy, dy, dz * dz))
        best[i:i + 256] = torch.nan_to_num(s, nan=math.inf, posinf=math.inf).amin(1) if P else best[i:i + 256]
    out = best if mut == "squared" else torch.sqrt(best)
    if mut == "neighbour_slot":
        out[1] = out[0]
    return out


def fp32_off_by_4ulp(out, bnd, sel):
    """One fp32 element among `sel` moved by 4 ulp: the one where that is largest against its allowance."""
    o = out.clone().flatten()
    a = o.double().abs()
    ulp = torch.exp2(torch.floor(torch.log2(a.clamp_min(2.0 ** -126))) - 23)
    ok = sel.flatten() & torch.isfinite(a) & (bnd.flatten() > 0) & (a > 0)
    i = int(torch.where(ok, 4 * ulp / bnd.flatten(), torch.zeros_like(ulp)).argmax())
    o[i] = float(o[i]) + 4 * float(ulp[i]) * (1 if o[i] >= 0 else -1)
    return o.view_as(out)


# ------------------------------------------------------------------------------------------------ case matrix
NN_CPU = [(P, Q) for P in (0, 1, 1023, 1024, 1025, 4097) for Q in (1, 255, 256, 257, 3136)]


def nn_case(i):
    P, Q = NN_CPU[i]
    return nn_points(NN_KINDS[i % 3], P, Q, seed=i)


# ------------------------------------------------------------------------------------------------ faithful emulation
def run_table(case, mut=None):
    name, pos, base, f0 = case
    val, _, bnd = rope_table_ref(pos, base, f0)
    return check(emulate_table(pos, base, f0, mut), val, bnd, f"table {name}", dims=("token", "column"))


def run_rope(case, mut=None):
    name, dt, B, N, H, D, fwd, kind = case
    tok, pos = rope_inputs(dt, B, N, H, D, kind, seed=D)
    val, bnd = rope_2d_ref(tok, pos, 100.0, fwd)
    out = emulate_rope(tok, pos, 100.0, fwd, mut if mut != "ulp4" else None)
    if mut == "ulp4":
        out = off_by_4ulp(out.reshape(-1, D), bnd.reshape(-1, D)).view_as(out)
    return check(out, val, bnd, f"rope {name}", dims=("b", "n", "head", "column"))


def run_postprocess(P, mut=None):
    pm = pm_inputs(P, seed=P, device="cpu")
    ref = postprocess_ref(pm)
    got = dict(zip(("pts3d", "pts3d_local", "conf"), emulate_postprocess(pm, mut if mut != "ulp4" else None)))
    if mut == "ulp4":
        small = (pm[:, 0:3].double().norm(dim=1) < 1)[:, None].expand(-1, 3)
        got["pts3d"] = fp32_off_by_4ulp(got["pts3d"], ref["pts3d"][1], small)
    worst = {}
    for k, (val, bnd) in ref.items():
        worst[k] = check(got[k], val, bnd, f"postprocess {k} P={P}", dims=("point", "channel")[:got[k].dim()])
    for k, lo in (("pts3d", 0), ("pts3d_local", 3)):
        assert zero_sign_ok(pm, got[k], lo), f"postprocess {k}: a zero vector lost its sign"
    return max(worst.values())


def run_nn(i, mut=None):
    q, db = nn_case(i)
    val, bnd = nn_ref(q, db)
    return check(emulate_nn(q, db, mut), val, bnd, f"nn P={db.shape[0]} Q={q.shape[0]} {NN_KINDS[i % 3]}",
                 dims=("query",))


PP_SIZES = [1, 18, 4000, 20000]


def test_faithful_emulation_within_half_the_bound():
    worst = {"table": max(run_table(c) for c in TABLE_CASES),
             "rope": max(run_rope(c) for c in ROPE_CASES),
             "postprocess": max(run_postprocess(P) for P in PP_SIZES),
             "scan": max(run_nn(i) for i in range(len(NN_CPU)))}
    print({k: round(v, 3) for k, v in worst.items()})
    assert max(worst.values()) <= 0.5, worst


def test_exact_classes_of_the_emulation():
    """The exact rows the allowance pins: NaN / inf queries and databases, duplicates, empty and all-NaN databases."""
    q = torch.tensor([[0.0, 0.0, 0.0], [math.nan, 0.0, 0.0], [1.0, 2.0, 3.0]])
    assert torch.isinf(emulate_nn(q, torch.zeros(0, 3))).all()
    allbad = torch.tensor([[math.nan, 0.0, 0.0], [0.0, math.inf, 0.0], [math.nan, math.nan, math.nan]])
    assert torch.isinf(emulate_nn(q, allbad)).all() and torch.isinf(nn_ref(q, allbad)[0]).all()
    out = emulate_nn(q, torch.tensor([[1.0, 2.0, 3.0], [math.nan, 2.0, 3.0]]))
    assert float(out[2]) == 0.0 and math.isinf(float(out[1]))


# ------------------------------------------------------------------------------------------------ planted faults
MUTATIONS = {
    "table:freq_index": TABLE_CASES[:4], "table:halves_swapped": TABLE_CASES[:4],
    "table:cos_sin_swapped": TABLE_CASES[:2], "table:f0_dropped": [c for c in TABLE_CASES if c[3] != 1.0][:3],
    "table:next_token_row": TABLE_CASES[:4],
    "rope:partner_q_minus_1": ROPE_CASES, "rope:head_skipped": ROPE_CASES,
    "rope:bf16_output": [c for c in ROPE_CASES if c[1] == torch.float16],
    "rope:ulp4": [c for c in ROPE_CASES if c[1] != torch.float32],
    "postprocess:clamp_removed": PP_SIZES, "postprocess:exp_minus_1": PP_SIZES,
    "postprocess:exp_for_1_plus_exp": PP_SIZES, "postprocess:groups_swapped": PP_SIZES, "postprocess:ulp4": PP_SIZES,
    "scan:last_tile_dropped": [i for i, (P, Q) in enumerate(NN_CPU) if P % 1024 and P > 1024],
    "scan:squared": list(range(len(NN_CPU))), "scan:neighbour_slot": [i for i, (P, Q) in enumerate(NN_CPU) if Q > 1 and P],
}
RUN = {"table": run_table, "rope": run_rope, "postprocess": run_postprocess, "scan": run_nn}


@pytest.mark.parametrize("mut", list(MUTATIONS))
def test_each_fault_is_rejected(mut):
    group, fault = mut.split(":")
    cases = MUTATIONS[mut]
    assert cases, mut
    for c in cases:
        try:
            RUN[group](c, fault)
        except AssertionError as e:
            msg = str(e)
            assert "element (" in msg or "zero vector" in msg, msg
            print(msg)
            return
    pytest.fail(f"{mut} passed the allowance in every case it applies to")
