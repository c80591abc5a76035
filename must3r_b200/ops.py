"""Operator-level Python wrappers over the C ABI (torch tensors in, torch tensors out).

These mirror the reference's operator seams (SURVEY.md §8b): nn.Linear / LayerNorm call sites,
CoreAttention.attention (must3r/model/blocks/attention.py:37) and curope.rope_2d
(dust3r/croco/models/curope/curope.cpp:49).  They require CUDA tensors; there is no fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib

F16 = {torch.float16: 0, torch.bfloat16: 1}


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)      # ops are called with the tensors' device current


def _p(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _req_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("must3r_b200 ops need CUDA tensors (no CPU fallback)")


def linear(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, act: str = "none",
           residual: Optional[torch.Tensor] = None, rowbias: Optional[torch.Tensor] = None, rb_period: int = 1,
           rb_first: int = 0, rope_tab: Optional[torch.Tensor] = None, rope_cols: int = 0,
           out: Optional[torch.Tensor] = None, out_dtype: Optional[torch.dtype] = None,
           rows_per_batch: int = 0, batch_stride_rows: int = 0, peer_ptrs=(), w_static: bool = False,
           norm_out: Optional[torch.Tensor] = None, norm_eps: float = 1e-6) -> torch.Tensor:
    """out = act(a @ w.T + bias [+rope]) [+ residual]; a [M,K] and w [N,K] fp16/bf16, fp32 accumulate.
    peer_ptrs: device pointers (ints) that receive a copy of the 16-bit output (fused GEMM -> all-gather).
    w_static: w is a weight that the previous launch on this stream does not write (lets the kernel fetch it early)."""
    _req_cuda(a, w)
    assert a.dtype in F16 and w.dtype == a.dtype and a.dim() == 2 and w.dim() == 2
    assert a.stride(1) == 1 and w.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K
    if out is None:
        out = torch.empty((M, N), device=a.device, dtype=out_dtype or a.dtype)
    assert out.stride(-1) == 1
    args = _lib.GemmArgs()
    args.A, args.lda = a.data_ptr(), a.stride(0)
    args.W, args.ldw = w.data_ptr(), w.stride(0)
    args.M, args.N, args.K = M, N, K
    args.is_bf16 = F16[a.dtype]
    args.bias = bias.data_ptr() if bias is not None else None
    args.act = {"none": 0, "gelu": 1}[act]
    if residual is not None:
        assert residual.dtype == torch.float32 and residual.stride(-1) == 1
        args.residual, args.ldr = residual.data_ptr(), residual.stride(-2)
    if rowbias is not None:
        args.rowbias, args.rb_period, args.rb_first = rowbias.data_ptr(), rb_period, rb_first
    if rope_tab is not None:
        assert rope_tab.dtype == torch.float32 and rope_tab.shape[-1] == 64 and rope_tab.is_contiguous()
        args.rope_tab, args.rope_cols, args.rope_period = rope_tab.data_ptr(), rope_cols, rope_tab.shape[0]
    args.out = out.data_ptr()
    args.ldc = out.stride(-2)
    args.out_dtype = 0 if out.dtype == torch.float32 else 1
    if out.dtype != torch.float32:
        assert out.dtype == a.dtype
    args.rows_per_batch, args.batch_stride_rows = rows_per_batch, batch_stride_rows
    args.w_static = 1 if w_static else 0
    args.n_peer_out = len(peer_ptrs)
    for i, ptr in enumerate(peer_ptrs):
        args.peer_out[i] = ptr
    if norm_out is not None:
        # LayerNorm emitted by the producing GEMM: norm_out = affine-free LayerNorm of the fp32 output rows, 16-bit
        assert norm_out.dtype == a.dtype and norm_out.shape == (M, N) and norm_out.stride(1) == 1
        args.norm_out, args.ldn, args.norm_eps = norm_out.data_ptr(), norm_out.stride(0), norm_eps
    _lib.check(_lib.lib().m3r_gemm(C.byref(args), _stream()), "gemm")
    return out


def linear_grouped(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], outs, *, peer_ptrs=None,
                   rows_per_batch: int = 0, batch_stride_rows: int = 0, max_ctas: int = 0) -> None:
    """`groups` GEMMs of one shape in a single launch: a [G, M, K], w [G, N, K] (any row stride between groups),
    bias [G, N] or None, outs = list of G 16-bit tensors [M, N] (one common row stride).
    rows_per_batch > 0: row r of every group goes to output row (r // rows_per_batch) * batch_stride_rows +
    r % rows_per_batch (the memory append into [B, cap, N] buffers).  max_ctas > 0: run on at most that many SMs."""
    _req_cuda(a, w)
    G, M, K = a.shape
    N = w.shape[1]
    assert a.is_contiguous() and w.stride(2) == 1 and w.stride(1) == K and len(outs) == G
    args = _lib.GemmArgs()
    args.A, args.lda, args.W, args.ldw = a.data_ptr(), K, w.data_ptr(), K
    args.M, args.N, args.K, args.is_bf16 = M, N, K, F16[a.dtype]
    args.bias = bias.data_ptr() if bias is not None else None
    args.ldc, args.out_dtype = outs[0].stride(0), 0 if outs[0].dtype == torch.float32 else 1
    args.rows_per_batch, args.batch_stride_rows = rows_per_batch, batch_stride_rows
    grp = _lib.GemmGroup()
    grp.groups, grp.w_group_rows, grp.max_ctas = G, w.stride(0) // K, max_ctas
    grp.bias_group = bias.stride(0) if bias is not None else 0
    for g in range(G):
        assert outs[g].stride(0) == outs[0].stride(0) and outs[g].stride(1) == 1
        grp.out[g] = outs[g].data_ptr()
    if peer_ptrs:
        args.n_peer_out = len(peer_ptrs[0])
        for g in range(G):
            for r, ptr in enumerate(peer_ptrs[g]):
                grp.peer_out[g * 8 + r] = ptr
    _lib.check(_lib.lib().m3r_gemm_grouped(C.byref(args), C.byref(grp), _stream()), "gemm_grouped")


def normalize16(x: torch.Tensor, eps: float, dtype: torch.dtype, add: Optional[torch.Tensor] = None, add_rows: int = 0) -> torch.Tensor:
    """Affine-free LayerNorm of fp32 rows -> 16-bit; `add` [P, D] is added to rows < add_rows with period P."""
    _req_cuda(x)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    M, D = x.shape
    out = torch.empty((M, D), device=x.device, dtype=dtype)
    _lib.check(_lib.lib().m3r_normalize16(_p(x), x.stride(0), _p(add), add.stride(0) if add is not None else 0,
                                          add_rows, add.shape[0] if add is not None else 1, eps, M, D, _p(out), out.stride(0),
                                          F16[dtype], _stream()), "normalize16")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float, *, add: Optional[torch.Tensor] = None,
              out_dtype: torch.dtype = torch.float16) -> torch.Tensor:
    _req_cuda(x)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    M, D = x.shape
    out = torch.empty((M, D), device=x.device, dtype=out_dtype)
    _lib.check(_lib.lib().m3r_layernorm(_p(x), x.stride(0), _p(add), add.stride(0) if add is not None else 0,
                                        _p(gamma), _p(beta), eps, M, D, _p(out), out.stride(0),
                                        0 if out_dtype == torch.float32 else 1, F16.get(out_dtype, 0), _stream()),
               "layernorm")
    return out


def layernorm16(x16: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float) -> torch.Tensor:
    """LayerNorm of 16-bit rows -> 16-bit rows of the same format (memory_mode 'raw': norm_y applied at use)."""
    _req_cuda(x16)
    assert x16.dtype in F16 and x16.dim() == 2 and x16.stride(1) == 1
    M, D = x16.shape
    out = torch.empty((M, D), device=x16.device, dtype=x16.dtype)
    _lib.check(_lib.lib().m3r_layernorm16(_p(x16), x16.stride(0), _p(gamma), _p(beta), eps, M, D, _p(out), out.stride(0),
                                          F16[x16.dtype], _stream()), "layernorm16")
    return out


def cast16(x: torch.Tensor, dtype: torch.dtype, add: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 [M,D] (+ optional fp32 `add`) -> 16-bit."""
    _req_cuda(x)
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    out = torch.empty(x.shape, device=x.device, dtype=dtype)
    if add is None:
        _lib.check(_lib.lib().m3r_cast16(_p(x), x.stride(0), x.shape[0], x.shape[1], _p(out), out.stride(0), F16[dtype],
                                         _stream()), "cast16")
    else:
        assert add.dtype == torch.float32 and add.shape == x.shape and add.stride(1) == 1
        _lib.check(_lib.lib().m3r_add_cast16(_p(x), x.stride(0), _p(add), add.stride(0), x.shape[0], x.shape[1], _p(out),
                                             out.stride(0), F16[dtype], _stream()), "add_cast16")
    return out


def rope_table(pos: torch.Tensor, base: float, f0: float) -> torch.Tensor:
    """pos [T,2] int64 -> [T,64] fp32 (cosY,sinY,cosX,sinX)."""
    _req_cuda(pos)
    assert pos.dtype == torch.int64 and pos.shape[-1] == 2 and pos.is_contiguous()
    T = pos.numel() // 2
    tab = torch.empty((T, 64), device=pos.device, dtype=torch.float32)
    _lib.check(_lib.lib().m3r_rope_table(_p(pos), T, base, f0, _p(tab), _stream()), "rope_table")
    return tab


def rope_2d(tokens: torch.Tensor, positions: torch.Tensor, base: float, fwd: float) -> None:
    """curope.rope_2d drop-in (dust3r/croco/models/curope/curope.cpp:49-69): in-place on tokens [B,N,H,D]."""
    if tokens.dim() != 4:
        raise RuntimeError("tokens must have 4 dimensions")
    if positions.dim() != 3:
        raise RuntimeError("positions must have 3 dimensions")
    if tokens.size(0) != positions.size(0):
        raise RuntimeError("batch size differs between tokens & positions")
    if tokens.size(1) != positions.size(1):
        raise RuntimeError("seq_length differs between tokens & positions")
    if positions.size(2) != 2:
        raise RuntimeError("positions.shape[2] must be equal to 2")
    if positions.device != tokens.device:
        raise RuntimeError("tokens and positions are not on the same device")
    if positions.dtype != torch.int64:                    # curope reads them through data_ptr<int64_t>(), which throws
        raise RuntimeError(f"expected scalar type Long but found {positions.dtype} (positions must be int64)")
    _req_cuda(tokens, positions)
    if tokens.stride(3) != 1:
        raise RuntimeError("tokens are not contiguous")
    B, N, H, D = tokens.shape
    dt = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}[tokens.dtype]
    positions = positions.contiguous()
    _lib.check(_lib.lib().m3r_rope_2d(_p(tokens), dt, B, N, H, D, tokens.stride(0), tokens.stride(1), tokens.stride(2),
                                      _p(positions), base, fwd, _stream()), "rope_2d")


def attention(q: torch.Tensor, k0: torch.Tensor, v0: torch.Tensor, *, B: int, H: int, Nq: int, Nk0: int,
              kv_bstride0: Optional[int] = None, k1: Optional[torch.Tensor] = None, v1: Optional[torch.Tensor] = None,
              Nk1: int = 0, kv_bstride1: Optional[int] = None, kv_group: int = 1, skip_lo: int = 0, skip_step: int = 0,
              skip_len: int = 0, out: Optional[torch.Tensor] = None, export: bool = False):
    """q: 2-D view [B*Nq, >=H*64] (row stride arbitrary); k/v: 2-D views whose rows are keys.  Returns [B*Nq, H*64], or with
    export=True the unnormalised attention state (o [B*Nq, H*64] fp32, ml [B*Nq, H, 2] fp32) of this key set (attn_merge)."""
    _req_cuda(q, k0, v0)
    assert q.dtype in F16 and q.stride(-1) == 1 and k0.stride(-1) == 1 and v0.stride(-1) == 1
    assert k0.stride(0) == v0.stride(0)
    exp_o = exp_ml = None
    if export:
        exp_o = torch.empty((B * Nq, H * 64), device=q.device, dtype=torch.float32)
        exp_ml = torch.empty((B * Nq, H, 2), device=q.device, dtype=torch.float32)
    elif out is None:
        out = torch.empty((B * Nq, H * 64), device=q.device, dtype=q.dtype)
    a = _lib.AttnArgs()
    a.Q, a.ldq = q.data_ptr(), q.stride(0)
    a.K0, a.V0, a.ldk0, a.Nk0 = k0.data_ptr(), v0.data_ptr(), k0.stride(0), Nk0
    a.kv_bstride0 = Nk0 if kv_bstride0 is None else kv_bstride0
    if Nk1 > 0:
        assert k1.stride(0) == v1.stride(0)
        a.K1, a.V1, a.ldk1, a.Nk1 = k1.data_ptr(), v1.data_ptr(), k1.stride(0), Nk1
        a.kv_bstride1 = Nk1 if kv_bstride1 is None else kv_bstride1
    if export:
        a.export_o, a.export_ml, a.ldo = exp_o.data_ptr(), exp_ml.data_ptr(), H * 64
    else:
        a.O, a.ldo = out.data_ptr(), out.stride(0)
    a.B, a.H, a.Nq, a.kv_group = B, H, Nq, kv_group
    a.skip_lo, a.skip_step, a.skip_len = skip_lo, skip_step, skip_len
    a.is_bf16 = F16[q.dtype]
    a.scale = 0.125
    _lib.check(_lib.lib().m3r_attention(C.byref(a), _stream()), "attention")
    return (exp_o, exp_ml) if export else out


def attn_merge(states, dtype: torch.dtype) -> torch.Tensor:
    """Merge attention states [(o, ml), ...] of the same queries over disjoint key sets -> normalised [rows, H*64] 16-bit."""
    n = len(states)
    rows, HD = states[0][0].shape
    H = HD // 64
    out = torch.empty((rows, HD), device=states[0][0].device, dtype=dtype)
    po = (C.c_void_p * n)(*[o.data_ptr() for o, _ in states])
    pml = (C.c_void_p * n)(*[ml.data_ptr() for _, ml in states])
    _lib.check(_lib.lib().m3r_attn_merge(po, pml, n, rows, H, _p(out), out.stride(0), F16[dtype], _stream()), "attn_merge")
    return out


def attn_state_fill(rows: int, H: int, device) -> tuple:
    """The attention state of an empty key set: o = 0, m = -inf, l = 0."""
    o = torch.empty((rows, H * 64), device=device, dtype=torch.float32)
    ml = torch.empty((rows, H, 2), device=device, dtype=torch.float32)
    _lib.check(_lib.lib().m3r_attn_state_fill(_p(o), _p(ml), rows, H, _stream()), "attn_state_fill")
    return o, ml


def im2col16(img: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    _req_cuda(img)
    assert img.dtype == torch.float32 and img.is_contiguous() and img.dim() == 4 and img.shape[1] == 3
    V, _, H, W = img.shape
    out = torch.empty((V * (H // 16) * (W // 16), 768), device=img.device, dtype=dtype)
    _lib.check(_lib.lib().m3r_im2col16(_p(img), V, H, W, _p(out), F16[dtype], _stream()), "im2col16")
    return out


def unpatchify(proj: torch.Tensor, V: int, H: int, W: int, C_: int = 7) -> torch.Tensor:
    _req_cuda(proj)
    assert proj.dtype == torch.float32 and proj.is_contiguous()
    out = torch.empty((V, H, W, C_), device=proj.device, dtype=torch.float32)
    _lib.check(_lib.lib().m3r_unpatchify(_p(proj), V, H, W, C_, _p(out), _stream()), "unpatchify")
    return out


def _frames_u8(src: torch.Tensor):
    """uint8 [V,H,W,3] CUDA view with pixel stride 3 and channel stride 1 (any row pitch / frame stride)."""
    _req_cuda(src)
    if src.dtype != torch.uint8 or src.dim() != 4 or src.shape[3] != 3 or src.stride(3) != 1 or src.stride(2) != 3:
        raise ValueError(f"expected RGB uint8 frames [V,H,W,3] with interleaved channels, got {tuple(src.shape)} "
                         f"{src.dtype} strides {src.stride()}")
    return src.shape[0], src.shape[1], src.shape[2], src.stride(1), src.stride(0)


def resample_pil_u8(src: torch.Tensor, tables, xk: int, yk: int, out_hw, row0: int, rows: int, tmp: torch.Tensor,
                    crop, out: Optional[torch.Tensor] = None, out_u8: Optional[torch.Tensor] = None) -> None:
    """Pillow-exact resize of uint8 frames src [V,H,W,3] to out_hw, then ImgNorm of the crop box (x, y, w, h) into `out`
    [V,3,h,w] fp32 and/or the resized uint8 frames into `out_u8` [V,out_h,out_w,3].  tables: CUDA tensors whose first bytes
    are (x bounds, x weights, y bounds, y weights), int32 (engine/images.py builds them); tmp: uint8 scratch of at least
    V * rows * out_w * 3 bytes."""
    V, H, W, pitch, vstride = _frames_u8(src)
    _req_cuda(tmp, out, out_u8, *tables)
    oh, ow = out_hw
    assert tmp.numel() * tmp.element_size() >= V * rows * ow * 3
    if out is not None:
        assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (V, 3, crop[3], crop[2])
    if out_u8 is not None:
        assert out_u8.dtype == torch.uint8 and out_u8.is_contiguous() and tuple(out_u8.shape) == (V, oh, ow, 3)
    xb, xw, yb, yw = tables
    _lib.check(_lib.lib().m3r_resample_pil_u8(_p(src), pitch, vstride, V, H, W, _p(xb), _p(xw), xk, ow, _p(yb), _p(yw), yk,
                                              oh, row0, rows, _p(tmp), _p(out_u8), crop[0], crop[1], crop[2], crop[3],
                                              _p(out), _stream()), "resample_pil_u8")


def resize_aa_bilinear_u8(src: torch.Tensor, tables, xk: int, yk: int, out_hw, tmp: torch.Tensor, out: torch.Tensor) -> None:
    """Antialiased bilinear resize (torchvision Resize) of ImgNorm(src), src uint8 [V,H,W,3] (a crop view is fine), into
    out [V,3,out_h,out_w] fp32.  tables: (x bounds int32, x weights fp32, y bounds, y weights) CUDA tensors; tmp: scratch
    of at least V * 3 * H * out_w fp32."""
    V, H, W, pitch, vstride = _frames_u8(src)
    _req_cuda(tmp, out, *tables)
    oh, ow = out_hw
    assert tmp.numel() * tmp.element_size() >= V * 3 * H * ow * 4
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (V, 3, oh, ow)
    xb, xw, yb, yw = tables
    _lib.check(_lib.lib().m3r_resize_aa_bilinear_u8(_p(src), pitch, vstride, V, H, W, _p(xb), _p(xw), xk, ow, _p(yb), _p(yw),
                                                    yk, oh, _p(tmp), _p(out), _stream()), "resize_aa_bilinear_u8")


def pointgrid_keys(pts: torch.Tensor, bucket: Optional[torch.Tensor], inv_h: float) -> torch.Tensor:
    """Grid-index sort keys of pts [P,3] fp32 with int32 buckets [P] (None = all 0): [P] int64 (csrc/pointgrid.cu)."""
    _req_cuda(pts, bucket)
    assert pts.dtype == torch.float32 and pts.is_contiguous() and pts.shape[-1] == 3
    assert bucket is None or (bucket.dtype == torch.int32 and bucket.is_contiguous() and bucket.numel() == pts.shape[0])
    keys = torch.empty((pts.shape[0],), dtype=torch.int64, device=pts.device)
    _lib.check(_lib.lib().m3r_pointgrid_keys(_p(pts), _p(bucket), pts.shape[0], inv_h, _p(keys), _stream()), "pointgrid_keys")
    return keys


def pointgrid_query(queries: torch.Tensor, qbucket: Optional[torch.Tensor], pts: torch.Tensor, cell_keys: torch.Tensor,
                    cell_off: torch.Tensor, bucket_cells: torch.Tensor, h: float, inv_h: float) -> torch.Tensor:
    """Distance from each query [Q,3] fp32 to the nearest indexed point of its bucket (int32 [Q], None = all 0): [Q] fp32,
    inf for an empty bucket.  The index tensors are those m3r_pointgrid_query documents (engine/keyframes.py builds them)."""
    _req_cuda(queries, qbucket, pts, cell_keys, cell_off, bucket_cells)
    assert queries.dtype == torch.float32 and queries.is_contiguous() and queries.shape[-1] == 3
    assert qbucket is None or (qbucket.dtype == torch.int32 and qbucket.is_contiguous() and qbucket.numel() == queries.shape[0])
    assert cell_keys.dtype == torch.int64 and cell_off.dtype == torch.int32 and bucket_cells.dtype == torch.int32
    out = torch.empty((queries.shape[0],), dtype=torch.float32, device=queries.device)
    _lib.check(_lib.lib().m3r_pointgrid_query(_p(queries), _p(qbucket), queries.shape[0], _p(pts), pts.shape[0], _p(cell_keys),
                                              _p(cell_off), cell_keys.shape[0], _p(bucket_cells), bucket_cells.shape[0] - 1,
                                              h, inv_h, _p(out), _stream()), "pointgrid_query")
    return out


def postprocess_raw(pm: torch.Tensor):
    _req_cuda(pm)
    assert pm.dtype == torch.float32 and pm.shape[-1] == 7
    pm = pm.contiguous()
    P = pm.numel() // 7
    pts = torch.empty(pm.shape[:-1] + (3,), device=pm.device, dtype=torch.float32)
    loc = torch.empty_like(pts)
    conf = torch.empty(pm.shape[:-1], device=pm.device, dtype=torch.float32)
    _lib.check(_lib.lib().m3r_postprocess(_p(pm), P, _p(pts), _p(loc), _p(conf), _stream()), "postprocess")
    return pts, loc, conf


# m3r_slam_record (include/must3r_b200.h): one view's camera and keyframe test, as a host numpy record
SLAM_RECORD = np.dtype([("c2w", "<f4", (4, 4)), ("w2c", "<f4", (4, 4)), ("focal", "<f4"), ("conf_mean", "<f4"),
                        ("conf_median", "<f4"), ("n_conf", "<i4"), ("score", "<f8"), ("keyframe", "<i4"),
                        ("reserved", "<i4")])


def overlap_mode_id(mode: str) -> int:
    """must3r/slam/model.py:72-90: 'meanconf', 'medianconf', or any mode containing 'nn' ('norm' divides by the depth)."""
    if mode == "meanconf":
        return 2
    if mode == "medianconf":
        return 3
    if "nn" in mode:
        return 1 if "norm" in mode else 0
    raise ValueError(f"Unknown overlap score method {mode}")


def slam_record_c2w(rec: torch.Tensor) -> torch.Tensor:
    """Device view [B,4,4] fp32 of the c2w field of records [B, SLAM_RECORD.itemsize] uint8."""
    return rec[:, :64].view(torch.float32).view(-1, 4, 4)


def slam_pose(pts3d: torch.Tensor, pts3d_local: torch.Tensor, conf: torch.Tensor, seq_focal: Optional[float] = None,
              is_first: bool = False, rec: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Focal, pose and confidence statistics of B views (csrc/slam.cu): pts3d, pts3d_local [B,H,W,3], conf [B,H,W] fp32
    contiguous.  Unless is_first, pts3d_local's z is scaled in place by seq_focal / focal when seq_focal is given.
    Returns the records [B, SLAM_RECORD.itemsize] uint8 on the device (or fills `rec`)."""
    _req_cuda(pts3d, pts3d_local, conf)
    for t in (pts3d, pts3d_local, conf):
        assert t.dtype == torch.float32 and t.is_contiguous()
    B, H, W = conf.shape
    assert pts3d.shape == (B, H, W, 3) and pts3d_local.shape == (B, H, W, 3)
    if rec is None:
        rec = torch.empty((B, SLAM_RECORD.itemsize), dtype=torch.uint8, device=conf.device)
    assert rec.shape == (B, SLAM_RECORD.itemsize) and rec.is_contiguous()
    _lib.check(_lib.lib().m3r_slam_pose(_p(pts3d), _p(pts3d_local), _p(conf), B, H, W, W / 2, H / 2,
                                        int(seq_focal is not None), 0.0 if seq_focal is None else float(seq_focal),
                                        int(bool(is_first)), _p(rec), _stream()), "slam_pose")
    return rec


def slam_pose_views(pts3d: torch.Tensor, pts3d_local: torch.Tensor, conf: torch.Tensor, seq_focals, is_first,
                    rec: Optional[torch.Tensor] = None) -> torch.Tensor:
    """slam_pose over B <= 64 views with one (seq_focal or None, is_first) per view, e.g. the frames of several cameras
    with their own agents' focals (csrc/slam.cu m3r_slam_pose_views): each record is bitwise slam_pose's for that view
    alone."""
    _req_cuda(pts3d, pts3d_local, conf)
    for t in (pts3d, pts3d_local, conf):
        assert t.dtype == torch.float32 and t.is_contiguous()
    B, H, W = conf.shape
    assert pts3d.shape == (B, H, W, 3) and pts3d_local.shape == (B, H, W, 3)
    assert len(seq_focals) == B and len(is_first) == B
    if rec is None:
        rec = torch.empty((B, SLAM_RECORD.itemsize), dtype=torch.uint8, device=conf.device)
    assert rec.shape == (B, SLAM_RECORD.itemsize) and rec.is_contiguous()
    has = (C.c_int32 * B)(*[int(f is not None) for f in seq_focals])
    foc = (C.c_float * B)(*[0.0 if f is None else float(f) for f in seq_focals])
    first = (C.c_int32 * B)(*[int(bool(x)) for x in is_first])
    _lib.check(_lib.lib().m3r_slam_pose_views(_p(pts3d), _p(pts3d_local), _p(conf), B, H, W, W / 2, H / 2, has, foc, first,
                                              _p(rec), _stream()), "slam_pose_views")
    return rec


def slam_keyframe_frames(dists: Optional[torch.Tensor], conf: torch.Tensor, pts3d_local: torch.Tensor, rec: torch.Tensor,
                         *, subsamp: Optional[int], mode: str, percentile: float, thr: float, min_conf_keyframe: float,
                         is_first) -> torch.Tensor:
    """slam_keyframe of F <= 64 frames in one launch (csrc/slam.cu m3r_slam_keyframe_frames): conf [F,H,W], pts3d_local
    [F,H,W,3] fp32 contiguous, dists [F, Q] (None for the conf modes), rec [F, SLAM_RECORD.itemsize], is_first F flags;
    each record is bitwise slam_keyframe's for that frame alone."""
    _req_cuda(dists, conf, pts3d_local, rec)
    F, H, W = conf.shape
    s = int(subsamp) if subsamp else 1
    m = overlap_mode_id(mode)
    assert conf.dtype == torch.float32 and conf.is_contiguous()
    assert pts3d_local.dtype == torch.float32 and pts3d_local.is_contiguous() and pts3d_local.shape == (F, H, W, 3)
    if m <= 1:
        assert dists is not None and dists.dtype == torch.float32 and dists.is_contiguous()
        assert dists.numel() == F * ((H + s - 1) // s) * ((W + s - 1) // s)
    assert rec.shape == (F, SLAM_RECORD.itemsize) and rec.is_contiguous() and len(is_first) == F
    first = (C.c_int32 * F)(*[int(bool(x)) for x in is_first])
    _lib.check(_lib.lib().m3r_slam_keyframe_frames(_p(dists) if m <= 1 else None, _p(conf), _p(pts3d_local), F, H, W, s, m,
                                                   float(percentile), float(thr), float(min_conf_keyframe), first, _p(rec),
                                                   _stream()), "slam_keyframe_frames")
    return rec


SCENE_VIEW = np.dtype([("pts3d", "<u8"), ("c2w", "<u8"), ("conf", "<u8"), ("img", "<u8"), ("H", "<i4"), ("W", "<i4"),
                       ("first_tile", "<i8")])           # m3r_scene_view
SCENE_TILE = 1024
SCENE_MAX_THR = 8


def scene_points(pts3d, conf, imgs, thresholds, c2w=None, out=None):
    """Point clouds of V views at T <= 8 confidence thresholds in one pass over the views (csrc/scene.cu).

    pts3d: V fp32 [H,W,3] (world points; local points when c2w, V fp32 [4,4] camera-to-world, is given), conf: V fp32
    [H,W], imgs: V fp32 [3,H,W] ImgNorm images, all contiguous CUDA tensors; views may differ in H x W.  Threshold t
    keeps the pixels with conf >= thresholds[t] (never a NaN conf), view after view in raster order.
    Returns (pts [N,3], col [N,3], counts): N = sum(counts), threshold t's points are rows sum(counts[:t]) onwards, col
    is clip(img * 0.5 + 0.5, 0, 1).  counts (host ints) are read back once to size the outputs.  out = (pts, col) fp32
    CUDA buffers of at least N rows receives the points instead; rows past N are not written."""
    V = len(conf)
    T = len(thresholds)
    if V < 1 or len(pts3d) != V or len(imgs) != V or (c2w is not None and len(c2w) != V):
        raise ValueError(f"scene_points: {len(pts3d)} pointmaps, {V} confidence maps, {len(imgs)} images")
    if not 1 <= T <= SCENE_MAX_THR:
        raise ValueError(f"scene_points: {T} thresholds (1..{SCENE_MAX_THR})")
    dev = conf[0].device
    table = np.zeros(V, dtype=SCENE_VIEW)
    first = 0
    for v in range(V):
        p, c, im = pts3d[v], conf[v], imgs[v]
        m = None if c2w is None else c2w[v]
        _req_cuda(p, c, im, m)
        H, W = c.shape
        for t, shape in ((p, (H, W, 3)), (c, (H, W)), (im, (3, H, W))) + (() if m is None else ((m, (4, 4)),)):
            if t.dtype != torch.float32 or not t.is_contiguous() or tuple(t.shape) != shape or t.device != dev:
                raise ValueError(f"scene_points: view {v}: expected contiguous fp32 {shape} on {dev}, got "
                                 f"{t.dtype} {tuple(t.shape)} on {t.device}")
        if H * W == 0:
            raise ValueError(f"scene_points: view {v} is empty")
        table[v] = (p.data_ptr(), 0 if m is None else m.data_ptr(), c.data_ptr(), im.data_ptr(), H, W, first)
        first += (H * W + SCENE_TILE - 1) // SCENE_TILE
    n_tiles = first
    views = torch.from_numpy(table.view(np.uint8)).pin_memory().to(dev, non_blocking=True)
    thr = torch.tensor([float(t) for t in thresholds], dtype=torch.float32).pin_memory().to(dev, non_blocking=True)
    tile_counts = torch.empty((T, n_tiles), dtype=torch.int32, device=dev)
    tile_off = torch.empty((T, n_tiles), dtype=torch.int64, device=dev)
    counts = torch.empty((T,), dtype=torch.int64, device=dev)
    _lib.check(_lib.lib().m3r_scene_count(_p(views), V, _p(thr), T, n_tiles, _p(tile_counts), _p(tile_off), _p(counts),
                                          _stream()), "scene_count")
    host = torch.empty((T,), dtype=torch.int64, pin_memory=True)
    host.copy_(counts, non_blocking=True)
    torch.cuda.current_stream(dev).synchronize()
    n = [int(v) for v in host.tolist()]
    total = sum(n)
    if out is None:
        pts = torch.empty((total, 3), dtype=torch.float32, device=dev)
        col = torch.empty((total, 3), dtype=torch.float32, device=dev)
    else:
        pts, col = out
        _req_cuda(pts, col)
        for b in (pts, col):
            if b.dtype != torch.float32 or not b.is_contiguous() or b.dim() != 2 or b.shape[1] != 3 or b.shape[0] < total:
                raise ValueError(f"scene_points: out buffers must be contiguous fp32 [>= {total}, 3]")
    if total:
        _lib.check(_lib.lib().m3r_scene_points(_p(views), V, _p(thr), T, n_tiles, _p(tile_off), _p(counts), _p(pts), _p(col),
                                               _stream()), "scene_points")
    return pts[:total], col[:total], n


def slam_keyframe(dists: Optional[torch.Tensor], conf: torch.Tensor, pts3d_local: torch.Tensor, rec: torch.Tensor, *,
                  subsamp: Optional[int], mode: str, percentile: float, thr: float, min_conf_keyframe: float,
                  is_first: bool) -> torch.Tensor:
    """Overlap score and keyframe decision of one view into its record rec [1, SLAM_RECORD.itemsize] (csrc/slam.cu).
    conf [H,W], pts3d_local [H,W,3] fp32 contiguous; dists = the distances of every subsampled pixel (::subsamp in both
    axes, row-major; None for the conf modes)."""
    _req_cuda(dists, conf, pts3d_local, rec)
    H, W = conf.shape
    s = int(subsamp) if subsamp else 1
    m = overlap_mode_id(mode)
    assert conf.dtype == torch.float32 and conf.is_contiguous()
    assert pts3d_local.dtype == torch.float32 and pts3d_local.is_contiguous() and pts3d_local.shape == (H, W, 3)
    if m <= 1:
        assert dists is not None and dists.dtype == torch.float32 and dists.is_contiguous()
        assert dists.numel() == ((H + s - 1) // s) * ((W + s - 1) // s)
    assert rec.shape[-1] == SLAM_RECORD.itemsize and rec.is_contiguous()
    _lib.check(_lib.lib().m3r_slam_keyframe(_p(dists) if m <= 1 else None, _p(conf), _p(pts3d_local), H, W, s, m,
                                            float(percentile), float(thr), float(min_conf_keyframe), int(bool(is_first)),
                                            _p(rec), _stream()), "slam_keyframe")
    return rec


# ------------------------------------------------------------------------------------------- baseline JPEG decoding
def jpeg_parse(data: bytes) -> "_lib.JpegInfo":
    """Header facts of a JPEG held in memory (m3r_jpeg_parse); info.eligible says whether jpeg_decode takes it.  A file
    that is not a JPEG comes back with eligible == 0."""
    info = _lib.JpegInfo()
    _lib.lib().m3r_jpeg_parse(data, len(data), C.byref(info))
    return info


def jpeg_prepare(data: bytes, info, orientation: int, dst_ptr: int, base_off: int) -> Optional["_lib.JpegDesc"]:
    """Tables, restart segments and unstuffed entropy-coded data of one image written at host address dst_ptr
    (info.prep_bytes bytes); the descriptor, or None when the data makes the file ineligible after all."""
    desc = _lib.JpegDesc()
    rc = _lib.lib().m3r_jpeg_prepare(data, len(data), C.byref(info), orientation, C.c_void_p(dst_ptr), base_off,
                                     C.byref(desc))
    if rc == 2:
        return None
    _lib.check(rc, "jpeg_prepare")
    return desc


def jpeg_plan(descs) -> int:
    """Fill the batch fields of a ctypes array of JpegDesc; returns the workspace bytes jpeg_decode needs."""
    n = _lib.lib().m3r_jpeg_plan(descs, len(descs))
    if n < 0:
        _lib.check(1, "jpeg_plan")
    return n


def jpeg_decode(descs, dev_blob: torch.Tensor, descs_off: int, work: torch.Tensor, status: torch.Tensor) -> None:
    """Decode a planned batch on the current stream; status [n] int32 gets each image's M3R_JPEG_E* bits."""
    _req_cuda(dev_blob, work, status)
    assert status.dtype == torch.int32 and status.numel() >= len(descs)
    _lib.check(_lib.lib().m3r_jpeg_decode(descs, len(descs), _p(dev_blob), descs_off, _p(work), work.numel(), _p(status),
                                          _stream()), "jpeg_decode")


# ------------------------------------------------------------------------------------------- PNG decoding
def png_parse(data: bytes) -> "_lib.PngInfo":
    """Chunk facts of a PNG held in memory (m3r_png_parse); info.eligible says whether png_decode takes it.  A file that
    is not a PNG comes back with eligible == 0."""
    info = _lib.PngInfo()
    _lib.lib().m3r_png_parse(data, len(data), C.byref(info))
    return info


def png_prepare(data: bytes, info, orientation: int, dst_ptr: int, base_off: int) -> "_lib.PngDesc":
    """Palette and concatenated IDAT payloads of one eligible image written at host address dst_ptr (info.prep_bytes
    bytes); its descriptor."""
    desc = _lib.PngDesc()
    _lib.check(_lib.lib().m3r_png_prepare(data, len(data), C.byref(info), orientation, C.c_void_p(dst_ptr), base_off,
                                          C.byref(desc)), "png_prepare")
    return desc


def png_plan(descs) -> int:
    """Fill the workspace fields of a ctypes array of PngDesc; returns the workspace bytes png_decode needs."""
    n = _lib.lib().m3r_png_plan(descs, len(descs))
    if n < 0:
        _lib.check(1, "png_plan")
    return n


def png_decode(descs, dev_blob: torch.Tensor, descs_off: int, work: torch.Tensor, status: torch.Tensor) -> None:
    """Decode a planned batch on the current stream; status [n] int32 gets each image's M3R_PNG_E* bits."""
    _req_cuda(dev_blob, work, status)
    assert status.dtype == torch.int32 and status.numel() >= len(descs)
    _lib.check(_lib.lib().m3r_png_decode(descs, len(descs), _p(dev_blob), descs_off, _p(work), work.numel(), _p(status),
                                         _stream()), "png_decode")
