"""ctypes mirrors of the weight structs of include/must3r_b200.h + helpers shared by encoder / decoder."""
from __future__ import annotations

import ctypes as C
from enum import Enum
from typing import Optional

import torch
import torch.nn as nn

from .. import _lib

vp, fp = C.c_void_p, C.c_void_p


class EncBlock(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "norm1_w", "norm1_b", "qkv_w", "qkv_b", "proj_w", "proj_b", "norm2_w", "norm2_b",
        "fc1_w", "fc1_b", "fc2_w", "fc2_b")]


class EncoderWeights(C.Structure):
    _fields_ = [("embed_dim", C.c_int32), ("depth", C.c_int32), ("num_heads", C.c_int32), ("mlp_hidden", C.c_int32),
                ("ln_eps", C.c_float), ("rope_base", C.c_float), ("rope_f0", C.c_float), ("is_bf16", C.c_int32),
                ("patch_w", C.c_void_p), ("patch_b", C.c_void_p), ("blocks", C.POINTER(EncBlock)),
                ("norm_w", C.c_void_p), ("norm_b", C.c_void_p)]


class DecBlock(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "a_w", "a_b", "proj_w", "proj_b", "q_w", "q_b", "cproj_w", "cproj_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b",
        "normy_w", "normy_b", "kv_w", "kv_b")]


class DecoderWeights(C.Structure):
    _fields_ = [("enc_dim", C.c_int32), ("embed_dim", C.c_int32), ("depth", C.c_int32), ("num_heads", C.c_int32),
                ("mlp_hidden", C.c_int32), ("out_dim", C.c_int32),
                ("ln_eps", C.c_float), ("fb_ln_eps", C.c_float), ("rope_base", C.c_float), ("rope_f0", C.c_float),
                ("is_bf16", C.c_int32), ("feedback", C.c_int32),
                ("embed_w", C.c_void_p), ("embed_b", C.c_void_p), ("image2_embed", C.c_void_p),
                ("blocks", C.POINTER(DecBlock)),
                ("fb1_w", C.c_void_p), ("fb1_b", C.c_void_p), ("fb2_w", C.c_void_p), ("fb2_b", C.c_void_p),
                ("head_w", C.c_void_p), ("head_b", C.c_void_p)]


class EncBlockE4M3(C.Structure):
    _fields_ = [("qkv_s", C.c_void_p), ("fc1_s", C.c_void_p)]


class DecBlockE4M3(C.Structure):
    _fields_ = [("a_s", C.c_void_p), ("q_s", C.c_void_p), ("fc1_s", C.c_void_p)]


class DecoderE4M3(C.Structure):
    _fields_ = [("blocks", C.POINTER(DecBlockE4M3)), ("fb1_s", C.c_void_p)]


class DecGroup(C.Structure):
    _fields_ = [("n_views", C.c_int32), ("N", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
                ("x_enc", C.c_void_p), ("pos", C.c_void_p), ("pointmaps", C.c_void_p)]


class DecoderCall(C.Structure):
    _fields_ = [("B", C.c_int32), ("G", C.c_int32), ("groups", C.POINTER(DecGroup)), ("Nm", C.c_int32),
                ("mem", C.POINTER(C.c_void_p)), ("mem_bstride_rows", C.c_int64), ("render", C.c_int32),
                ("is_init", C.c_int32), ("mem_out", C.POINTER(C.c_void_p)), ("mem_out_bstride_rows", C.c_int64),
                ("new_only", C.c_int32), ("n_peers", C.c_int32), ("peer_mem", C.POINTER(C.c_void_p)),
                ("mem_mode", C.c_int32),
                ("cp_world", C.c_int32), ("cp_rank", C.c_int32), ("cp_owner", C.c_int32),
                ("cp_stage", C.POINTER(C.c_void_p)), ("cp_slot_bytes", C.c_int64),
                ("cp_flag_slots", C.POINTER(C.c_void_p)), ("cp_flags_local", C.c_void_p), ("cp_epoch0", C.c_uint32)]


MEM_MODE_CODE = {"kv": 0, "norm_y": 1, "raw": 2}        # M3R_MEM_* (must3r/model/blocks/layers.py:9)


_lib.SIGNATURES.update({
    "m3r_encoder_workspace_bytes": (C.c_int64, [C.POINTER(EncoderWeights), C.c_int32, C.c_int32, C.c_int32]),
    "m3r_encoder_forward": (C.c_int, [C.POINTER(EncoderWeights), C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_decoder_workspace_bytes": (C.c_int64, [C.POINTER(DecoderWeights), C.POINTER(DecoderCall)]),
    "m3r_decoder_cp_slot_bytes": (C.c_int64, [C.POINTER(DecoderWeights), C.c_int64]),
    "m3r_decoder_forward": (C.c_int, [C.POINTER(DecoderWeights), C.POINTER(DecoderCall), C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_decoder_forward_ragged": (C.c_int, [C.POINTER(DecoderWeights), C.POINTER(DecoderCall), C.c_void_p, C.c_void_p,
                                             C.c_int64, C.c_void_p]),
    "m3r_encoder_forward_e4m3": (C.c_int, [C.POINTER(EncoderWeights), C.POINTER(EncBlockE4M3), C.c_void_p, C.c_int32, C.c_int32,
                                           C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_decoder_forward_e4m3": (C.c_int, [C.POINTER(DecoderWeights), C.POINTER(DecoderE4M3), C.POINTER(DecoderCall), C.c_void_p,
                                           C.c_void_p, C.c_int64, C.c_void_p]),
    "m3r_decoder_render_ragged": (C.c_int, [C.POINTER(DecoderWeights), C.POINTER(DecoderE4M3), C.POINTER(DecoderCall),
                                            C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
})

_lib.apply_signatures()

# ------------------------------------------------------------------------------------------------ precision
_PRECISION = {"dtype": torch.float16}


def set_precision(dtype) -> None:
    """Storage format of GEMM / attention operands and of the K|V memory.

    ``torch.float16`` (default): 10-bit mantissa, i.e. the precision class of the TF32 matmuls the
    reference's demos enable (demo.py:12) - the parity mode.  ``torch.bfloat16``: the amp dtype of the
    reference's decoder (`--amp bf16`).  Both run at the same tensor-core rate; accumulation, LayerNorm, softmax
    and the residual stream are fp32 either way.

    ``torch.float8_e4m3fn`` (or ``"fp8"``): a speed mode.  The linear layers fed by a LayerNorm (encoder qkv and fc1;
    decoder qkv, cross-attention projq, the memory projk|projv, fc1 and the feedback fc1) multiply e4m3 operands on the
    FP8 tensor cores: the normalised rows need no scale (|y| <= sqrt(D - 1)) and each weight row has one fp32 scale.
    Everything else - the other linear layers, attention, the K|V memory (``MUSt3R.memory_dtype()``) - runs as in
    ``bfloat16``.  Measured speed and error: README.md, "FP8 mode"."""
    if isinstance(dtype, str):
        dtype = {"fp16": torch.float16, "float16": torch.float16, "bf16": torch.bfloat16, "bfloat16": torch.bfloat16,
                 "fp8": torch.float8_e4m3fn, "float8_e4m3fn": torch.float8_e4m3fn}[dtype]
    assert dtype in (torch.float16, torch.bfloat16, torch.float8_e4m3fn)
    _PRECISION["dtype"] = dtype


def get_precision() -> torch.dtype:
    return _PRECISION["dtype"]


def is_fp8(dtype) -> bool:
    return dtype == torch.float8_e4m3fn


def operand16(dtype) -> torch.dtype:
    """The 16-bit format of the operands, outputs and memory of precision `dtype` (bf16 in the fp8 mode)."""
    return torch.bfloat16 if is_fp8(dtype) else dtype


class ActivationType(Enum):
    """must3r/model/blocks/head.py:8-10"""
    NORM_EXP = "norm_exp"
    LINEAR = "linear"


def parse_pos_embed(name: str):
    """must3r/model/blocks/pos_embed.py:7-22"""
    assert name.startswith("RoPE")
    f0 = 1.0
    if "_" in name:
        name, res = name.split("_")
        old, new = res.split(":")
        f0 = float(old) / float(new)
    return float(name[len("RoPE"):]), f0


class Mlp(nn.Module):
    """Parameter container with the key names of dust3r/croco/models/blocks.py:58-72 (fc1, fc2)."""

    def __init__(self, dim, hidden, out=None):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, out or dim)


class AttnParams(nn.Module):
    """Key names of must3r/model/blocks/attention.py:82-90 (qkv, proj)."""

    def __init__(self, dim):
        super().__init__()
        self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)


class CrossAttnParams(nn.Module):
    """Key names of must3r/model/blocks/attention.py:102-112 (projq, projk, projv, proj)."""

    def __init__(self, dim):
        super().__init__()
        self.projq = nn.Linear(dim, dim)
        self.projk = nn.Linear(dim, dim)
        self.projv = nn.Linear(dim, dim)
        self.proj = nn.Linear(dim, dim)


def init_like_reference(module: nn.Module) -> None:
    """BaseTransformer._init_weights (must3r/model/blocks/layers.py:23-33): xavier Linear, zero bias, LN (1,0)."""
    for m in module.modules():
        if isinstance(m, nn.Linear):
            nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.constant_(m.bias, 0)
        elif isinstance(m, nn.LayerNorm):
            nn.init.constant_(m.bias, 0)
            nn.init.constant_(m.weight, 1.0)


class WeightPack:
    """Device-resident kernel-format copies of a module's parameters (16-bit matrices, fp32 vectors)."""

    def __init__(self):
        self.keep = []

    def mat(self, t: torch.Tensor, dtype) -> int:
        x = t.detach().reshape(t.shape[0], -1).to(dtype).contiguous()
        self.keep.append(x)
        return x.data_ptr()

    def folded(self, lin_w: torch.Tensor, lin_b: Optional[torch.Tensor], gamma: torch.Tensor, beta: torch.Tensor):
        """Linear(LayerNorm(x)) with the affine moved into the Linear: W' = W diag(gamma), b' = b + W beta (fp32 maths;
        W' is rounded to the 16-bit operand format once, exactly like W would be).  -> (W' fp32 [N,K], b' fp32 [N])"""
        w = lin_w.detach().float()
        b = w @ beta.detach().float()
        if lin_b is not None:
            b = b + lin_b.detach().float()
        return w * gamma.detach().float()[None, :], b

    def mat8(self, w: torch.Tensor):
        """e4m3 copy of a [N, K] weight with one fp32 scale per row (output channel): scale = amax / 448 (1 for an
        all-zero row), W8 = round_e4m3(W / scale) with torch.float8_e4m3fn's round-to-nearest-even.  -> (W8 ptr, scale ptr)"""
        q, s = quantize_e4m3_rows(w)
        self.keep += [q, s]
        return q.data_ptr(), s.data_ptr()

    def vec(self, t: Optional[torch.Tensor]) -> Optional[int]:
        if t is None:
            return None
        x = t.detach().float().contiguous().reshape(-1)
        self.keep.append(x)
        return x.data_ptr()


E4M3_MAX = 448.0


def quantize_e4m3_rows(w: torch.Tensor):
    """(W8 [N, K] float8_e4m3fn, scale [N] fp32) with W ~= W8 * scale[:, None] (see WeightPack.mat8)."""
    w = w.detach().reshape(w.shape[0], -1).float()
    amax = w.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    q = (w / scale[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).contiguous()
    return q, scale.contiguous()


_WS = {}


def workspace(device: torch.device, nbytes: int, tag: str) -> torch.Tensor:
    """Grow-only scratch buffer per (device, current stream, tag): kernels of one stream are ordered, so reuse is safe;
    two host threads driving the model on their own streams (the reference's SLAM worker, slam.py:533) get their own."""
    key = (str(device), int(torch.cuda.current_stream(device).cuda_stream), tag)
    buf = _WS.get(key)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(int(nbytes * 1.25) + 1024, dtype=torch.uint8, device=device)
        _WS[key] = buf
    return buf


def stream_ptr(device=None) -> C.c_void_p:
    """The caller's current stream ON THE TENSORS' DEVICE (not on whatever device happens to be current)."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
