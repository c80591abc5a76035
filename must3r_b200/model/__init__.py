"""Model API of the reference (must3r/model/__init__.py): load_model, Dust3rEncoder, MUSt3R, CausalMUSt3R,
ActivationType, apply_activation, get_pointmaps_activation, get_dtype - backed by the sm_90a kernels."""
from __future__ import annotations

import re
from functools import partial  # noqa: F401  (constructor strings in checkpoints use it)

import torch
import torch.nn as nn  # noqa: F401

from .common import ActivationType, set_precision, get_precision  # noqa: F401
from .encoder import Dust3rEncoder  # noqa: F401
from .decoder import MUSt3R, CausalMUSt3R, MEMORY_MODES  # noqa: F401


def apply_activation(xyz, activation):
    """must3r/model/blocks/head.py:13-21 (+ must3r/tools/geometry.py:14-18)"""
    if isinstance(activation, str):
        activation = ActivationType(activation)
    if activation == ActivationType.NORM_EXP:
        d = xyz.norm(dim=-1, keepdim=True)
        return xyz / d.clip(min=1e-8) * torch.expm1(d)
    elif activation == ActivationType.LINEAR:
        return xyz
    raise ValueError(f"Unknown activation: {activation}")


def get_pointmaps_activation(decoder, verbose=True):
    """Activation the decoder's pointmaps expect; NORM_EXP for decoders that do not say (must3r/model/__init__.py:8-15)."""
    act = getattr(decoder, "pointmaps_activation", ActivationType.NORM_EXP)
    if verbose:
        print(f"pointmaps_activation set to {act}")
    return act


_AMP_DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}


def get_dtype(amp):
    """'fp16' / 'bf16' / falsy -> torch dtype (must3r/model/__init__.py:18-27)."""
    if amp in _AMP_DTYPES:
        return _AMP_DTYPES[amp]
    assert not amp
    return torch.float32


def convert_decoder_args(decoder_args):
    """Constructor string of a training checkpoint -> inference decoder (must3r/model/__init__.py:53-63): the causal training
    class becomes MUSt3R and the head is told not to assume landscape inputs."""
    text = "".join(decoder_args.split(" "))
    text = text.replace("CausalMUSt3R", "MUSt3R").replace("landscape_only=True", "landscape_only=False")
    if "landscape_only=False" in text:
        return text
    return f"{text[:-1]},landscape_only=False)"


_IMG_SIZE_RE = re.compile(r"img_size=\((\d+),(\d+)\)")
_POS_EMBED_RE = re.compile(r"pos_embed='([A-Za-z]+)(\d+)(?:_(\d+):(\d+))?'")


def set_image_size_in_args(model_args, img_size, verbose=True):
    """Point a constructor string at another (square) img_size and rename the adaptive RoPE accordingly
    (must3r/model/__init__.py:66-108): 'RoPE100' trained at 512 and run at 768 becomes 'RoPE100_512:768'; an existing
    '<name><freq>_<base>:<cur>' keeps its base; a string without pos_embed gets one appended."""
    text = "".join(model_args.split(" "))
    size = _IMG_SIZE_RE.search(text)
    if size is None:
        raise ValueError("No image_size tuple found in model args")
    side, other = (int(v) for v in size.groups())
    assert side == other
    rope = _POS_EMBED_RE.search(text)
    name, freq = (rope.group(1), int(rope.group(2))) if rope else ("RoPE", 100)
    adaptive = rope is not None and rope.group(3) is not None
    base, current = (int(rope.group(3)), int(rope.group(4))) if adaptive else (side, side)
    if verbose:
        print(f"image_size {side} -> {img_size}; pos_embed {name}{freq} (base size {base})")
    if img_size != side:
        text = text.replace(f"img_size=({side},{side})", f"img_size=({img_size},{img_size})")
    if img_size == current:
        return text
    renamed = f"pos_embed='{name}{freq}_{base}:{img_size}'"
    if rope is None:
        return f"{text[:-1]},{renamed})"
    return text[:rope.start()] + renamed + text[rope.end():]


def load_model(chkpt_path, encoder=None, decoder=None, device='cuda', img_size=None, memory_mode=None, verbose=True):
    """must3r/model/__init__.py:30-50: checkpoint {'args': Namespace(encoder=str, decoder=str), 'encoder': sd,
    'decoder': sd}; the constructor strings are evaluated against this package's classes."""
    ckpt = torch.load(chkpt_path, map_location='cpu', weights_only=False)
    encoder_args = encoder or ckpt['args'].encoder
    decoder_args = decoder or convert_decoder_args(ckpt['args'].decoder)
    if img_size is not None:
        encoder_args = set_image_size_in_args(encoder_args, img_size, verbose=verbose)
        decoder_args = set_image_size_in_args(decoder_args, img_size, verbose=verbose)
    scope = {"Dust3rEncoder": Dust3rEncoder, "MUSt3R": MUSt3R, "CausalMUSt3R": CausalMUSt3R, "partial": partial,
             "nn": nn, "torch": torch, "ActivationType": ActivationType}
    enc = eval(encoder_args, scope)
    dec = eval(decoder_args, scope)
    if memory_mode is not None:
        dec.change_memory_mode(memory_mode)
    enc.load_state_dict(ckpt['encoder'], strict=True)
    dec.load_state_dict(ckpt['decoder'], strict=True)
    enc.to(device)
    dec.to(device)
    enc.eval()
    dec.eval()
    return enc, dec
