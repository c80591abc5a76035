"""Attention seam of the reference (must3r/model/blocks/attention.py:5-79) on the wgmma kernel.

``toggle_memory_efficient_attention`` / ``is_memory_efficient_attention_enabled`` / ``has_xformers`` keep the names
callers flip at start-up (must3r/demo/gradio.py, must3r/slam/slam.py, eval.py call ``toggle_memory_efficient_attention``):
here they only record the flag - there is one attention backend, the sm_90a kernel, and no xFormers dependency.
``attention(q, k, v)`` has the calling convention of ``CoreAttention.attention`` after RoPE (:37,:66-79): ``[B,H,N,64]``
16-bit CUDA tensors in, ``[B,Nq,H*64]`` out; it is what the one-line patch of INTEGRATION.md §4 calls.
"""
import torch

from .. import ops

has_xformers = False
has_scaled_dot_product_attention = True
_use_memory_efficient_attention = False


def toggle_memory_efficient_attention(enabled: bool = True):
    global _use_memory_efficient_attention
    _use_memory_efficient_attention = enabled


def is_memory_efficient_attention_enabled():
    return _use_memory_efficient_attention


def attention(q, k, v, attn_mask=None):
    """softmax(q k^T / 8) v for [B,H,N,64] fp16/bf16 CUDA tensors -> [B,Nq,H*64] (heads merged like attention.py:75)."""
    if attn_mask is not None:
        raise NotImplementedError("boolean / additive masks: the decoder's own-token mask is a skip range of m3r_attention "
                                  "(must3r_b200.ops.attention skip_lo/skip_len); arbitrary masks are not on the hot path")
    B, H, Nq, D = q.shape
    if D != 64:
        raise RuntimeError("must3r_b200 attention is specialised for head_dim 64")
    if k.dtype != v.dtype or q.dtype != v.dtype:
        q, k = q.to(v.dtype), k.to(v.dtype)                        # attention.py:66-69
    Nk = k.shape[2]
    q2 = q.transpose(1, 2).reshape(B * Nq, H * D)
    k2 = k.transpose(1, 2).reshape(B * Nk, H * D)
    v2 = v.transpose(1, 2).reshape(B * Nk, H * D)
    return ops.attention(q2, k2, v2, B=B, H=H, Nq=Nq, Nk0=Nk).view(B, Nq, H * D)
