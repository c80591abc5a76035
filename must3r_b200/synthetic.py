"""Deterministic synthetic weights / inputs for parity tests, smoke and bench.

No real checkpoints exist offline, so every parity number is taken on seeded random weights laid out
with the reference's state-dict key names (SURVEY.md §3.1: encoder ``patch_embed.proj``,
``blocks_enc.{i}.*``, ``norm_enc``; decoder ``image2_embed``, ``feat_embed_enc_to_dec``,
``blocks_dec.{i}.*``, ``feedback_layer``, ``feedback_norm``, ``norm_dec``, ``head_dec.proj``).
Unlike the reference's default init (must3r/model/blocks/layers.py:23-33,
must3r/model/feedback_mechanism.py:26-35) biases, LayerNorm affines and the feedback fc2 are
randomised so that every code path carries signal (SURVEY.md §4).

Values come from a CPU ``torch.Generator`` so they are identical here and on the GPU box.
"""
from __future__ import annotations

import math
from typing import Dict, Tuple

import torch


def _lin(g, out_f, in_f, prefix, sd, bias=True, gain=1.0):
    a = gain * math.sqrt(6.0 / (in_f + out_f))  # xavier_uniform, as BaseTransformer._init_weights
    sd[prefix + ".weight"] = (torch.rand(out_f, in_f, generator=g) * 2 - 1) * a
    if bias:
        sd[prefix + ".bias"] = (torch.rand(out_f, generator=g) * 2 - 1) * 0.02


def _ln(g, dim, prefix, sd):
    sd[prefix + ".weight"] = 1.0 + 0.02 * torch.randn(dim, generator=g)
    sd[prefix + ".bias"] = 0.02 * torch.randn(dim, generator=g)


def encoder_state_dict(seed: int = 0, embed_dim: int = 1024, depth: int = 24, mlp_ratio: int = 4,
                       patch_size: int = 16) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device="cpu").manual_seed(1000 + seed)
    sd: Dict[str, torch.Tensor] = {}
    fan_in = 3 * patch_size * patch_size
    a = math.sqrt(6.0 / (fan_in + embed_dim))
    sd["patch_embed.proj.weight"] = (torch.rand(embed_dim, 3, patch_size, patch_size, generator=g) * 2 - 1) * a
    sd["patch_embed.proj.bias"] = (torch.rand(embed_dim, generator=g) * 2 - 1) * 0.02
    for i in range(depth):
        p = f"blocks_enc.{i}"
        _ln(g, embed_dim, p + ".norm1", sd)
        _lin(g, 3 * embed_dim, embed_dim, p + ".attn.qkv", sd)
        _lin(g, embed_dim, embed_dim, p + ".attn.proj", sd)
        _ln(g, embed_dim, p + ".norm2", sd)
        _lin(g, mlp_ratio * embed_dim, embed_dim, p + ".mlp.fc1", sd)
        _lin(g, embed_dim, mlp_ratio * embed_dim, p + ".mlp.fc2", sd)
    _ln(g, embed_dim, "norm_enc", sd)
    return sd


def decoder_state_dict(seed: int = 0, enc_embed_dim: int = 1024, embed_dim: int = 768, depth: int = 12,
                       mlp_ratio: int = 4, output_dim: int = 1792, feedback_type="single_mlp"
                       ) -> Dict[str, torch.Tensor]:
    g = torch.Generator(device="cpu").manual_seed(2000 + seed)
    sd: Dict[str, torch.Tensor] = {}
    sd["image2_embed"] = 0.02 * torch.randn(1, 1, embed_dim, generator=g)
    _lin(g, embed_dim, enc_embed_dim, "feat_embed_enc_to_dec", sd)
    for i in range(depth):
        p = f"blocks_dec.{i}"
        _ln(g, embed_dim, p + ".norm1", sd)
        _lin(g, 3 * embed_dim, embed_dim, p + ".attn.qkv", sd)
        _lin(g, embed_dim, embed_dim, p + ".attn.proj", sd)
        _ln(g, embed_dim, p + ".norm2", sd)
        _ln(g, embed_dim, p + ".norm_y", sd)
        for nm in ("projq", "projk", "projv", "proj"):
            _lin(g, embed_dim, embed_dim, p + ".cross_attn." + nm, sd)
        _ln(g, embed_dim, p + ".norm3", sd)
        _lin(g, mlp_ratio * embed_dim, embed_dim, p + ".mlp.fc1", sd)
        _lin(g, embed_dim, mlp_ratio * embed_dim, p + ".mlp.fc2", sd)
    if feedback_type == "single_mlp":
        _lin(g, 4 * embed_dim, embed_dim, "feedback_layer.fc1", sd)
        _lin(g, embed_dim, 4 * embed_dim, "feedback_layer.fc2", sd)
        _ln(g, embed_dim, "feedback_norm", sd)
    elif feedback_type == "single_linear":
        _lin(g, embed_dim, embed_dim, "feedback_layer", sd)
        _ln(g, embed_dim, "feedback_norm", sd)
    _ln(g, embed_dim, "norm_dec", sd)
    _lin(g, output_dim, embed_dim, "head_dec.proj", sd)
    return sd


def synthetic_views(n_views: int, H: int, W: int, seed: int = 2) -> Tuple[torch.Tensor, torch.Tensor]:
    """Images in the ImgNorm range [-1,1] (dust3r/dust3r/utils/image.py:23) and their true_shape."""
    g = torch.Generator(device="cpu").manual_seed(3000 + seed)
    imgs = torch.rand(n_views, 3, H, W, generator=g) * 2 - 1
    true_shape = torch.tensor([[H, W]] * n_views, dtype=torch.int64)
    return imgs, true_shape


def synthetic_frame(H: int, W: int, seed: int = 0) -> "np.ndarray":
    """A camera-like RGB uint8 frame [H,W,3]: per-channel gradients plus noise, with hard-edged saturated blocks and a
    black stripe, so that resampling filters ring against 0 and 255 and their clamping is exercised.  Integer arithmetic
    only, so every machine regenerates the same bytes."""
    g = torch.Generator(device="cpu").manual_seed(4000 + seed)
    y = torch.arange(H, dtype=torch.int64)[:, None, None]
    x = torch.arange(W, dtype=torch.int64)[None, :, None]
    mix = torch.randint(0, 256, (1, 1, 3), generator=g)
    img = (x * mix + y * (256 - mix)) * 120 // (256 * max(H + W - 2, 1))        # gradients, one direction per channel
    img = img + ((3 * x + 2 * y + mix) % 48) * 2 + 40                              # a sawtooth texture
    img = img + torch.randint(-40, 41, (H, W, 3), generator=g)                     # noise
    for _ in range(6):                                                             # saturated rectangles, hard edges
        y0, x0 = int(torch.randint(0, H, (1,), generator=g)), int(torch.randint(0, W, (1,), generator=g))
        h = int(torch.randint(4, max(5, H // 4), (1,), generator=g))
        w = int(torch.randint(4, max(5, W // 4), (1,), generator=g))
        img[y0:y0 + h, x0:x0 + w] = 255 * torch.randint(0, 2, (3,), generator=g)
    img[:, W // 3:W // 3 + max(1, W // 40)] = 0                                    # a black stripe next to bright content
    return img.clamp(0, 255).to(torch.uint8).numpy()


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    """‖a−b‖₂ / ‖b‖₂ (b is the reference)."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def camera_like_head_bias(dsd: Dict[str, torch.Tensor], gain: float = 0.5, depth: float = 2.0) -> Dict[str, torch.Tensor]:
    """Shift the decoder head's bias (in place) so that a random network predicts camera-like point maps: points in front
    of the camera (z > 0) whose x and y grow with the pixel's column and row inside each 16x16 patch (world and local
    channels alike).  The SLAM front end's Weiszfeld focal is then positive, as with a trained model."""
    i, j = torch.meshgrid(torch.arange(16.0), torch.arange(16.0), indexing="ij")
    bias = dsd["head_dec.proj.bias"].view(-1, 256)
    for c0 in (0, 3):
        bias[c0] += gain * ((j - 7.5) / 8).flatten()
        bias[c0 + 1] += gain * ((i - 7.5) / 8).flatten()
        bias[c0 + 2] += depth
    return dsd
