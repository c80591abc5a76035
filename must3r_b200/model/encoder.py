"""Dust3rEncoder with the reference's constructor, state-dict keys and forward signature
(must3r/model/encoder.py:13-65), executing on the sm_90a kernels through the C ABI."""
from __future__ import annotations

import ctypes as C
from functools import partial

import torch
import torch.nn as nn

from .. import _lib
from . import common as cm


class _PatchEmbed(nn.Module):
    """Key names of dust3r/croco/models/blocks.py:209-222 (patch_embed.proj = Conv2d(3, D, 16, 16))."""

    def __init__(self, img_size, patch_size, embed_dim):
        super().__init__()
        self.patch_size = (patch_size, patch_size)
        self.img_size = tuple(img_size)
        self.grid_size = (img_size[0] // patch_size, img_size[1] // patch_size)
        self.proj = nn.Conv2d(3, embed_dim, kernel_size=patch_size, stride=patch_size)


class _Block(nn.Module):
    """Key names of must3r/model/blocks/layers.py:36-49."""

    def __init__(self, dim, mlp_ratio, norm_layer):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = cm.AttnParams(dim)
        self.norm2 = norm_layer(dim)
        self.mlp = cm.Mlp(dim, int(dim * mlp_ratio))


class Dust3rEncoder(nn.Module):
    def __init__(self, img_size=(224, 224), patch_size=16, embed_dim=1024, depth=24, num_heads=16, mlp_ratio=4,
                 norm_layer=partial(nn.LayerNorm, eps=1e-6), patch_embed='PatchEmbedDust3R', pos_embed='RoPE100'):
        super().__init__()
        if patch_embed not in ('PatchEmbedDust3R', 'ManyAR_PatchEmbed'):
            raise AssertionError(patch_embed)           # dust3r/dust3r/patch_embed.py:14
        if patch_size != 16:
            raise ValueError("must3r_b200 kernels are specialised for patch_size 16")
        if embed_dim != num_heads * 64:
            raise ValueError("must3r_b200 kernels are specialised for head_dim 64")
        if isinstance(img_size, int):
            img_size = (img_size, img_size)
        self.embed_dim, self.depth, self.num_heads, self.patch_size = embed_dim, depth, num_heads, patch_size
        self.mlp_hidden = int(embed_dim * mlp_ratio)
        self.patch_embed_name = patch_embed
        self.patch_embed = _PatchEmbed(img_size, patch_size, embed_dim)
        self.max_seq_len = max(img_size) // patch_size
        self.grid_size = self.patch_embed.grid_size
        self.rope_base, self.rope_f0 = cm.parse_pos_embed(pos_embed)
        self.blocks_enc = nn.ModuleList([_Block(embed_dim, mlp_ratio, norm_layer) for _ in range(depth)])
        self.norm_enc = norm_layer(embed_dim)
        self.ln_eps = self.norm_enc.eps
        cm.init_like_reference(self)
        w = self.patch_embed.proj.weight.data
        nn.init.xavier_uniform_(w.view(w.shape[0], -1))   # croco blocks.py:236-238
        self._pack = None
        self._pos_cache = {}

    # ---- weight packing ------------------------------------------------------------------------------
    def _apply(self, fn, *a, **k):
        self._pack = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._pack = None
        return super().load_state_dict(*a, **k)

    def from_dust3r(self, state_dict, verbose=True):
        """encoder.py:54-61"""
        state_dict = {k.replace('enc_blocks', 'blocks_enc').replace('enc_norm', 'norm_enc'): v for k, v in state_dict.items()}
        inc = self.load_state_dict(state_dict, strict=False)
        assert len(inc.missing_keys) == 0
        return inc

    from_croco = from_dust3r

    def _packed(self, dtype):
        key = (dtype, str(self.norm_enc.weight.device))
        if self._pack is None or self._pack[0] != key:
            p = cm.WeightPack()
            fp8, d16 = cm.is_fp8(dtype), cm.operand16(dtype)
            blocks = (cm.EncBlock * self.depth)()
            blocks8 = (cm.EncBlockE4M3 * self.depth)() if fp8 else None
            for i, b in enumerate(self.blocks_enc):
                e = blocks[i]
                if fp8:
                    # norm1 / norm2 folded into qkv / fc1, which take e4m3 operands (m3r_encoder_forward_e4m3)
                    wq, bq = p.folded(b.attn.qkv.weight, b.attn.qkv.bias, b.norm1.weight, b.norm1.bias)
                    w1, b1 = p.folded(b.mlp.fc1.weight, b.mlp.fc1.bias, b.norm2.weight, b.norm2.bias)
                    (e.qkv_w, blocks8[i].qkv_s), e.qkv_b = p.mat8(wq), p.vec(bq)
                    (e.fc1_w, blocks8[i].fc1_s), e.fc1_b = p.mat8(w1), p.vec(b1)
                else:
                    e.norm1_w, e.norm1_b = p.vec(b.norm1.weight), p.vec(b.norm1.bias)
                    e.qkv_w, e.qkv_b = p.mat(b.attn.qkv.weight, dtype), p.vec(b.attn.qkv.bias)
                    e.norm2_w, e.norm2_b = p.vec(b.norm2.weight), p.vec(b.norm2.bias)
                    e.fc1_w, e.fc1_b = p.mat(b.mlp.fc1.weight, dtype), p.vec(b.mlp.fc1.bias)
                e.proj_w, e.proj_b = p.mat(b.attn.proj.weight, d16), p.vec(b.attn.proj.bias)
                e.fc2_w, e.fc2_b = p.mat(b.mlp.fc2.weight, d16), p.vec(b.mlp.fc2.bias)
            w = cm.EncoderWeights()
            w.embed_dim, w.depth, w.num_heads, w.mlp_hidden = self.embed_dim, self.depth, self.num_heads, self.mlp_hidden
            w.ln_eps, w.rope_base, w.rope_f0 = self.ln_eps, self.rope_base, self.rope_f0
            w.is_bf16 = 1 if d16 == torch.bfloat16 else 0
            w.patch_w, w.patch_b = p.mat(self.patch_embed.proj.weight, d16), p.vec(self.patch_embed.proj.bias)
            w.blocks = blocks
            w.norm_w, w.norm_b = p.vec(self.norm_enc.weight), p.vec(self.norm_enc.bias)
            self._pack = (key, w, blocks, p, blocks8)
        return self._pack[1]

    def _positions(self, h, w, device):
        """PositionGetter, croco blocks.py:195-207: cartesian_prod(arange(h), arange(w)) = (y, x)."""
        key = (h, w, str(device))
        if key not in self._pos_cache:
            self._pos_cache[key] = torch.cartesian_prod(torch.arange(h, device=device), torch.arange(w, device=device))
        return self._pos_cache[key]

    batches_well = True     # one call over many views is far more efficient than one call per view (engine: encode missing views up front)

    # ---- forward -------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, img, true_shape=None):
        """(img [V,3,H,W], true_shape [V,2]) -> (x [V,N,D] fp32, pos [V,N,2] int64), encoder.py:46-52."""
        if not img.is_cuda:
            raise RuntimeError("must3r_b200.Dust3rEncoder runs on CUDA only (no CPU fallback)")
        V, Cc, H, W = img.shape
        assert Cc == 3
        assert H % self.patch_size == 0, f"Input image height ({H}) is not a multiple of patch size ({self.patch_size})."
        assert W % self.patch_size == 0, f"Input image width ({W}) is not a multiple of patch size ({self.patch_size})."
        portrait = None
        if self.patch_embed_name == 'ManyAR_PatchEmbed':
            # dust3r/dust3r/patch_embed.py:42-70: batch is stored landscape; portrait views are transposed
            assert W >= H, f'img should be in landscape mode, but got {W=} {H=}'
            assert true_shape is not None and tuple(true_shape.shape) == (V, 2), f"true_shape has the wrong shape={None if true_shape is None else true_shape.shape}"
            height, width = true_shape.T
            portrait = ~(width >= height)
            if not bool(portrait.any()):
                portrait = None
        img = img.float().contiguous()
        gh, gw = H // 16, W // 16
        N = gh * gw
        if portrait is not None:
            x = img.new_empty((V, N, self.embed_dim))
            pos = torch.empty((V, N, 2), dtype=torch.int64, device=img.device)
            for sel, im in ((~portrait, img[~portrait]), (portrait, img[portrait].swapaxes(-1, -2).contiguous())):
                if im.shape[0] == 0:
                    continue
                xs, ps = self._run(im)
                x[sel], pos[sel] = xs, ps
            return x, pos
        return self._run(img)

    def _run(self, img):
        V, _, H, W = img.shape
        gh, gw = H // 16, W // 16
        N = gh * gw
        dtype = cm.get_precision()
        w = self._packed(dtype)
        lib = _lib.lib()
        pos1 = self._positions(gh, gw, img.device)
        out = torch.empty((V, N, self.embed_dim), dtype=torch.float32, device=img.device)
        nbytes = lib.m3r_encoder_workspace_bytes(C.byref(w), V, H, W)
        with torch.cuda.device(img.device):
            ws = cm.workspace(img.device, nbytes, "enc")
            args = (C.c_void_p(img.data_ptr()), V, H, W, C.c_void_p(pos1.data_ptr()), C.c_void_p(out.data_ptr()),
                    C.c_void_p(ws.data_ptr()), ws.numel(), cm.stream_ptr(img.device))
            blocks8 = self._pack[4]
            if blocks8 is None:
                _lib.check(lib.m3r_encoder_forward(C.byref(w), *args), "encoder_forward")
            else:
                _lib.check(lib.m3r_encoder_forward_e4m3(C.byref(w), blocks8, *args), "encoder_forward_e4m3")
        return out, pos1.view(1, N, 2).expand(V, -1, -1).clone()

