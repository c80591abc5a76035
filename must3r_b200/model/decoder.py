"""MUSt3R memory decoder with the reference's constructor, state-dict keys, forward / forward_list
signatures and memory-tuple format (must3r/model/decoder.py:14-350), executing on the sm_90a kernels.

Memory tuple (decoder.py:337): ``(list[depth] of Tensor[B,Nmem,2*D], labels int64 [B,Nmem], mem_nimgs,
mem_protected_imgs, mem_protected_tokens)``.  The K|V tensors are 16-bit (the precision set with
``set_precision``), ordinary caller-owned torch tensors: the engine's boolean-mask edits, in-place
assignments and pickling (must3r/engine/inference.py:205-228) work on them unchanged.
"""
from __future__ import annotations

import ctypes as C
from functools import partial

import torch
import torch.nn as nn

from .. import _lib
from . import common as cm

MEMORY_MODES = ['norm_y', 'kv', 'raw']


class MemArena:
    """Backing store of a memory that can grow in place: per level one [B, cap, mem_D] buffer, of which the first `tail`
    rows are handed out.  The memory tensors of the tuple are prefix views `buf[:, :rows]` tagged with their arena; an
    update call whose input memory is the LATEST version (rows == tail) and fits writes its new rows behind it instead of
    re-creating the reference's `torch.cat` (must3r/model/decoder.py:330).  Older versions stay valid (rows are only ever
    appended); a call on an older version, or one that does not fit, gets a fresh arena and a copy, exactly as before."""

    __slots__ = ("bufs", "cap", "tail")

    def __init__(self, bufs, cap):
        self.bufs, self.cap, self.tail = bufs, cap, 0

    def views(self, rows):
        out = [b[:, :rows] for b in self.bufs]
        for v in out:
            v._m3r_arena = self
        return out

    @staticmethod
    def of(mem_vals):
        """The arena behind a list of memory tensors, or None (foreign tensors, copies, re-sliced views)."""
        a = getattr(mem_vals[0], "_m3r_arena", None) if len(mem_vals) else None
        if a is None or len(a.bufs) != len(mem_vals):
            return None
        for m, b in zip(mem_vals, a.bufs):
            if getattr(m, "_m3r_arena", None) is not a or m.data_ptr() != b.data_ptr() or m.shape[1] > a.cap or m.stride(0) != b.stride(0):
                return None
        return a


class _CachedDecoderBlock(nn.Module):
    """Key names of must3r/model/blocks/layers.py:57-79."""

    def __init__(self, dim, mlp_ratio, norm_layer):
        super().__init__()
        self.norm1 = norm_layer(dim)
        self.attn = cm.AttnParams(dim)
        self.norm2 = norm_layer(dim)
        self.norm_y = norm_layer(dim)
        self.cross_attn = cm.CrossAttnParams(dim)
        self.norm3 = norm_layer(dim)
        self.mlp = cm.Mlp(dim, int(dim * mlp_ratio))


class _LinearHead(nn.Module):
    """Key names of must3r/model/blocks/head.py:63-67 (head_dec.proj)."""

    def __init__(self, embed_dim, output_dim, patch_size):
        super().__init__()
        self.patch_size = patch_size
        self.proj = nn.Linear(embed_dim, output_dim, bias=True)


class MUSt3R(nn.Module):
    def __init__(self, img_size=(224, 224), enc_embed_dim=1024, patch_size=16, embed_dim=768, output_dim=1792,
                 depth=12, num_heads=12, mlp_ratio=4, norm_layer=partial(nn.LayerNorm, eps=1e-6), act_layer=nn.GELU,
                 pos_embed='RoPE100', landscape_only=True, head='Linear', feedback_type=None, memory_mode="norm_y",
                 pointmaps_activation=cm.ActivationType.NORM_EXP, block_type=None, **kv):
        super().__init__()
        if head != 'Linear':
            raise ValueError(f'invalid head {head}')                       # decoder.py:80
        if patch_size != 16 or embed_dim != num_heads * 64:
            raise ValueError("must3r_b200 kernels are specialised for patch_size 16 and head_dim 64")
        if act_layer is not nn.GELU:
            raise ValueError("must3r_b200 implements the exact-erf GELU MLP only")
        assert memory_mode in MEMORY_MODES
        if isinstance(img_size, int):
            img_size = (img_size, img_size)
        self.pointmaps_activation = pointmaps_activation
        self.enc_embed_dim, self.embed_dim, self.depth = enc_embed_dim, embed_dim, depth
        self.attn_num_heads, self.output_dim, self.patch_size = num_heads, output_dim, patch_size
        self.mlp_hidden = int(embed_dim * mlp_ratio)
        self.landscape_only = landscape_only
        self.memory_mode = memory_mode
        self.max_seq_len = max(img_size) // patch_size
        self.grid_size = (img_size[0] // patch_size, img_size[1] // patch_size)
        self.rope_base, self.rope_f0 = cm.parse_pos_embed(pos_embed)
        # parameters, reference key names (decoder.py:49-80, feedback_mechanism.py:11-23)
        self.feat_embed_enc_to_dec = nn.Linear(enc_embed_dim, embed_dim, bias=True)
        self.image2_embed = nn.Parameter(torch.zeros(1, 1, embed_dim))
        self.blocks_dec = nn.ModuleList([_CachedDecoderBlock(embed_dim, mlp_ratio, norm_layer) for _ in range(depth)])
        self.feedback_type = feedback_type
        if feedback_type == 'single_mlp':
            self.feedback_layer = cm.Mlp(embed_dim, 4 * embed_dim, embed_dim)
            self.feedback_norm = nn.LayerNorm(embed_dim)
        elif feedback_type == 'single_linear':
            self.feedback_layer = nn.Linear(embed_dim, embed_dim)
            self.feedback_norm = nn.LayerNorm(embed_dim)
        else:
            assert not feedback_type
            self.feedback_layer, self.feedback_norm = None, None
        self.norm_dec = norm_layer(embed_dim)
        self.ln_eps = self.norm_dec.eps
        self.head_dec = _LinearHead(embed_dim, output_dim, patch_size)
        cm.init_like_reference(self)
        nn.init.normal_(self.image2_embed, std=.02)
        if feedback_type == 'single_mlp':                                  # feedback_mechanism.py:26-35
            nn.init.constant_(self.feedback_layer.fc2.bias, 0)
            nn.init.constant_(self.feedback_layer.fc2.weight, 0)
        elif feedback_type == 'single_linear':
            nn.init.constant_(self.feedback_layer.bias, 0)
            nn.init.constant_(self.feedback_layer.weight, 0)
        self._pack = None
        self._reserve_tokens = 0
        self._growth = 0.0

    def reserve_memory(self, n_tokens: int = 0, growth: float = 0.0):
        """Hint for the memory tensors this decoder allocates from now on: room for `n_tokens` rows per scene and / or
        geometric over-allocation by `growth` (e.g. 1.5), so that the following update calls append their rows in place
        (no O(Nmem) copy per call).  `reserve_memory()` restores exact-size allocation (the default)."""
        self._reserve_tokens, self._growth = int(n_tokens), float(growth)

    def memory_dtype(self):
        """dtype of the K|V memory tensors this decoder produces (the current 16-bit operand format; bf16 in fp8 mode)."""
        return cm.operand16(cm.get_precision())

    # ---- housekeeping identical to the reference -----------------------------------------------------
    def change_memory_mode(self, memory_mode="norm_y"):
        assert memory_mode in MEMORY_MODES
        self.memory_mode = memory_mode

    def from_dust3r(self, state_dict, verbose=True, load_head=False):
        """decoder.py:84-94"""
        state_dict = {k.replace('dec_blocks.', 'blocks_dec.').replace('decoder_embed.', 'feat_embed_enc_to_dec.').replace(
            'dec_norm.', 'norm_dec.'): v for k, v in state_dict.items()}
        if load_head:
            state_dict = {k.replace('downstream_head.proj.', 'head_dec.proj.'): v for k, v in state_dict.items()}
        return self.load_state_dict(state_dict, strict=False)

    from_croco = from_dust3r

    def _apply(self, fn, *a, **k):
        self._pack = None
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        self._pack = None
        return super().load_state_dict(*a, **k)

    def _packed(self, dtype):
        """Kernel-format weights (include/must3r_b200.h m3r_decoder_weights): every LayerNorm affine folded into the Linear
        that consumes it; per block the self-attention qkv and the memory K|V projection stacked into one [5D, D] matrix, all
        blocks in ONE contiguous [depth, 5D, D] array (so the memory append is one grouped GEMM)."""
        key = (dtype, str(self.norm_dec.weight.device))
        if self._pack is None or self._pack[0] != key:
            p = cm.WeightPack()
            D = self.embed_dim
            fp8, d16 = cm.is_fp8(dtype), cm.operand16(dtype)
            dev = self.norm_dec.weight.device
            blocks = (cm.DecBlock * self.depth)()
            # fp8: the LayerNorm-fed weights (a_w, q_w, fc1_w, fb1_w) are e4m3 with one fp32 scale per row
            w8 = cm.DecoderE4M3() if fp8 else None
            blocks8 = (cm.DecBlockE4M3 * self.depth)() if fp8 else None
            a_w_all = torch.empty((self.depth, 5 * D, D), dtype=dtype, device=dev)
            a_b_all = torch.empty((self.depth, 5 * D), dtype=torch.float32, device=dev)
            a_s_all = torch.empty((self.depth, 5 * D), dtype=torch.float32, device=dev)
            p.keep += [a_w_all, a_b_all, a_s_all]
            esz = a_w_all.element_size()
            for i, b in enumerate(self.blocks_dec):
                e = blocks[i]
                ca = b.cross_attn
                wq, bq = p.folded(b.attn.qkv.weight, b.attn.qkv.bias, b.norm1.weight, b.norm1.bias)
                kv_w = torch.cat([ca.projk.weight, ca.projv.weight], 0)
                kv_b = torch.cat([ca.projk.bias, ca.projv.bias], 0)
                wk, bk = p.folded(kv_w, kv_b, b.norm_y.weight, b.norm_y.bias)
                if fp8:
                    a_w_all[i, :3 * D], a_s_all[i, :3 * D] = cm.quantize_e4m3_rows(wq)
                    a_w_all[i, 3 * D:], a_s_all[i, 3 * D:] = cm.quantize_e4m3_rows(wk)
                    blocks8[i].a_s = a_s_all.data_ptr() + i * 5 * D * 4
                else:
                    a_w_all[i, :3 * D] = wq.to(dtype)
                    a_w_all[i, 3 * D:] = wk.to(dtype)
                a_b_all[i, :3 * D] = bq
                a_b_all[i, 3 * D:] = bk
                e.a_w = a_w_all.data_ptr() + i * 5 * D * D * esz
                e.a_b = a_b_all.data_ptr() + i * 5 * D * 4
                e.proj_w, e.proj_b = p.mat(b.attn.proj.weight, d16), p.vec(b.attn.proj.bias)
                wq2, bq2 = p.folded(ca.projq.weight, ca.projq.bias, b.norm2.weight, b.norm2.bias)
                w1, b1 = p.folded(b.mlp.fc1.weight, b.mlp.fc1.bias, b.norm3.weight, b.norm3.bias)
                if fp8:
                    (e.q_w, blocks8[i].q_s), (e.fc1_w, blocks8[i].fc1_s) = p.mat8(wq2), p.mat8(w1)
                else:
                    e.q_w, e.fc1_w = p.mat(wq2, dtype), p.mat(w1, dtype)
                e.q_b, e.fc1_b = p.vec(bq2), p.vec(b1)
                e.cproj_w, e.cproj_b = p.mat(ca.proj.weight, d16), p.vec(ca.proj.bias)
                e.fc2_w, e.fc2_b = p.mat(b.mlp.fc2.weight, d16), p.vec(b.mlp.fc2.bias)
                e.normy_w, e.normy_b = p.vec(b.norm_y.weight), p.vec(b.norm_y.bias)
                e.kv_w, e.kv_b = p.mat(kv_w, d16), p.vec(kv_b)          # memory_mode norm_y / raw: projected at use
            w = cm.DecoderWeights()
            w.enc_dim, w.embed_dim, w.depth, w.num_heads = self.enc_embed_dim, self.embed_dim, self.depth, self.attn_num_heads
            w.mlp_hidden, w.out_dim = self.mlp_hidden, self.output_dim
            w.ln_eps, w.rope_base, w.rope_f0 = self.ln_eps, self.rope_base, self.rope_f0
            w.is_bf16 = 1 if d16 == torch.bfloat16 else 0
            w.embed_w, w.embed_b = p.mat(self.feat_embed_enc_to_dec.weight, d16), p.vec(self.feat_embed_enc_to_dec.bias)
            w.image2_embed = p.vec(self.image2_embed)
            w.blocks = blocks
            if self.feedback_type == 'single_mlp':
                w.feedback, w.fb_ln_eps = 1, self.feedback_norm.eps
                f1, fb = p.folded(self.feedback_layer.fc1.weight, self.feedback_layer.fc1.bias, self.feedback_norm.weight, self.feedback_norm.bias)
                w.fb1_w, w.fb1_b = self._fb1(p, f1, dtype, w8), p.vec(fb)
                w.fb2_w, w.fb2_b = p.mat(self.feedback_layer.fc2.weight, d16), p.vec(self.feedback_layer.fc2.bias)
            elif self.feedback_type == 'single_linear':
                w.feedback, w.fb_ln_eps = 2, self.feedback_norm.eps
                f1, fb = p.folded(self.feedback_layer.weight, self.feedback_layer.bias, self.feedback_norm.weight, self.feedback_norm.bias)
                w.fb1_w, w.fb1_b = self._fb1(p, f1, dtype, w8), p.vec(fb)
            else:
                w.feedback, w.fb_ln_eps = 0, 1e-5
            hw, hb = p.folded(self.head_dec.proj.weight, self.head_dec.proj.bias, self.norm_dec.weight, self.norm_dec.bias)
            w.head_w, w.head_b = p.mat(hw, d16), p.vec(hb)
            if fp8:
                w8.blocks = blocks8
            self._pack = (key, w, blocks, p, w8, blocks8)
        return self._pack[1]

    @staticmethod
    def _fb1(p, f1, dtype, w8):
        if w8 is None:
            return p.mat(f1, dtype)
        ptr, w8.fb1_s = p.mat8(f1)
        return ptr

    # ---- forward -------------------------------------------------------------------------------------
    @torch.no_grad()
    def forward(self, x, pos, true_shape, current_mem=None, render=False, return_feats=False):
        """decoder.py:267-350.  Tensor form: x [B,nimgs,N,Denc], pos [B,nimgs,N,2], true_shape [B,nimgs,2]
        -> (mem, pointmaps [B,nimgs,H,W,7] fp32); list form (one entry per aspect ratio) -> list of pointmaps."""
        if return_feats:
            raise NotImplementedError("return_feats (training/debug only) is outside the inference hot path")
        if isinstance(x, (list, tuple)):
            return self.forward_list(list(x), list(pos), list(true_shape), current_mem, render)
        assert not render or current_mem is not None                    # decoder.py:278
        mem, pms = self.forward_list([x], [pos], [true_shape], current_mem, render)
        return mem, pms[0]

    @torch.no_grad()
    def update_tokens(self, x, pos, true_shape, current_mem=None, mem_lengths=None):
        """Memory-update call that returns only this call's new post-feedback K|V tokens
        (list[depth] of [B, n*N, 2D]) and the raw pointmaps, instead of the concatenated memory
        (= ``mem'[0][l][:, Nm:]`` of ``forward``).  Used by the sharded multi-GPU schedule (SURVEY.md §8e).

        ``mem_lengths`` (memory_mode 'kv'): B host integers, scene b's memory being rows [0, mem_lengths[b]) of
        ``current_mem[0][l][b]`` - e.g. a [B, cap, 2D] arena holding one SLAM session per scene.  The scenes are decoded
        in one call (csrc/model.cu m3r_decoder_forward_ragged), each attending only to its own rows, exactly as B separate
        calls would; the lengths travel to the device without a host synchronisation.

        x, pos and true_shape may also be lists with one entry per aspect-ratio group, as for ``forward_list``; the
        pointmaps are then a list too."""
        if isinstance(x, (list, tuple)):
            _, pms, new_tokens = self.forward_list(list(x), list(pos), list(true_shape), current_mem, render=False,
                                                   _new_only=True, _mem_lengths=mem_lengths)
            return new_tokens, pms
        _, pms, new_tokens = self.forward_list([x], [pos], [true_shape], current_mem, render=False, _new_only=True,
                                               _mem_lengths=mem_lengths)
        return new_tokens, pms[0]

    @torch.no_grad()
    def render_tokens(self, x, pos, true_shape, current_mem, mem_lengths):
        """Render call over B scenes whose memories hold different numbers of tokens (memory_mode 'kv'): x [B,n,N,Denc],
        pos [B,n,N,2], true_shape [B,n,2] -> raw pointmaps [B,n,H,W,7] fp32.  ``mem_lengths``: B host integers, scene b's
        memory being rows [0, mem_lengths[b]) of ``current_mem[0][l][b]`` (e.g. a [B, cap, 2D] arena holding one scene per
        slot).  Each scene's views attend only to its own rows (csrc/model.cu m3r_decoder_render_ragged), as B separate
        ``forward(..., render=True)`` calls would; nothing is written into the memory, and the lengths travel to the device
        without a host synchronisation."""
        _, pms = self.forward_list([x], [pos], [true_shape], current_mem, render=True, _mem_lengths=mem_lengths)
        return pms[0]

    @torch.no_grad()
    def update_tokens_to_peers(self, x, pos, true_shape, current_mem, peer_ptrs):
        """Same update, but the post-feedback K|V GEMM epilogue also stores the new rows straight into every rank's memory
        buffer: ``peer_ptrs[r][l]`` = device pointer (int) of rank r's level-l buffer at the row where this rank's tokens
        belong (fused GEMM -> all-gather over NVLink peer memory; the caller synchronises the ranks afterwards)."""
        _, pms, new_tokens = self.forward_list([x], [pos], [true_shape], current_mem, render=False, _new_only=True,
                                               _peer_ptrs=peer_ptrs)
        return new_tokens, pms[0]

    @torch.no_grad()
    def forward_list(self, x, pos, true_shape, current_mem=None, render=False, return_feats=False, _new_only=False,
                     _peer_ptrs=None, _cp=None, _mem_lengths=None):
        """decoder.py:158-265.  `_cp` (engine/context_parallel.py): dict(world, rank, owner, stage_ptrs, slot_bytes, flag_slots,
        flags_local, epoch0) - the memory is sharded over `world` GPUs and `current_mem` is this rank's shard."""
        if not x[0].is_cuda:
            raise RuntimeError("must3r_b200.MUSt3R runs on CUDA only (no CPU fallback)")
        dev = x[0].device
        w = self._packed(cm.get_precision())
        w8 = self._pack[4]
        dtype = self.memory_dtype()
        lib = _lib.lib()
        D, G = self.embed_dim, len(x)
        mem_D = 2 * D if self.memory_mode == "kv" else D                  # decoder.py:189,277
        if _peer_ptrs and self.memory_mode != "kv":
            raise RuntimeError("peer output (fused gather) needs memory_mode='kv'")
        B = x[0].shape[0]
        groups = (cm.DecGroup * G)()
        keep, outs = [], []
        Nt, n_total = 0, 0
        for i in range(G):
            Bi, n, N, Denc = x[i].shape
            assert Bi == B and Denc == self.enc_embed_dim
            hw = getattr(true_shape[i], "_m3r_hw", None)
            if hw is None:
                # like the reference (head.py:31-32) this reads true_shape on the host: a device sync when it is a CUDA
                # tensor.  must3r_b200.engine attaches the host copy as `_m3r_hw` so the launch thread never stalls.
                ts = true_shape[i].reshape(B * n, 2)
                assert bool((ts == ts[:1]).all()), 'true_shape must be all identical'   # head.py:31
                hw = tuple(int(v) for v in ts[0].tolist())
            H, W = hw
            if self.landscape_only and H > W:
                raise NotImplementedError("landscape_only=True with portrait views: load_model converts the head to "
                                          "landscape_only=False (must3r/model/__init__.py:55); do the same here")
            xi = x[i].reshape(B * n * N, Denc).float().contiguous()
            pi = pos[i].reshape(B * n * N, 2).to(torch.int64).contiguous()
            pm = torch.empty((B, n, H, W, self.output_dim // 256), dtype=torch.float32, device=dev)
            keep += [xi, pi]
            outs.append(pm)
            g = groups[i]
            g.n_views, g.N, g.H, g.W = n, N, H, W
            g.x_enc, g.pos, g.pointmaps = xi.data_ptr(), pi.data_ptr(), pm.data_ptr()
            Nt += n * N
            n_total += n

        call = cm.DecoderCall()
        call.B, call.G, call.groups = B, G, groups
        call.render = 1 if render else 0
        call.is_init = 1 if current_mem is None else 0
        call.mem_mode = cm.MEM_MODE_CODE[self.memory_mode]
        if current_mem is None:
            mem_vals, labels, mem_nimgs, mem_pi, mem_pt = None, torch.zeros((B, 0), dtype=torch.int64, device=dev), 0, 0, 0
            Nm = 0
        else:
            mem_vals, labels, mem_nimgs, mem_pi, mem_pt = current_mem
            Nm = mem_vals[0].shape[1]
        nm_scene = None
        if _mem_lengths is not None:
            lengths = [int(n) for n in _mem_lengths]
            if self.memory_mode != "kv" or not (_new_only or render) or current_mem is None or _peer_ptrs or _cp is not None:
                raise ValueError("mem_lengths needs memory_mode='kv', a memory and update_tokens or render_tokens")
            if len(lengths) != B or min(lengths) < 0 or max(lengths) < 1 or max(lengths) > Nm:
                raise ValueError(f"mem_lengths {lengths}: one length in [0, {Nm}] per scene ({B}), the longest >= 1")
            Nm = max(lengths)
            mem_vals = [m[:, :Nm] for m in mem_vals]
            nm_scene = torch.tensor(lengths, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
            keep.append(nm_scene)
        call.Nm = Nm
        mem_ptrs = (C.c_void_p * self.depth)()
        if Nm > 0:
            mv = []
            for l in range(self.depth):
                m = mem_vals[l]
                assert m.shape[0] == B and m.shape[2] == mem_D, \
                    f"memory rows are {m.shape[2]} wide, memory_mode={self.memory_mode!r} expects {mem_D}"
                if m.dtype != dtype or m.stride(2) != 1 or m.stride(1) != mem_D:
                    m = m.to(dtype).contiguous()
                mv.append(m)
                mem_ptrs[l] = m.data_ptr()
            keep.append(mv)
            bstrides = {m.stride(0) // mem_D if B > 1 else Nm for m in mv}
            assert len(bstrides) == 1
            call.mem = mem_ptrs
            call.mem_bstride_rows = bstrides.pop()
        out_ptrs = (C.c_void_p * self.depth)()
        new_mem = None
        if _cp is not None:
            assert B == 1 and self.memory_mode == "kv" and current_mem is not None and not _new_only and not _peer_ptrs
            call.cp_world, call.cp_rank, call.cp_owner = _cp["world"], _cp["rank"], 1 if _cp["owner"] else 0
            call.cp_stage, call.cp_slot_bytes = _cp["stage_ptrs"], _cp["slot_bytes"]
            call.cp_flag_slots, call.cp_flags_local, call.cp_epoch0 = _cp["flag_slots"], _cp["flags_local"], _cp["epoch0"]
        store_new = not render and (_cp is None or _cp["owner"])
        if store_new:
            rows = Nt if _new_only else Nm + Nt
            if _new_only:
                new_mem = [torch.empty((B, rows, mem_D), dtype=dtype, device=dev) for _ in range(self.depth)]
                cap = rows
            else:
                # append in place when the input is the latest version of an arena with room left (mem_out[l] == mem[l]:
                # the library then copies nothing); otherwise a fresh arena (exact size unless reserve_memory asked for more)
                arena = MemArena.of(mv) if Nm > 0 else None
                if arena is None or arena.tail != Nm or Nm + Nt > arena.cap:
                    cap = max(rows, self._reserve_tokens, int(rows * self._growth))
                    arena = MemArena([torch.empty((B, cap, mem_D), dtype=dtype, device=dev) for _ in range(self.depth)], cap)
                cap = arena.cap
                new_mem = arena.views(rows)
                arena.tail = rows
            for l in range(self.depth):
                out_ptrs[l] = new_mem[l].data_ptr()
            call.mem_out = out_ptrs
            call.mem_out_bstride_rows = cap
            call.new_only = 1 if _new_only else 0
            if _peer_ptrs:
                flat = (C.c_void_p * (len(_peer_ptrs) * self.depth))()
                for r, ptrs in enumerate(_peer_ptrs):
                    for l in range(self.depth):
                        flat[r * self.depth + l] = ptrs[l]
                call.n_peers, call.peer_mem = len(_peer_ptrs), flat
                keep.append(flat)
        nbytes = lib.m3r_decoder_workspace_bytes(C.byref(w), C.byref(call))
        with torch.cuda.device(dev):           # the library keys its per-stream state (side streams, scratch) on the current device
            ws = cm.workspace(dev, nbytes, "dec")
            if render and nm_scene is not None:
                _lib.check(lib.m3r_decoder_render_ragged(C.byref(w), None if w8 is None else C.byref(w8), C.byref(call),
                                                         C.c_void_p(nm_scene.data_ptr()), C.c_void_p(ws.data_ptr()),
                                                         ws.numel(), cm.stream_ptr(dev)), "decoder_render_ragged")
            elif w8 is not None:
                _lib.check(lib.m3r_decoder_forward_e4m3(C.byref(w), C.byref(w8), C.byref(call), None if nm_scene is None else
                                                        C.c_void_p(nm_scene.data_ptr()), C.c_void_p(ws.data_ptr()),
                                                        ws.numel(), cm.stream_ptr(dev)), "decoder_forward_e4m3")
            elif nm_scene is None:
                _lib.check(lib.m3r_decoder_forward(C.byref(w), C.byref(call), C.c_void_p(ws.data_ptr()), ws.numel(),
                                                   cm.stream_ptr(dev)), "decoder_forward")
            else:
                _lib.check(lib.m3r_decoder_forward_ragged(C.byref(w), C.byref(call), C.c_void_p(nm_scene.data_ptr()),
                                                          C.c_void_p(ws.data_ptr()), ws.numel(), cm.stream_ptr(dev)),
                           "decoder_forward_ragged")
        if _new_only:
            return None, outs, new_mem
        if render:
            out = tuple(current_mem)                                       # decoder.py:251,340: memory returned untouched
        elif not store_new:
            # context parallel, another rank stores this call's tokens: this shard is unchanged, the scene's counters advance
            tot = mem_nimgs + n_total
            out = (list(mem_vals), labels, tot, tot, labels.shape[1])
        else:
            new_labels, off = [], 0
            for i in range(G):                                             # decoder.py:237-247
                n, N = groups[i].n_views, groups[i].N
                li = torch.arange(n, dtype=labels.dtype, device=labels.device).view(1, n, 1).repeat(B, 1, N).view(B, n * N)
                new_labels.append(li + mem_nimgs + off)
                off += n
            mem_labels = torch.cat([labels] + new_labels, dim=1)
            tot = mem_nimgs + n_total
            out = (new_mem, mem_labels, tot, tot, mem_labels.shape[1])
        return out, outs


class CausalMUSt3R(MUSt3R):
    """Training-time variant (decoder.py:353); for inference `load_model` rewrites it to MUSt3R
    (must3r/model/__init__.py:53-63).  Accepts and ignores the training-only kwargs."""

    def __init__(self, protected_imgs=1, mem_dropout=0.0, dropout_mode='temporary', use_xformers_mask=False,
                 use_mem_mask=False, **kw):
        super().__init__(**kw)
