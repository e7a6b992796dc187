"""Causal Wan DiT on the sm_90a kernels — host-side mirror of the reference's model classes.

Mirrors ``wan/modules/causal_model.py`` (CausalWanModel :526, CausalWanAttentionBlock :400,
CausalWanSelfAttention :174, CausalHead :495) and ``wan/modules/model.py``
(WanT2VCrossAttention :171): same class names, constructor arguments, attributes and
state-dict keys, so reference checkpoints load with ``load_state_dict`` and the reference's
callers (release_server.py:542-736, pipeline/causal_inference.py) drive it unchanged.

The modules only HOLD parameters; the arithmetic is a fixed schedule of calls into
libkrea_b200.so (``ops``):

    per block:  add_modulation -> ln_modulate -> GEMM(to_qkv) -> qkv_norm_rope(+KV append)
                -> attention -> GEMM(o, gate+residual) -> ln_affine -> GEMM(q) -> rmsnorm
                -> attention(text K/V) -> GEMM(o, residual) -> ln_modulate -> GEMM(ffn.0, GELU)
                -> GEMM(ffn.2, gate+residual)

There is no eager fallback: CPU tensors raise (ops._req).
"""
from __future__ import annotations

import math
import os
import types
from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import ops


def _linear(x: torch.Tensor, lin: nn.Linear, **kw) -> torch.Tensor:
    """nn.Linear of a DiT block on the GEMM kernels: bf16 by default, FP8 (dynamic per-tensor activation cast +
    e4m3 wgmma GEMM) when ``realtime_video_b200.fp8.quantize_`` attached quantised weights to the module."""
    q = getattr(lin, "_kr_fp8", None)
    if q is None:
        return ops.gemm(x, lin.weight, lin.bias, **kw)
    return ops.linear_fp8(x, q[0], q[1], lin.bias, **kw)


def rope_angles(max_seq_len: int, dim: int, theta: float = 10000.0) -> torch.Tensor:
    """Rotation angles pos * theta^(-2i/dim), float64 (reference rope_params, model.py:28-35)."""
    return torch.outer(torch.arange(max_seq_len, dtype=torch.float64),
                       1.0 / torch.pow(theta, torch.arange(0, dim, 2, dtype=torch.float64).div(dim)))


class BlockMaskSpec:
    """What ``_prepare_blockwise_causal_attn_mask`` returns here: the parameters of the reference's
    BlockMask (causal_model.py:109-141) — the kernel evaluates the rule per tile instead of
    materialising a mask."""

    def __init__(self, num_frames, frame_seqlen, num_frame_per_block, local_attn_size):
        self.num_frames, self.frame_seqlen = num_frames, frame_seqlen
        self.num_frame_per_block, self.local_attn_size = num_frame_per_block, local_attn_size

    @property
    def block_len(self) -> int:
        return self.frame_seqlen * self.num_frame_per_block

    @property
    def window(self) -> int:
        return 0 if self.local_attn_size == -1 else self.local_attn_size * self.frame_seqlen


class WanRMSNorm(nn.Module):
    def __init__(self, dim, eps=1e-5):
        super().__init__()
        self.dim, self.eps = dim, eps
        self.weight = nn.Parameter(torch.ones(dim))


class WanLayerNorm(nn.LayerNorm):
    def __init__(self, dim, eps=1e-6, elementwise_affine=False):
        super().__init__(dim, elementwise_affine=elementwise_affine, eps=eps)


class CausalWanSelfAttention(nn.Module):
    """Parameter holder + KV-cache index algebra of causal_model.py:174-397."""

    def __init__(self, dim, num_heads, local_attn_size=-1, sink_size=0, qk_norm=True, eps=1e-6):
        assert dim % num_heads == 0
        super().__init__()
        self.dim, self.num_heads, self.head_dim = dim, num_heads, dim // num_heads
        self.local_attn_size, self.sink_size = local_attn_size, sink_size
        self.qk_norm, self.eps = qk_norm, eps
        # frozen at construction like the reference (:192); rescaled by the real frame length
        self._max_attention_frames = 21 if local_attn_size == -1 else local_attn_size
        self.max_attention_size = 32760 if local_attn_size == -1 else local_attn_size * 1560
        self.fused_projections = False
        self.num_frame_per_block = 1
        self.q, self.k = nn.Linear(dim, dim), nn.Linear(dim, dim)
        self.v, self.o = nn.Linear(dim, dim), nn.Linear(dim, dim)
        self.norm_q = WanRMSNorm(dim, eps=eps) if qk_norm else nn.Identity()
        self.norm_k = WanRMSNorm(dim, eps=eps) if qk_norm else nn.Identity()

    @torch.no_grad()
    def fuse_projections(self):
        """causal_model.py:204-216 — to_qkv = cat(q, k, v), q/k/v kept."""
        if self.fused_projections:
            return
        w = torch.cat([self.q.weight.data, self.k.weight.data, self.v.weight.data])
        b = torch.cat([self.q.bias.data, self.k.bias.data, self.v.bias.data])
        with torch.device("meta"):
            self.to_qkv = nn.Linear(w.shape[1], w.shape[0], bias=True)
        self.to_qkv.load_state_dict({"weight": w, "bias": b}, strict=True, assign=True)
        self.fused_projections = True


class WanT2VCrossAttention(nn.Module):
    """Parameter holder of wan/modules/model.py:171-228."""

    def __init__(self, dim, num_heads, window_size=(-1, -1), qk_norm=True, eps=1e-6):
        super().__init__()
        self.dim, self.num_heads, self.head_dim = dim, num_heads, dim // num_heads
        self.window_size, self.qk_norm, self.eps = window_size, qk_norm, eps
        self.q, self.k = nn.Linear(dim, dim), nn.Linear(dim, dim)
        self.v, self.o = nn.Linear(dim, dim), nn.Linear(dim, dim)
        self.norm_q = WanRMSNorm(dim, eps=eps) if qk_norm else nn.Identity()
        self.norm_k = WanRMSNorm(dim, eps=eps) if qk_norm else nn.Identity()


class CausalWanAttentionBlock(nn.Module):
    def __init__(self, cross_attn_type, dim, ffn_dim, num_heads, local_attn_size=-1, sink_size=0,
                 qk_norm=True, cross_attn_norm=False, eps=1e-6):
        super().__init__()
        if cross_attn_type != "t2v_cross_attn":
            raise NotImplementedError("only the t2v cross-attention is on the hot path (SURVEY.md §2)")
        self.dim, self.ffn_dim, self.num_heads = dim, ffn_dim, num_heads
        self.local_attn_size, self.qk_norm, self.cross_attn_norm, self.eps = \
            local_attn_size, qk_norm, cross_attn_norm, eps
        self.norm1 = WanLayerNorm(dim, eps)
        self.self_attn = CausalWanSelfAttention(dim, num_heads, local_attn_size, sink_size, qk_norm, eps)
        self.norm3 = WanLayerNorm(dim, eps, elementwise_affine=True) if cross_attn_norm else nn.Identity()
        self.cross_attn = WanT2VCrossAttention(dim, num_heads, (-1, -1), qk_norm, eps)
        self.norm2 = WanLayerNorm(dim, eps)
        self.ffn = nn.Sequential(nn.Linear(dim, ffn_dim), nn.GELU(approximate="tanh"), nn.Linear(ffn_dim, dim))
        self.modulation = nn.Parameter(torch.randn(1, 6, dim) / dim ** 0.5)


class CausalHead(nn.Module):
    def __init__(self, dim, out_dim, patch_size, eps=1e-6):
        super().__init__()
        self.dim, self.out_dim, self.patch_size, self.eps = dim, out_dim, patch_size, eps
        self.norm = WanLayerNorm(dim, eps)
        self.head = nn.Linear(dim, math.prod(patch_size) * out_dim)
        self.modulation = nn.Parameter(torch.randn(1, 2, dim) / dim ** 0.5)


class CausalWanModel(nn.Module):
    """Mirror of CausalWanModel (causal_model.py:526-1173), inference path only."""

    def __init__(self, model_type="t2v", patch_size=(1, 2, 2), text_len=512, in_dim=16, dim=2048,
                 ffn_dim=8192, freq_dim=256, text_dim=4096, out_dim=16, num_heads=16, num_layers=32,
                 local_attn_size=-1, sink_size=0, qk_norm=True, cross_attn_norm=True, eps=1e-6):
        super().__init__()
        if model_type != "t2v":
            raise NotImplementedError("i2v is outside the hot path (SURVEY.md §2 row 18)")
        if (dim // num_heads) != 128:
            raise NotImplementedError("attention kernel supports head_dim 128 (all Wan 2.1 models)")
        if not qk_norm:
            raise NotImplementedError("qk_norm=False: the RMSNorm is fused into the RoPE / KV-append kernel; every "
                                      "Wan 2.1 checkpoint has qk_norm=True")
        self.config = types.SimpleNamespace(
            model_type=model_type, patch_size=patch_size, text_len=text_len, in_dim=in_dim, dim=dim,
            ffn_dim=ffn_dim, freq_dim=freq_dim, text_dim=text_dim, out_dim=out_dim,
            num_heads=num_heads, num_layers=num_layers, local_attn_size=local_attn_size,
            sink_size=sink_size, qk_norm=qk_norm, cross_attn_norm=cross_attn_norm, eps=eps)
        self.model_type, self.patch_size, self.text_len = model_type, tuple(patch_size), text_len
        self.in_dim, self.dim, self.ffn_dim, self.freq_dim = in_dim, dim, ffn_dim, freq_dim
        self.text_dim, self.out_dim, self.num_heads, self.num_layers = text_dim, out_dim, num_heads, num_layers
        self.local_attn_size, self.qk_norm, self.cross_attn_norm, self.eps = \
            local_attn_size, qk_norm, cross_attn_norm, eps

        self.patch_embedding = nn.Conv3d(in_dim, dim, kernel_size=patch_size, stride=patch_size)
        self.text_embedding = nn.Sequential(nn.Linear(text_dim, dim), nn.GELU(approximate="tanh"),
                                            nn.Linear(dim, dim))
        self.time_embedding = nn.Sequential(nn.Linear(freq_dim, dim), nn.SiLU(), nn.Linear(dim, dim))
        self.time_projection = nn.Sequential(nn.SiLU(), nn.Linear(dim, dim * 6))
        self.blocks = nn.ModuleList([
            CausalWanAttentionBlock("t2v_cross_attn", dim, ffn_dim, num_heads, local_attn_size,
                                    sink_size, qk_norm, cross_attn_norm, eps) for _ in range(num_layers)])
        self.head = CausalHead(dim, out_dim, patch_size, eps)

        d = dim // num_heads
        ang = torch.cat([rope_angles(1024, d - 4 * (d // 6)), rope_angles(1024, 2 * (d // 6)),
                         rope_angles(1024, 2 * (d // 6))], dim=1)
        # plain attribute like the reference (:636-645): complex128 [1024, d/2], not a buffer
        self.freqs = torch.polar(torch.ones_like(ang), ang)
        self._rope_angles = ang
        self._rope_table: Optional[torch.Tensor] = None      # device float32 (cos, sin)
        self.sp = None          # optional parallel.SequenceParallel (single-stream multi-GPU mode)
        self.pp = None          # optional parallel.LayerPipeline (layer-sharded multi-GPU mode, BASELINE configs[2])
        self.use_block_fwd = os.environ.get("KR_BLOCK_FWD", "0") not in ("", "0")   # one C-ABI call per block
        # "sage": the cached self-attention and the cross-attention run on the INT8/FP8 quantised kernels (the
        # reference's sageattention backend on H100); None: bf16 attention everywhere
        self.attn_quant = "sage" if os.environ.get("KR_SAGE_ATTN", "0") not in ("", "0") else None
        self.init_weights()
        self.gradient_checkpointing = False
        self.block_mask = None
        self.num_frame_per_block = 1
        self.independent_first_frame = False

    # ----------------------------------------------------------------------------------------
    def init_weights(self):
        """causal_model.py:1151-1173."""
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
        nn.init.xavier_uniform_(self.patch_embedding.weight.flatten(1))
        for m in self.text_embedding.modules():
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, std=.02)
        for m in self.time_embedding.modules():
            if isinstance(m, nn.Linear):
                nn.init.normal_(m.weight, std=.02)
        nn.init.zeros_(self.head.head.weight)

    @staticmethod
    def _prepare_blockwise_causal_attn_mask(device, num_frames: int = 21, frame_seqlen: int = 1560,
                                            num_frame_per_block=1, local_attn_size=-1) -> BlockMaskSpec:
        """causal_model.py:663-674 — returns the mask RULE; nothing is materialised."""
        return BlockMaskSpec(num_frames, frame_seqlen, num_frame_per_block, local_attn_size)

    @property
    def kv_cache_heads(self) -> int:
        """Heads held by this rank's self-attention KV cache (all of them unless sequence-parallel)."""
        return self.num_heads if self.sp is None else self.sp.local_heads(self.num_heads)

    def _rope(self, device) -> torch.Tensor:
        if self._rope_table is None or self._rope_table.device != device:
            a = self._rope_angles
            self._rope_table = torch.stack([a.cos(), a.sin()], dim=-1).float().contiguous().to(device)
        return self._rope_table

    # ----------------------------------------------------------------------------------------
    def _embed_text(self, context: torch.Tensor) -> torch.Tensor:
        """text_embedding over the zero-padded prompt (causal_model.py:895-902).  Its only consumer is the
        cross-attention K/V projection, so ``forward_tokens`` calls it only on passes where some block's
        ``crossattn_cache`` is not initialised (the reference recomputes it on every forward and discards it)."""
        te = self.text_embedding
        ctx = context
        if ctx.shape[0] < self.text_len:
            ctx = torch.cat([ctx, ctx.new_zeros(self.text_len - ctx.shape[0], ctx.shape[1])])
        ctx = ctx.to(te[0].weight.dtype).contiguous()
        h = ops.gemm(ctx, te[0].weight, te[0].bias, epilogue=ops.EPI_BIAS_GELU)
        return ops.gemm(h, te[2].weight, te[2].bias)

    @staticmethod
    def _cache_slot(sa: CausalWanSelfAttention, kv_cache, L: int, Dh: int, fs: int, current_start: int, mask):
        """KV-cache index algebra of causal_model.py:305-392 for a call that appends L token rows: returns the cache
        views [rows, Dh], the slot [local_start, local_end) this call writes, the RoPE start frame and the new global
        end index; performs the rolling-window eviction (:358-373) when the slot would overflow."""
        kc = kv_cache["k"][0].view(-1, Dh)       # [cache_rows, heads_local*128]
        vc = kv_cache["v"][0].view(-1, Dh)
        kv_size = kc.shape[0]
        if mask is not None:
            # recompute branch (:305-348): positions 0..f-1, cache[:, :L] = K,V, block-causal mask
            local_start, local_end, start_frame, current_end = 0, L, 0, L
        else:
            # cache branch (:349-392)
            start_frame = current_start // fs
            current_end = current_start + L
            sink_tokens = sa.sink_size * fs
            g_end, l_end = int(kv_cache["global_end_index"]), int(kv_cache["local_end_index"])
            if sa.local_attn_size != -1 and current_end > g_end and L + l_end > kv_size:
                evicted = L + l_end - kv_size
                rolled = l_end - evicted - sink_tokens
                for c in (kc, vc):      # left-shift the window, keeping the sink tokens (:363-373)
                    ops.kv_roll(c, sink_tokens, sink_tokens + evicted, rolled)
                local_end = l_end + current_end - g_end - evicted
            else:
                local_end = l_end + current_end - g_end
            local_start = local_end - L
        if local_start < 0 or local_end > kv_size:
            raise RuntimeError(f"KV cache overflow: slot [{local_start}, {local_end}) of {kv_size}")
        return kc, vc, local_start, local_end, start_frame, current_end

    def _unmasked_attention(self, q, k, v, heads: int, out=None):
        """Attention without a mask (cache branch, cross-attention) on the tier ``attn_quant`` selects."""
        if self.attn_quant is None:
            return ops.attention(q, k, v, heads=heads, out=out)
        if self.attn_quant == "sage":
            return ops.sage_attention(q, k, v, heads=heads, out=out)
        raise ValueError(f"attn_quant must be 'sage' or None, got {self.attn_quant!r}")

    def _self_attention(self, blk: CausalWanAttentionBlock, h, grid, kv_cache, current_start, mask):
        """causal_model.py:218-397: projections, q/k RMSNorm, RoPE, cache write, attention.
        The cache slot is resolved first so the fused QKV GEMM writes its V third straight into
        the V cache (split output) and the RMSNorm+RoPE kernel writes K in place."""
        sa = blk.self_attn
        sp = self.sp
        n_loc, D = h.shape                       # local token rows
        L = n_loc if sp is None else n_loc * sp.world
        r0 = 0 if sp is None else sp.rank * n_loc
        heads = sa.num_heads if sp is None else sp.local_heads(sa.num_heads)
        Dh = heads * sa.head_dim                 # cache row width on this rank
        f, gh, gw = grid
        fs = gh * gw
        kc, vc, local_start, local_end, start_frame, current_end = self._cache_slot(sa, kv_cache, L, Dh, fs,
                                                                                    current_start, mask)
        k_slot, v_slot = kc[local_start:local_end], vc[local_start:local_end]
        if sp is not None and sp.p2p:
            # sequence-parallel, exchange done by the kernels: project MY rows (all heads); the RMSNorm+RoPE kernel
            # stores every head's columns straight into the owning rank's q buffer / K slot / V slot over NVLink;
            # after the barrier this rank attends ALL rows of ITS heads and scatters the output rows back
            if sa.fused_projections:
                qkv = _linear(h, sa.to_qkv)
                q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
            else:
                q = _linear(h, sa.q)
                k = _linear(h, sa.k)
                v = _linear(h, sa.v)
            q_full, o_heads, o_rows = sp.exchange_buffers(L)
            ops.qkv_norm_rope_p2p(q, k, v, sa.norm_q.weight, sa.norm_k.weight,
                                  sp.peer_ptrs(q_full[r0:]), Dh, sp.peer_ptrs(k_slot[r0:]), Dh,
                                  sp.peer_ptrs(v_slot[r0:]), Dh, sp.world, Dh, self._rope(h.device),
                                  head_dim=sa.head_dim, grid_h=gh, grid_w=gw, start_frame=start_frame, eps=sa.eps,
                                  row_offset=r0)
            kv_cache["global_end_index"] = current_end
            kv_cache["local_end_index"] = local_end
            sp.barrier()
            if mask is not None:
                pad = math.ceil(L / 128) * 128 - L
                ops.attention(q_full, kc[:L], vc[:L], heads=heads, block_len=mask.block_len, window=mask.window,
                              pad_keys=pad, out=o_heads)
            else:
                max_att = sa._max_attention_frames * fs if sa.local_attn_size == -1 else sa.local_attn_size * fs
                lo = max(0, local_end - max_att)
                self._unmasked_attention(q_full, kc[lo:local_end], vc[lo:local_end], heads, out=o_heads)
            ops.comm_scatter_rows(o_heads, sp.peer_ptrs(o_rows[:, sp.rank * Dh:]), D, n_loc, sp.world)
            sp.barrier()
            return o_rows
        if sp is not None:
            # sequence-parallel over torch.distributed collectives (NCCL baseline / gloo in the CPU tests): project
            # / normalise / rotate MY rows (all heads), then one
            # all-to-all per tensor turns them into ALL rows of MY heads; K and V are received
            # straight into this rank's head-sharded cache slot
            if sa.fused_projections:
                qkv = _linear(h, sa.to_qkv)
                q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
            else:
                q = _linear(h, sa.q)
                k = _linear(h, sa.k)
                v = _linear(h, sa.v)
            rq = torch.empty(n_loc, D, dtype=h.dtype, device=h.device)
            rk = torch.empty(n_loc, D, dtype=h.dtype, device=h.device)
            ops.qkv_norm_rope(q, k, None, sa.norm_q.weight, sa.norm_k.weight, rq, rk, None,
                              self._rope(h.device), head_dim=sa.head_dim, grid_h=gh, grid_w=gw,
                              start_frame=start_frame, eps=sa.eps, row_offset=r0)
            q_full = sp.rows_to_heads(rq)
            sp.rows_to_heads(rk, out=k_slot)
            sp.rows_to_heads(v.contiguous(), out=v_slot)
            kv_cache["global_end_index"] = current_end
            kv_cache["local_end_index"] = local_end
            if mask is not None:
                pad = math.ceil(L / 128) * 128 - L
                o = ops.attention(q_full, kc[:L], vc[:L], heads=heads, block_len=mask.block_len,
                                  window=mask.window, pad_keys=pad)
            else:
                max_att = sa._max_attention_frames * fs if sa.local_attn_size == -1 else sa.local_attn_size * fs
                lo = max(0, local_end - max_att)
                o = self._unmasked_attention(q_full, kc[lo:local_end], vc[lo:local_end], heads)
            return sp.heads_to_rows(o)
        if sa.fused_projections and (2 * D) % 256 == 0:
            qk = torch.empty(L, 2 * D, dtype=h.dtype, device=h.device)
            _linear(h, sa.to_qkv, out=qk, out2=v_slot, n_split=2 * D)
            q, k, v = qk[:, :D], qk[:, D:], None
        elif sa.fused_projections:
            qkv = _linear(h, sa.to_qkv)
            q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
        else:
            q = _linear(h, sa.q)
            k = _linear(h, sa.k)
            _linear(h, sa.v, out=v_slot)
            v = None
        rq = torch.empty(L, D, dtype=h.dtype, device=h.device)
        ops.qkv_norm_rope(q, k, v, sa.norm_q.weight, sa.norm_k.weight, rq, k_slot,
                          v_slot if v is not None else None, self._rope(h.device), head_dim=sa.head_dim,
                          grid_h=gh, grid_w=gw, start_frame=start_frame, eps=sa.eps)
        kv_cache["global_end_index"] = current_end
        kv_cache["local_end_index"] = local_end
        if mask is not None:
            pad = math.ceil(L / 128) * 128 - L
            return ops.attention(rq, kc[:L], vc[:L], heads=sa.num_heads, block_len=mask.block_len,
                                 window=mask.window, pad_keys=pad)
        max_att = sa._max_attention_frames * fs if sa.local_attn_size == -1 else sa.local_attn_size * fs
        lo = max(0, local_end - max_att)
        return self._unmasked_attention(rq, kc[lo:local_end], vc[lo:local_end], sa.num_heads)

    def _cross_attention(self, blk: CausalWanAttentionBlock, h, ctx, cache):
        """wan/modules/model.py:171-228 (K/V of the prompt computed once, cached by assignment)."""
        ca = blk.cross_attn
        D = self.dim
        q = _linear(h, ca.q)
        ops.rmsnorm(q, ca.norm_q.weight, ca.eps, out=q)
        if cache is not None and cache["is_init"]:
            k, v = cache["k"], cache["v"]
        else:
            k = _linear(ctx, ca.k)
            ops.rmsnorm(k, ca.norm_k.weight, ca.eps, out=k)
            v = _linear(ctx, ca.v)
            k = k.view(1, -1, ca.num_heads, ca.head_dim)
            v = v.view(1, -1, ca.num_heads, ca.head_dim)
            if cache is not None:
                cache["is_init"] = True
                cache["k"], cache["v"] = k, v
        return self._unmasked_attention(q, k[0].reshape(-1, D), v[0].reshape(-1, D), ca.num_heads)

    # -- whole block as ONE C-ABI call (kr_dit_block_fwd) ---------------------------------------------------------
    # Opt-in (KR_BLOCK_FWD=1 or ``model.use_block_fwd = True``): the C function issues exactly the launches of the
    # per-op schedule below (tests/test_block_fwd_cpu.py compares the two launch sequences call by call); what changes
    # is the host side — one ctypes crossing per block instead of 14 and no temporary tensors.
    def _block_fwd_eligible(self, blk: CausalWanAttentionBlock, x, crossattn_cache) -> bool:
        sa, ca = blk.self_attn, blk.cross_attn
        return (self.sp is None and self.attn_quant is None and x.dtype == torch.bfloat16 and sa.fused_projections and (2 * self.dim) % 256 == 0
                and sa.qk_norm and ca.qk_norm and crossattn_cache is not None and bool(crossattn_cache["is_init"])
                and getattr(ops, "_prof", None) is None
                # not inside a CUDA-graph capture: the scratch workspace is cached across calls and must not come from
                # a capture's private memory pool
                and not (x.is_cuda and torch.cuda.is_current_stream_capturing())
                and not any(hasattr(m, "_kr_fp8") for m in (sa.to_qkv, sa.o, ca.q, ca.o, blk.ffn[0], blk.ffn[2])))

    def _block_one_call(self, blk: CausalWanAttentionBlock, x, e0, grid, kv_cache, crossattn_cache, current_start, mask):
        sa, ca = blk.self_attn, blk.cross_attn
        L, D = x.shape
        _, gh, gw = grid
        fs = gh * gw
        kc, vc, local_start, local_end, start_frame, current_end = self._cache_slot(sa, kv_cache, L, D, fs,
                                                                                    current_start, mask)
        if mask is not None:
            lo, block_len, window, pad = 0, mask.block_len, mask.window, math.ceil(L / 128) * 128 - L
        else:
            max_att = sa._max_attention_frames * fs if sa.local_attn_size == -1 else sa.local_attn_size * fs
            lo, block_len, window, pad = max(0, local_end - max_att), 0, 0, 0
        n3 = blk.norm3 if isinstance(blk.norm3, nn.LayerNorm) else None
        ops.dit_block_fwd(
            x, e0, blk.modulation, self._rope(x.device),
            w_qkv=sa.to_qkv.weight, b_qkv=sa.to_qkv.bias, norm_q=sa.norm_q.weight, norm_k=sa.norm_k.weight,
            w_o=sa.o.weight, b_o=sa.o.bias, k_cache=kc, v_cache=vc, local_start=local_start, local_end=local_end,
            attn_lo=lo, norm3_w=None if n3 is None else n3.weight, norm3_b=None if n3 is None else n3.bias,
            w_cq=ca.q.weight, b_cq=ca.q.bias, norm_cq=ca.norm_q.weight,
            ck=crossattn_cache["k"][0].reshape(-1, D), cv=crossattn_cache["v"][0].reshape(-1, D),
            w_co=ca.o.weight, b_co=ca.o.bias, w_ffn0=blk.ffn[0].weight, b_ffn0=blk.ffn[0].bias,
            w_ffn2=blk.ffn[2].weight, b_ffn2=blk.ffn[2].bias, heads=sa.num_heads, rows_per_frame=fs, grid_h=gh,
            grid_w=gw, start_frame=start_frame, eps_block=blk.eps, eps_qk=sa.eps,
            eps_norm3=0.0 if n3 is None else n3.eps, eps_cross=ca.eps, block_len=block_len, window=window, pad_keys=pad)
        kv_cache["global_end_index"] = current_end
        kv_cache["local_end_index"] = local_end
        return x

    def _block(self, blk: CausalWanAttentionBlock, x, e0, grid, ctx, kv_cache, crossattn_cache,
               current_start, mask):
        """causal_model.py:440-492; x [L, D] is updated in place."""
        fs = grid[1] * grid[2]
        if self.use_block_fwd and self._block_fwd_eligible(blk, x, crossattn_cache):
            return self._block_one_call(blk, x, e0, grid, kv_cache, crossattn_cache, current_start, mask)
        r0 = 0 if self.sp is None else self.sp.rank * x.shape[0]       # global index of my first row
        emod = ops.add_modulation(blk.modulation, e0)                    # [F, 6, D]
        h = ops.ln_modulate(x, eps=blk.eps, mod=emod, shift_idx=0, scale_idx=1, rows_per_frame=fs,
                            row_offset=r0)
        y = self._self_attention(blk, h, grid, kv_cache, current_start, mask)
        sa = blk.self_attn
        _linear(y, sa.o, epilogue=ops.EPI_BIAS_GATE_RES, residual=x,
                 gate=emod[:, 2], rows_per_gate=fs, out=x, row_offset=r0)
        n3 = blk.norm3
        if isinstance(n3, nn.LayerNorm):
            hc = ops.ln_modulate(x, eps=n3.eps, weight=n3.weight, bias=n3.bias, out=h)
        else:
            hc = x          # cross_attn_norm=False: the residual stream itself; `h` stays the scratch buffer
        y = self._cross_attention(blk, hc, ctx, crossattn_cache)
        ca = blk.cross_attn
        _linear(y, ca.o, epilogue=ops.EPI_BIAS_RES, residual=x, out=x)
        h = ops.ln_modulate(x, eps=blk.eps, mod=emod, shift_idx=3, scale_idx=4, rows_per_frame=fs, out=h,
                            row_offset=r0)
        hid = _linear(h, blk.ffn[0], epilogue=ops.EPI_BIAS_GELU)
        _linear(hid, blk.ffn[2], epilogue=ops.EPI_BIAS_GATE_RES, residual=x,
                 gate=emod[:, 5], rows_per_gate=fs, out=x, row_offset=r0)
        return x

    # ----------------------------------------------------------------------------------------
    def forward_tokens(self, x: torch.Tensor, t: torch.Tensor, context: torch.Tensor, kv_cache,
                       crossattn_cache, current_start: int = 0):
        """One sample: x [C, F, H, W] (any strides), t [F], context [<=512, text_dim] ->
        head output [F*h*w, prod(patch)*out_dim] plus the token grid."""
        dt = self.patch_embedding.weight.dtype
        C, Fr, H, W = x.shape
        grid = (Fr, H // self.patch_size[1], W // self.patch_size[2])
        tok = ops.patchify(x.to(dt))
        r0 = 0
        if self.sp is not None:                      # my contiguous share of the token rows
            r0, n_loc = self.sp.rows(tok.shape[0])
            tok = tok[r0:r0 + n_loc]
        pw = self.patch_embedding.weight.view(self.dim, -1)
        xs = ops.gemm(tok, pw, self.patch_embedding.bias)                                   # [L, D]
        # time embeddings (causal_model.py:888-892): sinusoid in fp64 (model.py:15-24), bf16 MLPs
        half = self.freq_dim // 2
        pos = t.flatten().to(torch.float64)
        sinus = torch.outer(pos, torch.pow(10000, -torch.arange(half, dtype=torch.float64,
                                                                 device=pos.device).div(half)))
        emb = torch.cat([torch.cos(sinus), torch.sin(sinus)], dim=1).to(dt)
        te, tp = self.time_embedding, self.time_projection
        e = ops.gemm(ops.activation(ops.gemm(emb, te[0].weight, te[0].bias), "silu"), te[2].weight, te[2].bias)
        e0 = ops.gemm(ops.activation(e, "silu"), tp[1].weight, tp[1].bias).view(Fr, 6, self.dim)
        pp = self.pp
        if pp is not None and self.sp is not None:
            raise RuntimeError("layer pipeline and sequence parallelism are alternative multi-GPU modes")
        lo, hi = (0, len(self.blocks)) if pp is None else pp.layers(len(self.blocks))
        mine = range(lo, hi)                          # the blocks this rank runs (all of them on one GPU)
        need_text = crossattn_cache is None or not all(crossattn_cache[i]["is_init"] for i in mine)
        ctx = self._embed_text(context) if need_text else None
        mask = self.block_mask
        if pp is not None and not pp.first:
            xs = pp.recv_from_previous(xs)            # residual stream after the previous stage's layers
        for i in mine:
            xs = self._block(self.blocks[i], xs, e0, grid, ctx, kv_cache[i],
                             crossattn_cache[i] if crossattn_cache is not None else None,
                             current_start, mask)
        if pp is not None and not pp.last:
            pp.send_to_next(xs)
        # head (causal_model.py:512-523, :951)
        fs = grid[1] * grid[2]
        if pp is None or pp.last:
            ehead = ops.add_modulation(self.head.modulation, e.view(Fr, 1, self.dim).expand(Fr, 2, self.dim).contiguous())
            h = ops.ln_modulate(xs, eps=self.head.eps, mod=ehead, shift_idx=0, scale_idx=1, rows_per_frame=fs,
                                row_offset=r0)
            out = ops.gemm(h, self.head.head.weight, self.head.head.bias)
        else:
            out = torch.empty(xs.shape[0], self.head.head.weight.shape[0], dtype=xs.dtype, device=xs.device)
        if pp is not None:
            out = pp.broadcast_from_last(out)        # every rank carries the denoising loop on
        if self.sp is not None:
            out = self.sp.gather_rows(out)           # every rank needs the full latent for the next step
        return out, grid

    def _forward_inference(self, x, t, context, seq_len, clip_fea=None, y=None, kv_cache=None,
                           crossattn_cache=None, current_start: int = 0, cache_start: int = 0):
        """causal_model.py:825-954.  x [B, C, F, H, W]; t [B, F]; context list/tensor of
        [L_text, text_dim]; returns flow [B, C_out, F, H, W]."""
        if kv_cache is None:
            raise NotImplementedError("the no-cache (training) forward is outside the hot path")
        outs = []
        for b in range(len(x)):
            xb = x[b]
            C, Fr, H, W = xb.shape
            assert (Fr * (H // 2) * (W // 2)) <= seq_len
            kv_b = kv_cache if len(x) == 1 else [
                {"k": c["k"][b:b + 1], "v": c["v"][b:b + 1], "global_end_index": c["global_end_index"],
                 "local_end_index": c["local_end_index"]} for c in kv_cache]
            head_out, _ = self.forward_tokens(xb, t[b], context[b], kv_b, crossattn_cache, current_start)
            if len(x) > 1:
                for c, cb in zip(kv_cache, kv_b):
                    if b == len(x) - 1:
                        c["global_end_index"], c["local_end_index"] = cb["global_end_index"], cb["local_end_index"]
            flow, _ = ops.unpatchify_x0(head_out, None, None, self.out_dim, Fr, H, W)   # [F, C, H, W]
            outs.append(flow.permute(1, 0, 2, 3))
        return torch.stack(outs)

    def forward(self, *args, **kwargs):
        return self._forward_inference(*args, **kwargs)
