"""UMT5 text encoder (SURVEY.md §8f.3) on the sm_90a kernels: the reference's ``T5Encoder`` with
``shared_pos=False`` (wan/modules/t5.py:267-313; umt5-xxl: dim 4096, 64 heads x 64, ffn 10240, 24 layers,
32 relative-position buckets, :456-469).  Off the per-frame path — it runs once per prompt / prompt change
(release_server.py:459-468, :642) — so the schedule favours reuse of the existing kernels over launch count:

  T5LayerNorm (RMS, no mean subtraction, :53-66)        -> kr_rmsnorm
  q|k projection, V^T projection, o / fc2 (+ residual)  -> kr_gemm (no biases anywhere in T5)
  per head: scores = q_h k_h^T (T5 does not scale)      -> kr_gemm (bf16 scores, as the reference's einsum)
            + relative-position bias + key padding mask -> tensor add (host-side torch op on [L, L])
            softmax in fp32 -> bf16 (:110-111)          -> kr_softmax_rows
            o_h = P V_h                                 -> kr_gemm against the rows of V^T
  FFN: fc2(fc1(x) * gelu_tanh(gate(x)))  (:123-141)     -> kr_gemm (+GELU epilogue), tensor multiply

The module keeps the reference's state-dict keys (``token_embedding.weight``, ``blocks.N.{norm1,norm2}.weight``,
``blocks.N.attn.{q,k,v,o}.weight``, ``blocks.N.pos_embedding.embedding.weight``,
``blocks.N.ffn.{gate.0,fc1,fc2}.weight``, ``norm.weight``) so the umt5-xxl checkpoint loads unchanged.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
from torch import nn

from . import ops

UMT5_XXL = dict(vocab=256384, dim=4096, dim_attn=4096, dim_ffn=10240, num_heads=64, num_layers=24, num_buckets=32)


def relative_position_bucket(lq: int, lk: int, num_buckets: int = 32, max_dist: int = 128,
                             device=None) -> torch.Tensor:
    """Bidirectional T5 buckets of rel = key - query (t5.py:233-264) -> int64 [lq, lk]."""
    rel = torch.arange(lk, device=device)[None, :] - torch.arange(lq, device=device)[:, None]
    nb = num_buckets // 2
    buckets = (rel > 0).long() * nb
    rel = rel.abs()
    max_exact = nb // 2
    large = max_exact + (torch.log(rel.float() / max_exact) / math.log(max_dist / max_exact) * (nb - max_exact)).long()
    large = torch.min(large, torch.full_like(large, nb - 1))
    return buckets + torch.where(rel < max_exact, rel, large)


class T5LayerNorm(nn.Module):
    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.dim, self.eps = dim, eps
        self.weight = nn.Parameter(torch.ones(dim))


class T5Attention(nn.Module):
    def __init__(self, dim, dim_attn, num_heads):
        super().__init__()
        assert dim_attn % num_heads == 0
        self.dim, self.dim_attn, self.num_heads, self.head_dim = dim, dim_attn, num_heads, dim_attn // num_heads
        self.q = nn.Linear(dim, dim_attn, bias=False)
        self.k = nn.Linear(dim, dim_attn, bias=False)
        self.v = nn.Linear(dim, dim_attn, bias=False)
        self.o = nn.Linear(dim_attn, dim, bias=False)


class T5FeedForward(nn.Module):
    def __init__(self, dim, dim_ffn):
        super().__init__()
        self.dim, self.dim_ffn = dim, dim_ffn
        self.gate = nn.Sequential(nn.Linear(dim, dim_ffn, bias=False), nn.GELU(approximate="tanh"))
        self.fc1 = nn.Linear(dim, dim_ffn, bias=False)
        self.fc2 = nn.Linear(dim_ffn, dim, bias=False)


class T5RelativeEmbedding(nn.Module):
    def __init__(self, num_buckets, num_heads):
        super().__init__()
        self.num_buckets, self.num_heads = num_buckets, num_heads
        self.embedding = nn.Embedding(num_buckets, num_heads)


class T5SelfAttention(nn.Module):
    def __init__(self, dim, dim_attn, dim_ffn, num_heads, num_buckets):
        super().__init__()
        self.norm1 = T5LayerNorm(dim)
        self.attn = T5Attention(dim, dim_attn, num_heads)
        self.norm2 = T5LayerNorm(dim)
        self.ffn = T5FeedForward(dim, dim_ffn)
        self.pos_embedding = T5RelativeEmbedding(num_buckets, num_heads)


class T5Encoder(nn.Module):
    """``forward(ids [B, L] int64, mask [B, L] or None) -> [B, L, dim]`` in the dtype of the weights (bf16)."""

    def __init__(self, vocab, dim, dim_attn, dim_ffn, num_heads, num_layers, num_buckets, shared_pos=False,
                 dropout=0.1):
        super().__init__()
        if shared_pos:
            raise NotImplementedError("UMT5 uses per-layer position embeddings (shared_pos=False)")
        self.dim, self.dim_attn, self.dim_ffn = dim, dim_attn, dim_ffn
        self.num_heads, self.num_layers, self.num_buckets = num_heads, num_layers, num_buckets
        self.token_embedding = nn.Embedding(vocab, dim)
        self.blocks = nn.ModuleList([T5SelfAttention(dim, dim_attn, dim_ffn, num_heads, num_buckets)
                                     for _ in range(num_layers)])
        self.norm = T5LayerNorm(dim)
        self._bias_delta = None         # ((L, device, dtype), [layers][heads, 2L-1])

    def _bias_by_offset(self, L: int, device, dtype):
        """Per layer, the relative-position bias as a function of the offset k - q (t5.py:221-264): row d of the
        [2L-1] table is embedding[bucket(d - (L-1))].  Gathered once per (L, device, dtype) — the weights are static —
        so the layer loop below issues kernels only."""
        key = (L, str(device), dtype)
        if self._bias_delta is None or self._bias_delta[0] != key:
            b = relative_position_bucket(L, L, self.num_buckets, device=device)          # [L, L] buckets of k - q
            by_offset = torch.cat([b[L - 1, :L - 1], b[0, :]])                              # offsets -(L-1) .. L-1
            tabs = [blk.pos_embedding.embedding.weight.to(dtype)[by_offset].t().contiguous() for blk in self.blocks]
            self._bias_delta = (key, tabs)
        return self._bias_delta[1]

    def _encode_one(self, ids: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
        """ids [L], mask [L] or None -> [L, dim].  Per layer: rmsnorm, q/k/v GEMMs, ONE attention launch
        (kr_t5_attn: bias + mask + fp32 softmax in the kernel), o GEMM (+residual), rmsnorm, gate GEMM (GELU),
        fc1 GEMM (x gate in the epilogue), fc2 GEMM (+residual) — no torch arithmetic."""
        dt = self.token_embedding.weight.dtype
        if ids.is_cuda and dt != torch.bfloat16:
            raise TypeError(f"T5Encoder runs on bf16 weights (the server casts it: release_server.py:141 "
                            f"text_encoder.to(dtype=torch.bfloat16)); got {dt}")
        L = ids.shape[0]
        n = self.num_heads
        x = self.token_embedding.weight[ids].contiguous()                     # [L, dim]
        tabs = self._bias_by_offset(L, x.device, dt)
        km = None if mask is None else (mask != 0).to(torch.uint8).contiguous()
        for blk, bias_delta in zip(self.blocks, tabs):
            at = blk.attn
            h = ops.rmsnorm(x, blk.norm1.weight, blk.norm1.eps)
            q = ops.gemm(h, at.q.weight, None)                                # [L, dim_attn]
            k = ops.gemm(h, at.k.weight, None)
            v = ops.gemm(h, at.v.weight, None)
            o = ops.t5_attention(q, k, v, bias_delta, km, heads=n)
            ops.gemm(o, at.o.weight, None, epilogue=ops.EPI_BIAS_RES, residual=x, out=x)
            h = ops.rmsnorm(x, blk.norm2.weight, blk.norm2.eps)
            g = ops.gemm(h, blk.ffn.gate[0].weight, None, epilogue=ops.EPI_BIAS_GELU)
            f = ops.gemm(h, blk.ffn.fc1.weight, None, epilogue=ops.EPI_MUL, residual=g)      # fc1(x) * gelu(gate(x))
            ops.gemm(f, blk.ffn.fc2.weight, None, epilogue=ops.EPI_BIAS_RES, residual=x, out=x)
        return ops.rmsnorm(x, self.norm.weight, self.norm.eps)

    @torch.no_grad()
    def forward(self, ids: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        outs = [self._encode_one(ids[b], None if mask is None else mask[b]) for b in range(ids.shape[0])]
        return torch.stack(outs)


def umt5_xxl_encoder(device=None, dtype=torch.bfloat16, **overrides) -> T5Encoder:
    """T5Encoder with the umt5-xxl dimensions (t5.py:456-469), parameters allocated on ``device``."""
    cfg = dict(UMT5_XXL)
    cfg.update(overrides)
    prev = torch.get_default_dtype()
    try:
        torch.set_default_dtype(dtype)
        if device is not None:
            with torch.device(device):
                m = T5Encoder(**cfg)
        else:
            m = T5Encoder(**cfg)
    finally:
        torch.set_default_dtype(prev)
    return m.eval().requires_grad_(False)
