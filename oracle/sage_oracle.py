"""TEST INFRASTRUCTURE — torch oracle for the quantised attention tier (kr_sage_quantize / kr_sage_attn; not shipped,
only tests/ import it).  Runs on CPU or CUDA tensors.

Parity unpinned: the reference's H100 attention backend is the sageattention 2.2.1 wheel
(``sageattn_qk_int8_pv_fp8_cuda_sm90`` with ``qk_quant_gran="per_thread"``, ``smooth_k=True``,
``pv_accum_dtype="fp32+fp32"``), which is built for CPython 3.11 with sm_90 binaries only: it cannot be loaded under
Python 3.12 and is not available where the GPU tests run.  This module restates its published algorithm (the
wheel's ``core.py`` and ``triton/quant_per_thread.py``) as the numerics contract the kernels share:

* K smoothing: ``k_mean = bf16(mean over the Lkv rows)`` per channel, ``k_s = bf16(k - k_mean)`` (softmax is invariant
  to a per-channel shift of every key).
* Q, K -> INT8 per thread: ``scale = amax / 127 + 1e-7``, ``x_i8 = trunc(x / scale + 0.5 sign(x))`` in fp32.  A Q group
  is (head, 16-row block b, t < 8) = rows 16b+t and 16b+8+t; a K group is (head, 128-key block c, t < 4) = keys
  128c + 8i + 2t + e (i < 16, e < 2): exactly the rows / columns one thread holds in the wgmma S fragment.
* V -> e4m3 per channel: ``v_scale = max(amax, 1e-12) / 448``, ``v8 = e4m3_satfinite(v / v_scale)``, stored transposed
  with the keys of every 16 in the order ``PERM``.
* Attention over 128-key tiles in order: ``S = s32(q_i8 k_i8^T) * (q_scale * softmax_scale * log2 e) * k_scale``, exact
  running max, ``P = exp2(S - m)``, ``l += sum P`` (unquantised), ``O = O * alpha + e4m3(448 P) @ v8`` in fp32,
  ``out = bf16(O * v_scale / (448 l))``.  The P scale and the accumulation cadence are this project's stated choice
  (the wheel's kernel is binary-only).
"""
from __future__ import annotations

import math

import torch

E4M3_MAX = 448.0
LOG2E = 1.4426950408889634
# stored position p of every 16 keys holds key PERM[p]: the k32 e4m3 register-A layout of a thread's S fragment
PERM = [0, 1, 8, 9, 2, 3, 10, 11, 4, 5, 12, 13, 6, 7, 14, 15]


def q_group_rows(b: int, t: int) -> list:
    """Rows of Q scale group (b, t)."""
    return [16 * b + t, 16 * b + 8 + t]


def k_group_keys(c: int, t: int) -> list:
    """Keys of K scale group (c, t)."""
    return [128 * c + 8 * i + 2 * t + e for i in range(16) for e in range(2)]


def permute_keys(x: torch.Tensor) -> torch.Tensor:
    """[..., n*16] in key order -> stored order (position p of every 16 holds key PERM[p])."""
    n = x.shape[-1] // 16
    idx = (torch.arange(n)[:, None] * 16 + torch.tensor(PERM)[None, :]).flatten().to(x.device)
    return x.index_select(-1, idx)


def unpermute_keys(x: torch.Tensor) -> torch.Tensor:
    """Inverse of :func:`permute_keys`."""
    inv = [PERM.index(k) for k in range(16)]
    n = x.shape[-1] // 16
    idx = (torch.arange(n)[:, None] * 16 + torch.tensor(inv)[None, :]).flatten().to(x.device)
    return x.index_select(-1, idx)


def _div(x: torch.Tensor, d: float) -> torch.Tensor:
    """x / d as an IEEE fp32 division on every device (torch turns a CUDA tensor / python scalar into a multiplication
    by the reciprocal)."""
    return x / torch.full_like(x, d)


def _quant_i8(x: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    return torch.trunc(x / scale + 0.5 * torch.sign(x)).to(torch.int8)


def e4m3(x: torch.Tensor) -> torch.Tensor:
    """Round to nearest even, saturating (float8_e4m3fn)."""
    return x.clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def k_mean_of(k: torch.Tensor) -> torch.Tensor:
    """bf16 of the fp64 mean over the rows: k [Lkv, W] -> [W] bf16."""
    return k.double().mean(0).to(torch.bfloat16)


def quantize(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, k_mean: torch.Tensor | None = None,
             smooth: bool = True) -> dict:
    """q [Lq, heads*128], k / v [Lkv, heads*128] bf16 -> the buffers of kr_sage_quantize (same shapes and bytes):
    q_i8 int8 [Lq, W], q_scale fp32 [heads, nqb, 8], k_mean bf16 [W], k_i8 int8 [Lkv, W], k_scale fp32 [heads, nkb, 4],
    v_t8 uint8 (e4m3 bits) [W, nkb*128], v_scale fp32 [W].  ``k_mean`` defaults to :func:`k_mean_of`; ``smooth=False``
    quantises K without subtracting a mean (for comparison only)."""
    Lq, W = q.shape
    Lkv = k.shape[0]
    H = heads
    nqb, nkb = (Lq + 15) // 16, (Lkv + 127) // 128
    dev = q.device
    # Q
    x = torch.zeros(nqb * 16, W, dtype=torch.float32, device=dev)
    x[:Lq] = q.float()
    xg = x.view(nqb, 2, 8, H, 128)                                   # row = 16b + 8r + t
    q_scale = _div(xg.abs().amax(dim=(1, 4)), 127) + 1e-7                  # [nqb, 8, H]
    q_i8 = _quant_i8(xg, q_scale[:, None, :, :, None]).view(nqb * 16, W)[:Lq].contiguous()
    q_scale = q_scale.permute(2, 0, 1).contiguous()                   # [H, nqb, 8]
    # K
    if k_mean is None:
        k_mean = k_mean_of(k) if smooth else torch.zeros(W, dtype=torch.bfloat16, device=dev)
    ks = torch.zeros(nkb * 128, W, dtype=torch.float32, device=dev)
    ks[:Lkv] = (k - k_mean[None, :]).float()                          # torch's bf16 subtraction
    kg = ks.view(nkb, 16, 4, 2, H, 128)                               # key = 128c + 8i + 2t + e
    k_scale = _div(kg.abs().amax(dim=(1, 3, 5)), 127) + 1e-7               # [nkb, 4, H]
    k_i8 = _quant_i8(kg, k_scale[:, None, :, None, :, None]).view(nkb * 128, W)[:Lkv].contiguous()
    k_scale = k_scale.permute(2, 0, 1).contiguous()                   # [H, nkb, 4]
    # V
    v_scale = _div(v.float().abs().amax(0).clamp(min=1e-12), E4M3_MAX)
    v8 = torch.zeros(nkb * 128, W, dtype=torch.float8_e4m3fn, device=dev)
    v8[:Lkv] = e4m3(v.float() / v_scale[None, :])
    v_t8 = permute_keys(v8.view(torch.uint8).t()).contiguous()       # [W, nkb*128]
    return dict(q_i8=q_i8, q_scale=q_scale, k_mean=k_mean, k_i8=k_i8, k_scale=k_scale, v_t8=v_t8, v_scale=v_scale)


def attention_from_quantized(buf: dict, Lq: int, Lkv: int, heads: int, softmax_scale: float | None = None) -> torch.Tensor:
    """The kernel's attention on given quantised buffers -> bf16 [Lq, heads*128]."""
    H = heads
    W = H * 128
    nkb = (Lkv + 127) // 128
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(128)
    dev = buf["q_i8"].device
    sl2 = torch.tensor(softmax_scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    rows = torch.arange(Lq, device=dev)
    qs = buf["q_scale"][:, rows // 16, rows % 8] * sl2.to(dev)                      # [H, Lq]
    keys = torch.arange(128, device=dev)
    qf = buf["q_i8"].view(Lq, H, 128).permute(1, 0, 2).double()                     # [H, Lq, 128]
    kf = buf["k_i8"].view(Lkv, H, 128).permute(1, 0, 2).double()                    # [H, Lkv, 128]
    v8 = unpermute_keys(buf["v_t8"]).view(torch.float8_e4m3fn).float()              # [W, nkb*128] key order
    v8 = v8.view(H, 128, nkb * 128).transpose(1, 2)                                  # [H, keys, 128]
    m = torch.full((H, Lq, 1), -math.inf, dtype=torch.float32, device=dev)
    l = torch.zeros(H, Lq, 1, dtype=torch.float32, device=dev)
    o = torch.zeros(H, Lq, 128, dtype=torch.float32, device=dev)
    for c in range(nkb):
        k0, k1 = 128 * c, min(128 * c + 128, Lkv)
        acc = torch.bmm(qf, kf[:, k0:k1].transpose(1, 2)).float()                  # exact: |acc| < 2^24
        ks = buf["k_scale"][:, c, (keys[:k1 - k0] // 2) % 4]                        # [H, n]
        s = acc * (qs[:, :, None] * ks[:, None, :])
        m_new = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp2(m - m_new)
        p = torch.exp2(s - m_new)
        l = l * alpha + p.sum(-1, keepdim=True)
        pt = e4m3(p * E4M3_MAX).float()
        o = o * alpha + torch.bmm(pt.double(), v8[:, k0:k1].double()).float()
        m = m_new
    out = o * buf["v_scale"].view(H, 1, 128) * (1.0 / (E4M3_MAX * l))
    return out.permute(1, 0, 2).reshape(Lq, W).to(torch.bfloat16)


def sage_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, softmax_scale: float | None = None,
                   smooth: bool = True) -> torch.Tensor:
    """quantize + attention_from_quantized."""
    buf = quantize(q, k, v, heads, smooth=smooth)
    return attention_from_quantized(buf, q.shape[0], k.shape[0], heads, softmax_scale)


def exact_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int,
                    softmax_scale: float | None = None) -> torch.Tensor:
    """fp32 softmax(scale q k^T) v, [Lq, heads*128] -> fp32."""
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(128)
    Lq, Lkv = q.shape[0], k.shape[0]
    qf = q.float().view(Lq, heads, 128).transpose(0, 1)
    kf = k.float().view(Lkv, heads, 128).transpose(0, 1)
    vf = v.float().view(Lkv, heads, 128).transpose(0, 1)
    p = torch.softmax(torch.bmm(qf, kf.transpose(1, 2)) * softmax_scale, dim=-1)
    return torch.bmm(p, vf).transpose(0, 1).reshape(Lq, heads * 128)
