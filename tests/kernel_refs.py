"""Float64 restatements of single kernels, shared by the per-kernel GPU parity tests and checked on the CPU by
``tests/test_kernel_refs_cpu.py`` against ``oracle/dit_oracle.py``, ``oracle/vae_oracle.py`` and torch.

Every function computes in float64 on the device of its inputs and rounds to the 16-bit storage type exactly at
the points the kernel's header comment names (``r16``), so a correct kernel differs from it only where its fp32
arithmetic lands on the other side of a 16-bit rounding boundary: at most one unit in the last place (``ulp``).
Each function also returns the unrounded float64 value where a test bounds the whole rounding chain.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import dit_oracle as O
from oracle import vae_oracle as V

F64 = torch.float64
_MANT = {torch.bfloat16: 7, torch.float16: 10}


def r16(x: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """Round a float64 tensor to ``dtype`` (round-to-nearest-even) and return it as float64."""
    return x.to(dtype).to(F64)


def ulp(x: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """Spacing of ``dtype`` values at |x| (float64; the smallest normal spacing at 0)."""
    tiny = torch.finfo(dtype).tiny
    e = torch.floor(torch.log2(x.double().abs().clamp_min(tiny)))
    return torch.exp2(e - _MANT[dtype])


def ulp_excess(got: torch.Tensor, ref: torch.Tensor, dtype=torch.bfloat16):
    """(max |got - ref| / ulp(ref), fraction of elements that are not bit-identical)."""
    g, r = got.double(), ref.double()
    d = (g - r).abs()
    return float((d / ulp(r, dtype)).max()), float((d != 0).double().mean())


# ---------------------------------------------------------------------------------------------
# kr_dit_elem.cu
# ---------------------------------------------------------------------------------------------
def ln_modulate(x, eps, weight=None, bias=None, mod=None, shift_idx=0, scale_idx=1, rows_per_frame=0,
                row_offset=0):
    """y = r16(LN(x) [* w + b]);  out = r16(r16(y * r16(1 + scale[f])) + shift[f]),  f = (row + row_offset) // rpf.
    Returns (out, exact, prod): ``exact`` without any rounding, ``prod`` = y * (1 + scale) (float64 magnitudes of the
    product rounding point, for the rounding-chain bound)."""
    xd = x.double()
    w = None if weight is None else weight.double()
    b = None if bias is None else bias.double()
    exact = O.layer_norm(xd, eps, w, b)
    y = r16(exact)
    if mod is None:
        return y, exact, exact
    f = (torch.arange(x.shape[0], device=x.device) + row_offset) // rows_per_frame
    sc, sh = mod[f, scale_idx].double(), mod[f, shift_idx].double()
    prod = y * r16(1 + sc)
    return r16(r16(prod) + sh), exact * (1 + sc) + sh, prod


def rope_table_f32(head_dim: int, device) -> torch.Tensor:
    """The kernel's (cos, sin) float32 table [1024, head_dim/2, 2] built from the oracle's angles."""
    a = O.rope_table(head_dim)
    return torch.stack([a.cos(), a.sin()], dim=-1).float().contiguous().to(device)


def qk_norm_rope(x, weight, eps, head_dim, grid_h, grid_w, start_frame=0):
    """One of q / k: r16(rope(r16(r16(x * rsqrt(mean x^2 + eps)) * w))) over rows [0, L), L a multiple of
    grid_h * grid_w (row r is frame r // (h*w) + start_frame, row (r % (h*w)) // w, column r % w).
    Returns (rounded, exact)."""
    L, D = x.shape
    hw = grid_h * grid_w
    assert L % hw == 0
    grid = (L // hw, grid_h, grid_w)
    ang = O.rope_table(head_dim).to(x.device)
    xd = x.double()
    n = O.rms_norm(xd, torch.ones(D, dtype=F64, device=x.device), eps)
    a = r16(r16(n) * weight.double())
    out = O.rope_apply(a.view(L, D // head_dim, head_dim), grid, ang, start_frame).reshape(L, D)
    exact = O.rope_apply((n * weight.double()).view(L, D // head_dim, head_dim), grid, ang,
                         start_frame).reshape(L, D)
    return r16(out), exact


def rmsnorm(x, weight, eps):
    """r16(r16(x * rsqrt(mean x^2 + eps)) * w) (model.py:69-85 in bf16)."""
    xd = x.double()
    n = O.rms_norm(xd, torch.ones(x.shape[-1], dtype=F64, device=x.device), eps)
    return r16(r16(n) * weight.double())


def silu(x):
    return F.silu(x.double())


def gelu_tanh(x):
    return F.gelu(x.double(), approximate="tanh")


def patchify(x):
    """x [C, F, H, W] -> [F*(H/2)*(W/2), 4C] in the Conv3d(1,2,2) weight order (c, ph, pw)
    (causal_model.py:614-615: the conv is a matmul of these rows with weight.flatten(1))."""
    C, Fr, H, W = x.shape
    t = x.reshape(C, Fr, H // 2, 2, W // 2, 2).permute(1, 2, 4, 0, 3, 5)    # f, hh, ww, c, ph, pw
    return t.reshape(Fr * (H // 2) * (W // 2), C * 4)


def unpatchify(head_out, C, Fr, H, W):
    """head_out [F*h2*w2, 4C] with column order (ph, pw, c) -> [F, C, H, W] (causal_model.py:1145-1147)."""
    u = head_out.reshape(Fr, H // 2, W // 2, 2, 2, C)                       # f, hh, ww, ph, pw, c
    return u.permute(0, 5, 1, 3, 2, 4).reshape(Fr, C, H, W)


def flow_to_x0(flow, xt, sigma):
    """bf16(double(xt) - sigma[f] * double(flow)) (utils/wan_wrapper.py:181-205), sigma [F] float64."""
    return (xt.double() - sigma.double().view(-1, 1, 1, 1) * flow.double()).to(flow.dtype)


# ---------------------------------------------------------------------------------------------
# kr_attn.cu
# ---------------------------------------------------------------------------------------------
def attention(q, k, v, heads, block_len=0, window=0, pad_keys=0, softmax_scale=None):
    """softmax(scale * q k^T) v per head in float64 -> [Lq, heads*128] float64.

    With ``block_len`` the keys are right-padded with ``pad_keys`` zero rows (score 0, value 0) and the block-causal
    rule of the oracle (``kv < ends[q]``, optional ``kv >= ends[q] - window``) is applied over the padded length, as
    causal_model.py:316-348 pads before FlexAttention."""
    Lq, Lkv = q.shape[0], k.shape[0]
    d = 128
    scale = 1.0 / math.sqrt(d) if softmax_scale is None else softmax_scale
    qd = q.double().view(Lq, heads, d).transpose(0, 1)
    kd = k.double().view(Lkv, heads, d).transpose(0, 1)
    vd = v.double().view(Lkv, heads, d).transpose(0, 1)
    if block_len and pad_keys:
        kd = torch.cat([kd, kd.new_zeros(heads, pad_keys, d)], dim=1)
        vd = torch.cat([vd, vd.new_zeros(heads, pad_keys, d)], dim=1)
    s = (qd @ kd.transpose(1, 2)) * scale
    if block_len:
        m = O.block_causal_mask(Lq, kd.shape[1], block_len, window, q.device)
        s = s.masked_fill(~m, float("-inf"))
    return (torch.softmax(s, dim=-1) @ vd).transpose(0, 1).reshape(Lq, heads * d)


def rel_rows_heads(got, ref, heads):
    """Relative L2 error of every (row, head) 128-vector; returns the [L, heads] float64 tensor."""
    g = got.double().view(got.shape[0], heads, -1)
    r = ref.double().view(ref.shape[0], heads, -1)
    return (g - r).norm(dim=-1) / r.norm(dim=-1).clamp_min(1e-300)


# ---------------------------------------------------------------------------------------------
# kr_vae.cu
# ---------------------------------------------------------------------------------------------
def vae_rmsnorm(x, gamma, dtype):
    """RMS_norm of vae.py:39-54 on channels-last x [..., C] with the 16-bit eager rounding points:
    n = r16(||x||), y = r16(x / n), y = r16(r16(y * sqrt(C)) * gamma).  Returns (rounded, exact)."""
    xd = x.double()
    C = x.shape[-1]
    n = r16(xd.norm(dim=-1, keepdim=True), dtype)
    y = r16(xd / n.clamp_min(1e-12), dtype)
    y = r16(r16(y * math.sqrt(C), dtype) * gamma.double(), dtype)
    exact = V.rms_norm(xd.movedim(-1, 1), gamma.double().view(-1, *([1] * (x.dim() - 2)))).movedim(1, -1) \
        if x.dim() >= 2 else None
    return y, exact


def vae_rmsnorm_silu(x, gamma, dtype):
    """The kernel's output r16(SiLU(y)) of :func:`vae_rmsnorm` (SiLU evaluated on the rounded y), and SiLU(exact)."""
    y, exact = vae_rmsnorm(x, gamma, dtype)
    return r16(F.silu(y), dtype), F.silu(exact)


def softmax_rows(s):
    return torch.softmax(s.double(), dim=-1)
