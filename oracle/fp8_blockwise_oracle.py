"""TEST INFRASTRUCTURE — CPU oracle for the block-scaled FP8 linear (not shipped; only tests/ import it), the PerBlock
counterpart of oracle/fp8_rowwise_oracle.py: ``Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]),
PerBlock([128, 128])])`` gives one scale per 1 x 128 group of an activation row and one per 128 x 128 block of the
weight ``W[N, K]`` (the DeepSeek-V3 FP8 recipe).

Per group (block) ``g``: ``amax_g = max|x_g|`` in fp32 clamped at 1e-12, ``q_g = sat_e4m3(x_g * (448 / amax_g))``
rounding to nearest even with ``448 / amax_g`` a true fp32 division, ``scale_g = amax_g / 448``.  Activation scales are
returned k-block-major, ``[cols / 128, rows]``, the layout the kernels store; weight scales ``[N / 128, K / 128]``.  The
product is ``sum_kb (x_q[:, kb] @ w_q[:, kb]^T) * sa[kb, m] * sw[n / 128, kb]``, i.e. ``torch._scaled_mm`` with
``BlockWise1x128`` / ``BlockWise128x128`` scales.

What is pinned and what is not: torchao is not in the image, so parity with its scale formula is unpinned, as for
PerTensor and PerRow.  The scaled matmul is compared with ``torch._scaled_mm`` on the GPU where torch and cuBLAS accept
block scales (tests/test_fp8_blockwise_gpu.py).  An all-zero group quantises to zeros."""
from __future__ import annotations

import torch

from oracle.fp8_oracle import E4M3_MAX

BLOCK = 128


def _cast(x: torch.Tensor, amax: torch.Tensor) -> torch.Tensor:
    amax = amax.clamp(min=1e-12)
    mul = torch.full_like(amax, E4M3_MAX) / amax
    return (x * mul).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def quantize_per_group(x: torch.Tensor):
    """x [rows, cols] (cols % 128 == 0) -> (e4m3 [rows, cols], fp32 scales [cols / 128, rows] = amax_g / 448)."""
    rows, cols = x.shape
    xg = x.float().reshape(rows, cols // BLOCK, BLOCK)
    amax = xg.abs().amax(dim=-1, keepdim=True).clamp(min=1e-12)
    q = _cast(xg, amax).reshape(rows, cols)
    return q, (amax / E4M3_MAX).squeeze(-1).t().contiguous()


def quantize_per_block(w: torch.Tensor):
    """w [N, K] (N, K % 128 == 0) -> (e4m3 [N, K], fp32 scales [N / 128, K / 128] = amax_b / 448)."""
    N, K = w.shape
    wb = w.float().reshape(N // BLOCK, BLOCK, K // BLOCK, BLOCK)
    amax = wb.abs().amax(dim=(1, 3), keepdim=True).clamp(min=1e-12)
    q = _cast(wb, amax).reshape(N, K)
    return q, (amax / E4M3_MAX).reshape(N // BLOCK, K // BLOCK)


def dequantize_groups(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """e4m3 [rows, cols] and k-block-major scales [cols / 128, >= rows] -> float64 [rows, cols]."""
    rows, cols = q.shape
    s = scale[:, :rows].double().t().repeat_interleave(BLOCK, dim=1)
    return q.double() * s


def dequantize_blocks(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """e4m3 [N, K] and block scales [N / 128, K / 128] -> float64 [N, K]."""
    s = scale.double().repeat_interleave(BLOCK, dim=0).repeat_interleave(BLOCK, dim=1)
    return q.double() * s


def matmul_blockwise(xq, sx, wq, sw) -> torch.Tensor:
    """The exact block-scaled product in float64: sum_kb (x_q[:, kb] @ w_q[:, kb]^T) * sx[kb, m] * sw[n / 128, kb]."""
    return dequantize_groups(xq, sx) @ dequantize_blocks(wq, sw).t()


def linear_fp8_blockwise(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    """bf16(block-scaled product + bias), x and w given in bf16 / fp32 (quantised here)."""
    xq, sx = quantize_per_group(x)
    wq, sw = quantize_per_block(w)
    y = matmul_blockwise(xq, sx, wq, sw)
    if bias is not None:
        y = y + bias.double()
    return y.to(torch.bfloat16)
