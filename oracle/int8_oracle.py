"""TEST INFRASTRUCTURE — CPU oracle for the INT8 linear (not shipped; only tests/ import it):
``Int8DynamicActivationInt8WeightConfig()``, torchao's W8A8 config, restated from its published definition.

- Activations, per token, symmetric: ``amax_r = max(max|x[r]|, 1e-12)`` in fp32,
  ``q = clamp(rint(x * (127 / amax_r)), -127, 127)`` with ``127 / amax_r`` a true fp32 division and ``rint`` rounding
  half to even; the stored scale is ``s_r = amax_r / 127`` (fp32).
- Weights, per output channel, symmetric over [-128, 127]: ``s_n = amax_n / 127.5`` (floored at
  ``torch.finfo(float32).eps`` so an all-zero channel quantises to zeros), ``q = clamp(rint(w / s_n), -128, 127)``.
- GEMM: ``acc = sum_k q_a * q_w`` in s32, exact; ``v = (float(acc) * s_r) * s_n`` in fp32, in that order; then the
  bf16 epilogue chain of the 16-bit GEMM (bias, GELU, gate + residual, residual).  One fp32 dequantisation and one
  bf16 rounding: these are the kernel's rounding points; torchao's own dequantisation rounds elsewhere and is not
  reproduced.
- |acc| <= 127 * 128 * K < 2^31 for K <= 132104.

torchao is not in the image, so parity with it is unpinned, as for the FP8 tiers.  The integer product is pinned to
``torch._int_mm`` on the CPU (tests/test_int8_cpu.py)."""
from __future__ import annotations

import torch

I8_MAX_K = 132104


def quantize_act_rows(x: torch.Tensor):
    """x [rows, cols] -> (int8 [rows, cols], fp32 [rows] scales amax_r / 127)."""
    amax = x.float().abs().amax(dim=-1, keepdim=True).clamp(min=1e-12)
    mul = torch.full_like(amax, 127.0) / amax            # a true division (``127 / t`` is reciprocal * 127 in torch)
    q = torch.round(x.float() * mul).clamp(-127, 127).to(torch.int8)
    return q, (amax / 127.0).squeeze(-1)


def quantize_weight_rows(w: torch.Tensor):
    """w [N, K] -> (int8 [N, K], fp32 [N] scales amax_n / 127.5)."""
    amax = w.float().abs().amax(dim=1, keepdim=True)
    scale = (amax / 127.5).clamp(min=torch.finfo(torch.float32).eps)
    q = torch.round(w.float() / scale).clamp(-128, 127).to(torch.int8)
    return q, scale.squeeze(1)


def int_mm(a_q: torch.Tensor, w_q: torch.Tensor) -> torch.Tensor:
    """Exact s32 sums a_q [M, K] @ w_q [N, K]^T, as int64 (every value is below 2^31 for K <= 132104)."""
    return a_q.long() @ w_q.long().t()


def dequantize(acc: torch.Tensor, s_a: torch.Tensor, s_w: torch.Tensor) -> torch.Tensor:
    """The kernel's fp32 dequantisation: (float(acc) * s_a[m]) * s_w[n]."""
    return (acc.float() * s_a.float()[:, None]) * s_w.float()[None, :]


def linear_int8(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    """bf16(v + bias) with both operands quantised here: the EPI_BIAS output of the INT8 linear."""
    aq, sa = quantize_act_rows(x)
    wq, sw = quantize_weight_rows(w)
    v = dequantize(int_mm(aq, wq), sa, sw)
    if bias is not None:
        v = v + bias.float()
    return v.to(torch.bfloat16)
