"""TEST INFRASTRUCTURE — CPU oracle for the row-scaled FP8 linear (not shipped; only tests/ import it), the PerRow
counterpart of oracle/fp8_oracle.py: ``Float8DynamicActivationFloat8WeightConfig(granularity=PerRow())`` gives one scale
per activation row (token) and one per weight output channel (one row of ``W[N, K]``).

Restates torchao's published per-row algorithm the way fp8_oracle.py restates the per-tensor one:
``amax_r = max|x[r, :]|`` in fp32 clamped at 1e-12, ``q = sat_e4m3(x * (448 / amax_r))`` rounding to nearest even,
``scale_r = amax_r / 448``; the output is ``bf16((x_q @ w_q^T) * scale_a[m] * scale_w[n] + bias)``, i.e.
``torch._scaled_mm(x_q, w_q.t(), scale_a=[M, 1], scale_b=[1, N], out_dtype=bf16)``.

What is pinned and what is not: torchao is not in the image, so parity with its scale formula is unpinned, as for
PerTensor.  The scaled matmul is pinned to ``torch._scaled_mm`` with row-wise scales on the GPU only
(tests/test_fp8_rowwise_gpu.py): torch's CPU backend accepts per-tensor scales only.  A zero row quantises to zeros
and its output is the bias."""
from __future__ import annotations

import torch

from oracle.fp8_oracle import E4M3_MAX


def quantize_per_row(x: torch.Tensor):
    """x [rows, cols] -> (e4m3 tensor, dequantisation scales amax_r / 448 as fp32 [rows]).  ``448 / amax_r`` is a true
    fp32 division (torch evaluates ``scalar / tensor`` as ``reciprocal * scalar``, which differs in the last bit and
    then flips ties of the e4m3 rounding)."""
    amax = x.float().abs().amax(dim=-1, keepdim=True).clamp(min=1e-12)
    mul = torch.full_like(amax, E4M3_MAX) / amax
    q = (x.float() * mul).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q, (amax / E4M3_MAX).squeeze(-1)


def linear_fp8_rowwise(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    """bf16((x_q @ w_q^T) * scale_a[m] * scale_w[n] + bias) with per-row activation and per-output-channel weight
    scales, x and w given in bf16 / fp32 (quantised here)."""
    xq, sx = quantize_per_row(x)
    wq, sw = quantize_per_row(w)
    y = (xq.float() @ wq.float().t()) * sx[:, None] * sw[None, :]
    if bias is not None:
        y = y + bias.float()
    return y.to(torch.bfloat16)
