"""fp32 torch stand-ins of tests/cpu_ops_emulation_fp8_rows.py plus the block-scaled FP8 (torchao PerBlock) entry
points — TEST INFRASTRUCTURE for tests/test_fp8_blockwise_cpu.py, which monkeypatches ``dit.ops`` with this module.
Contracts: include/krea_b200_fp8_blocks.h kr_fp8_quantize_blocks / kr_ln_modulate_fp8_blocks / kr_gemm_fp8_blockwise;
the e4m3 bytes and group scales are the oracle's (oracle/fp8_blockwise_oracle.py quantize_per_group)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import fp8_blockwise_oracle as F8B
from realtime_video_b200.ops import Fp8Blocks
from tests.cpu_ops_emulation_fp8_rows import *  # noqa: F401,F403  (every stand-in the DiT schedule calls)
from tests.cpu_ops_emulation import _store, gemm


def _cast_blocks(x, q, scale):
    xq, s = F8B.quantize_per_group(x.reshape(-1, x.shape[-1]))
    return Fp8Blocks(_store(q, xq.view(torch.uint8)), _store(scale, s), x.dtype)


def fp8_quantize_blocks(x, q=None, scale=None):
    """kr_fp8_quantize_blocks contract: -> Fp8Blocks(e4m3 bytes as uint8 [rows, cols], amax_g / 448 fp32
    [cols / 128, rows])."""
    return _cast_blocks(x, q, scale)


def ln_modulate_fp8_blocks(x, *, eps, weight=None, bias=None, mod=None, shift_idx=0, scale_idx=1, rows_per_frame=0,
                           out=None, row_offset=0, q=None, scale=None):
    """kr_ln_modulate_fp8_blocks contract: the per-group cast of ln_modulate's output, computed in one step; the
    16-bit output only when ``out`` is given."""
    y = F.layer_norm(x.float(), (x.shape[-1],), None if weight is None else weight.float(),
                     None if bias is None else bias.float(), eps)
    if mod is not None:
        fr = (torch.arange(x.shape[0]) + row_offset) // rows_per_frame
        y = y * (1 + mod.float()[fr, scale_idx]) + mod.float()[fr, shift_idx]
    y = y.to(x.dtype)
    if out is not None:
        out.copy_(y)
    return _cast_blocks(y, q, scale)


def gemm_fp8_blockwise(a, w_q, scale_w, bias=None, **kw):
    """kr_gemm_fp8_blockwise contract: sum_kb (a.q @ w_q^T)[kb] * a.scale[kb, m] * scale_w[n / 128, kb] + bias, then
    the epilogue (the scales folded into the operands)."""
    xq = F8B.dequantize_groups(a.q.view(torch.float8_e4m3fn), a.scale).float()
    wf = F8B.dequantize_blocks(w_q.view(torch.float8_e4m3fn), scale_w).float()
    return gemm(xq, wf, bias, **kw)


def linear_fp8_blockwise(x, w_q, scale_w, bias=None, **kw):
    """kr_fp8_quantize_blocks (unless ``x`` is already an Fp8Blocks) + kr_gemm_fp8_blockwise."""
    if not isinstance(x, Fp8Blocks):
        x = fp8_quantize_blocks(x)
    return gemm_fp8_blockwise(x, w_q, scale_w, bias, **kw)
