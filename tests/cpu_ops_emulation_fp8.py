"""fp32 torch stand-ins of tests/cpu_ops_emulation.py plus the row-scaled (torchao PerRow) and block-scaled (PerBlock)
FP8 entry points and the ``fast_accum`` argument of the FP8 linears — TEST INFRASTRUCTURE for
tests/test_fp8_rowwise_cpu.py, tests/test_fp8_blockwise_cpu.py and tests/test_fp8_fast_accum_cpu.py, which monkeypatch
``dit.ops`` with this module.  Contracts: include/krea_b200.h kr_fp8_quantize_rows / kr_ln_modulate_fp8 /
kr_gemm_fp8_rowwise[_fast] / kr_gemm_fp8_fast and include/krea_b200_fp8_blocks.h kr_fp8_quantize_blocks /
kr_ln_modulate_fp8_blocks / kr_gemm_fp8_blockwise; the e4m3 bytes and scales are the oracles'
(oracle/fp8_rowwise_oracle.py quantize_per_row, oracle/fp8_blockwise_oracle.py quantize_per_group).  Both
accumulation modes approximate the same exact product of the quantised operands, so ``fast_accum`` changes no
arithmetic here; ``entry_points`` records which C entry point each FP8 linear stands for."""
from __future__ import annotations

import torch

from oracle import fp8_blockwise_oracle as F8B
from oracle import fp8_rowwise_oracle as F8R
from realtime_video_b200.ops import Fp8Blocks, Fp8Rows
from tests import cpu_ops_emulation as _tensor
from tests.cpu_ops_emulation import *  # noqa: F401,F403  (every stand-in the DiT schedule calls)
from tests.cpu_ops_emulation import _store, gemm

entry_points = []


def _cast_rows(x, q, scale):
    xq, s = F8R.quantize_per_row(x.reshape(-1, x.shape[-1]))
    return Fp8Rows(_store(q, xq.view(torch.uint8)), _store(scale, s.float()), x.dtype)


def _cast_blocks(x, q, scale):
    xq, s = F8B.quantize_per_group(x.reshape(-1, x.shape[-1]))
    return Fp8Blocks(_store(q, xq.view(torch.uint8)), _store(scale, s), x.dtype)


def _ln_modulate_cast(cast, x, *, q=None, scale=None, out=None, **kw):
    """ln_modulate with its output cast in the same step; the 16-bit output only when ``out`` is given."""
    return cast(_tensor.ln_modulate(x, out=out, **kw), q, scale)


def linear_fp8(x, w_q, scale_w, bias=None, *, fast_accum=False, **kw):
    """kr_fp8_quantize + kr_gemm_fp8 or kr_gemm_fp8_fast."""
    entry_points.append("kr_gemm_fp8_fast" if fast_accum else "kr_gemm_fp8")
    return _tensor.linear_fp8(x, w_q, scale_w, bias, **kw)


def fp8_quantize_rows(x, q=None, scale=None):
    """kr_fp8_quantize_rows contract: -> Fp8Rows(e4m3 bytes as uint8 [rows, cols], amax_r / 448 fp32 [rows])."""
    return _cast_rows(x, q, scale)


def ln_modulate_fp8(x, **kw):
    """kr_ln_modulate_fp8 contract: the per-row cast of ln_modulate's output, computed in one step."""
    return _ln_modulate_cast(_cast_rows, x, **kw)


def gemm_fp8_rowwise(a, w_q, scale_w, bias=None, **kw):
    """kr_gemm_fp8_rowwise contract: (a.q @ w_q^T) * a.scale[m] * scale_w[n] + bias, then the epilogue."""
    xq = a.q.view(torch.float8_e4m3fn).float() * a.scale.float()[:, None]   # fold the row scales into the operands
    wf = w_q.view(torch.float8_e4m3fn).float() * scale_w.float()[:, None]
    return gemm(xq, wf, bias, **kw)


def linear_fp8_rowwise(x, w_q, scale_w, bias=None, *, fast_accum=False, **kw):
    """kr_fp8_quantize_rows (unless ``x`` is already an Fp8Rows) + kr_gemm_fp8_rowwise or kr_gemm_fp8_rowwise_fast."""
    entry_points.append(("kr_gemm_fp8_rowwise_fast" if fast_accum else "kr_gemm_fp8_rowwise",
                         isinstance(x, Fp8Rows)))
    if not isinstance(x, Fp8Rows):
        x = fp8_quantize_rows(x)
    return gemm_fp8_rowwise(x, w_q, scale_w, bias, **kw)


def fp8_quantize_blocks(x, q=None, scale=None):
    """kr_fp8_quantize_blocks contract: -> Fp8Blocks(e4m3 bytes as uint8 [rows, cols], amax_g / 448 fp32
    [cols / 128, rows])."""
    return _cast_blocks(x, q, scale)


def ln_modulate_fp8_blocks(x, **kw):
    """kr_ln_modulate_fp8_blocks contract: the per-group cast of ln_modulate's output, computed in one step."""
    return _ln_modulate_cast(_cast_blocks, x, **kw)


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
