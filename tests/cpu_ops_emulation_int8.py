"""fp32 torch stand-ins of tests/cpu_ops_emulation_fp8.py plus the INT8 entry points — TEST INFRASTRUCTURE for
tests/test_int8_cpu.py, which monkeypatches ``dit.ops`` with this module.  Contracts: include/krea_b200_int8.h
kr_i8_quantize_rows / kr_ln_modulate_i8 / kr_gemm_i8_rowwise; the s8 bytes and scales are the oracle's
(oracle/int8_oracle.py quantize_act_rows) and the GEMM dequantises the exact integer product the oracle's way.
``entry_points`` records, per INT8 linear, whether its input arrived already cast."""
from __future__ import annotations

import torch

from oracle import int8_oracle as I8
from realtime_video_b200.ops import I8Rows
from tests import cpu_ops_emulation as _tensor
from tests.cpu_ops_emulation_fp8 import *  # noqa: F401,F403  (every stand-in the DiT schedule calls)
from tests.cpu_ops_emulation_fp8 import _store

entry_points = []


def _cast_rows(x, q, scale):
    xq, s = I8.quantize_act_rows(x.reshape(-1, x.shape[-1]))
    return I8Rows(_store(q, xq), _store(scale, s.float()), x.dtype)


def i8_quantize_rows(x, q=None, scale=None):
    """kr_i8_quantize_rows contract: -> I8Rows(int8 [rows, cols], amax_r / 127 fp32 [rows])."""
    return _cast_rows(x, q, scale)


def ln_modulate_i8(x, *, q=None, scale=None, out=None, **kw):
    """kr_ln_modulate_i8 contract: the per-row s8 cast of ln_modulate's output, computed in one step."""
    return _cast_rows(_tensor.ln_modulate(x, out=out, **kw), q, scale)


def gemm_i8_rowwise(a, w_q, scale_w, bias=None, **kw):
    """kr_gemm_i8_rowwise contract: (float(a.q @ w_q^T) * a.scale[m]) * scale_w[n] + bias, then the epilogue (the
    exact integer product, dequantised, through the 16-bit GEMM stand-in's epilogue with an identity operand)."""
    v = I8.dequantize(I8.int_mm(a.q, w_q), a.scale[:a.q.shape[0]], scale_w)
    return _tensor.gemm(v, torch.eye(v.shape[1]), bias, **kw)


def linear_i8(x, w_q, scale_w, bias=None, **kw):
    """kr_i8_quantize_rows (unless ``x`` is already an I8Rows) + kr_gemm_i8_rowwise."""
    entry_points.append(("kr_gemm_i8_rowwise", isinstance(x, I8Rows)))
    if not isinstance(x, I8Rows):
        x = i8_quantize_rows(x)
    return gemm_i8_rowwise(x, w_q, scale_w, bias, **kw)
