"""fp32 torch stand-ins of tests/cpu_ops_emulation.py plus the row-scaled FP8 (torchao PerRow) entry points — TEST
INFRASTRUCTURE for tests/test_fp8_rowwise_cpu.py, which monkeypatches ``dit.ops`` with this module.  Contracts:
include/krea_b200.h kr_fp8_quantize_rows / kr_ln_modulate_fp8 / kr_gemm_fp8_rowwise; the e4m3 bytes and row scales
are the oracle's (oracle/fp8_rowwise_oracle.py quantize_per_row)."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import fp8_rowwise_oracle as F8R
from realtime_video_b200.ops import Fp8Rows
from tests.cpu_ops_emulation import *  # noqa: F401,F403  (every stand-in the DiT schedule calls)
from tests.cpu_ops_emulation import _store, gemm


def fp8_quantize_rows(x, q=None, scale=None):
    """kr_fp8_quantize_rows contract: -> Fp8Rows(e4m3 bytes as uint8 [rows, cols], amax_r / 448 fp32 [rows])."""
    xq, s = F8R.quantize_per_row(x.reshape(-1, x.shape[-1]))
    return Fp8Rows(_store(q, xq.view(torch.uint8)), _store(scale, s.float()), x.dtype)


def ln_modulate_fp8(x, *, eps, weight=None, bias=None, mod=None, shift_idx=0, scale_idx=1, rows_per_frame=0, out=None,
                    row_offset=0, q=None, scale=None):
    """kr_ln_modulate_fp8 contract: the per-row cast of ln_modulate's output, computed in one step; the 16-bit
    output only when ``out`` is given."""
    y = F.layer_norm(x.float(), (x.shape[-1],), None if weight is None else weight.float(),
                     None if bias is None else bias.float(), eps)
    if mod is not None:
        fr = (torch.arange(x.shape[0]) + row_offset) // rows_per_frame
        y = y * (1 + mod.float()[fr, scale_idx]) + mod.float()[fr, shift_idx]
    y = y.to(x.dtype)
    if out is not None:
        out.copy_(y)
    xq, s = F8R.quantize_per_row(y)
    return Fp8Rows(_store(q, xq.view(torch.uint8)), _store(scale, s.float()), x.dtype)


def gemm_fp8_rowwise(a, w_q, scale_w, bias=None, **kw):
    """kr_gemm_fp8_rowwise contract: (a.q @ w_q^T) * a.scale[m] * scale_w[n] + bias, then the epilogue."""
    xq = a.q.view(torch.float8_e4m3fn).float() * a.scale.float()[:, None]   # fold the row scales into the operands
    wf = w_q.view(torch.float8_e4m3fn).float() * scale_w.float()[:, None]
    return gemm(xq, wf, bias, **kw)


def linear_fp8_rowwise(x, w_q, scale_w, bias=None, **kw):
    """kr_fp8_quantize_rows (unless ``x`` is already an Fp8Rows) + kr_gemm_fp8_rowwise."""
    if not isinstance(x, Fp8Rows):
        x = fp8_quantize_rows(x)
    return gemm_fp8_rowwise(x, w_q, scale_w, bias, **kw)
