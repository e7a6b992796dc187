"""The stand-ins of tests/cpu_ops_emulation_fp8_rows.py with the ``fast_accum`` argument of the FP8 linears — TEST
INFRASTRUCTURE for tests/test_fp8_fast_accum_cpu.py, which monkeypatches ``dit.ops`` with this module.  Both
accumulation modes approximate the same exact product of the quantised operands, so the arithmetic is the stand-ins'
own; what this module adds is the record of which C entry point each call stands for (``entry_points``)."""
from __future__ import annotations

from realtime_video_b200.ops import Fp8Rows
from tests import cpu_ops_emulation as _tensor
from tests import cpu_ops_emulation_fp8_rows as _rows
from tests.cpu_ops_emulation_fp8_rows import *  # noqa: F401,F403  (every stand-in the DiT schedule calls)

entry_points = []


def linear_fp8(x, w_q, scale_w, bias=None, *, fast_accum=False, **kw):
    """kr_fp8_quantize + kr_gemm_fp8 or kr_gemm_fp8_fast."""
    entry_points.append("kr_gemm_fp8_fast" if fast_accum else "kr_gemm_fp8")
    return _tensor.linear_fp8(x, w_q, scale_w, bias, **kw)


def linear_fp8_rowwise(x, w_q, scale_w, bias=None, *, fast_accum=False, **kw):
    """kr_fp8_quantize_rows (unless ``x`` is already an Fp8Rows) + kr_gemm_fp8_rowwise or kr_gemm_fp8_rowwise_fast."""
    entry_points.append(("kr_gemm_fp8_rowwise_fast" if fast_accum else "kr_gemm_fp8_rowwise",
                         isinstance(x, Fp8Rows)))
    return _rows.linear_fp8_rowwise(x, w_q, scale_w, bias, **kw)
