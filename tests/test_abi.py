"""The C-ABI library loads on a CPU-only box and exports every symbol include/krea_b200.h
declares (no compute calls here)."""
import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    from realtime_video_b200 import _lib
    _lib.build()
    return _lib.load()


def header_symbols():
    text = (ROOT / "include" / "krea_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(kr_[a-z0-9_]+)\s*\(", text)))


def test_every_declared_symbol_is_exported(lib):
    names = header_symbols()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"{n} declared in krea_b200.h but not exported"


def test_bindings_cover_the_header(lib):
    from realtime_video_b200 import _lib
    declared = set(header_symbols()) - {"kr_version", "kr_last_error", "kr_gemm_workspace_bytes",
                                             "kr_jpeg_workspace_bytes", "kr_dit_block_workspace_bytes"}   # non-int returns
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)


def test_version_and_error_string(lib):
    assert lib.kr_version() >= 100
    assert isinstance(lib.kr_last_error(), (bytes, type(None)))


def test_argument_validation_needs_no_gpu(lib):
    """Bad arguments are rejected before any CUDA call: codes are negative, message is set."""
    rc = lib.kr_gemm(0, 0, None, 0, None, 0, None, None, 0, 1, 1, 1, None, 0, None, 0, 0, ctypes.c_float(1.0), None, 0, 0,
                     0, None)
    assert rc == -1 and b"null" in lib.kr_last_error()
    rc = lib.kr_attn_fwd(5, None, 0, None, 0, None, 0, None, 0, 1, 1, 1, ctypes.c_float(1.0), 0, 0, 0, 0, None)
    assert rc == -1


def test_product_path_has_no_cpu_fallback():
    import torch
    from realtime_video_b200 import _lib, ops
    with pytest.raises(_lib.KreaB200Error):
        ops.gemm(torch.zeros(4, 64, dtype=torch.bfloat16), torch.zeros(32, 64, dtype=torch.bfloat16))


def test_product_never_imports_the_oracle():
    pkg = ROOT / "realtime_video_b200"
    for f in pkg.rglob("*.py"):
        src = f.read_text()
        assert "from oracle" not in src and "import oracle" not in src, f"{f} imports the oracle"


def test_gemm_kernel_plan_for_the_bench_shapes():
    """Host-only query: which kernel kr_gemm serves a shape with on a 132-SM part (the CPU box falls back to 132).
    M = 4680 token rows: the 2-CTA cluster kernel is costed at its measured throughput (a pair-tile wave = 1.62
    single-CTA waves), so every bench shape stays on the single-CTA kernels: the wide projections on the fixed width
    (1), the N = 5120 ones (740 tiles = 5.6 waves of 256-wide tiles) and the prompt projection on the wave-fitted
    width (4)."""
    from realtime_video_b200 import _lib
    lib = _lib.load()
    assert lib.kr_gemm_kernel_id(0, 4680, 15360, 5120) == 1      # to_qkv
    assert lib.kr_gemm_kernel_id(1, 4680, 13824, 5120) == 1      # ffn.0 + GELU
    assert lib.kr_gemm_kernel_id(2, 4680, 5120, 5120) == 4       # o + gate/residual
    assert lib.kr_gemm_kernel_id(2, 4680, 5120, 13824) == 4      # ffn.2 + gate/residual
    assert lib.kr_gemm_kernel_id(0, 512, 10240, 4096) == 4       # prompt k/v: wave-fitted width
    assert lib.kr_gemm_kernel_id(4, 4680, 15360, 5120) == 1      # fp32-output epilogue: single-CTA only
