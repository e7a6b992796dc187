"""ctypes binding of libkrea_b200.so (the C ABI declared in include/krea_b200.h).

The library is built in-tree by :func:`build` (``nvcc -gencode arch=compute_90a,code=sm_90a``)
so the ``.so`` travels with the repository snapshot.  There is no CPU or eager fallback: every
op raises if the library is missing or a call returns a non-zero code (the reference's error
convention is plain Python exceptions, SURVEY.md §8b).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import threading
from pathlib import Path

_PKG_DIR = Path(__file__).resolve().parent
_CSRC = _PKG_DIR / "csrc"
LIB_PATH = _PKG_DIR / "libkrea_b200.so"
SOURCES = ["kr_host.cu", "kr_gemm.cu", "kr_gemm2.cu", "kr_gemm_sk.cu", "kr_gemm_fp8.cu", "kr_attn.cu", "kr_sage.cu", "kr_t5attn.cu", "kr_dit_elem.cu", "kr_vae.cu", "kr_jpeg.cu", "kr_dit_block.cu", "kr_api.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "--shared", "-Xcompiler", "-fPIC", "-cudart", "static",
]

_lock = threading.Lock()
_lib = None


class KreaB200Error(RuntimeError):
    """A C-ABI call returned a non-zero code."""


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise FileNotFoundError("nvcc not found")


def _sources() -> list[Path]:
    return [_CSRC / s for s in SOURCES if (_CSRC / s).exists()]


def needs_build() -> bool:
    if not LIB_PATH.exists():
        return True
    t = LIB_PATH.stat().st_mtime
    deps = list(_CSRC.glob("*.cu")) + list(_CSRC.glob("*.cuh")) + list(_CSRC.glob("*.h"))
    deps += list((_PKG_DIR.parent / "include").glob("*.h"))
    return any(d.exists() and d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source into libkrea_b200.so for sm_90a (cross-compiles without a GPU)."""
    with _lock:
        if not force and not needs_build():
            return LIB_PATH
        objs = []
        procs = []
        build_dir = _PKG_DIR / "build"
        build_dir.mkdir(exist_ok=True)
        base = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo",
                "-std=c++17", "-Xcompiler", "-fPIC"]
        for src in _sources():
            obj = build_dir / (src.stem + ".o")
            objs.append(obj)
            procs.append((src, subprocess.Popen(base + ["-c", "-o", str(obj), str(src)],
                                                stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        for src, p in procs:
            out, _ = p.communicate()
            if p.returncode != 0:
                raise RuntimeError(f"nvcc failed on {src.name}:\n{out.decode(errors='replace')}")
            if verbose and out:
                print(out.decode(errors="replace"))
        tmp = LIB_PATH.with_suffix(".so.tmp")
        link = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "--shared", "-cudart",
                "static", "-o", str(tmp)] + [str(o) for o in objs]
        r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc link failed:\n{r.stdout.decode(errors='replace')}")
        os.replace(tmp, LIB_PATH)
        return LIB_PATH


_vp = ctypes.c_void_p
_i = ctypes.c_int
_f = ctypes.c_float
_l = ctypes.c_long
_sz = ctypes.c_size_t



class KrDitBlockParams(ctypes.Structure):
    """``KrDitBlockParams`` of include/krea_b200.h, field for field."""
    _fields_ = [
        ("L", _i), ("D", _i), ("ffn", _i), ("heads", _i), ("head_dim", _i),
        ("frames", _i), ("rows_per_frame", _i),
        ("grid_h", _i), ("grid_w", _i), ("start_frame", _i),
        ("cross_attn_norm", _i),
        ("eps_block", _f), ("eps_qk", _f), ("eps_norm3", _f), ("eps_cross", _f),
        ("x", _vp), ("ldx", _i),
        ("e0", _vp), ("lde0_frame", _i),
        ("modulation", _vp),
        ("rope", _vp),
        ("w_qkv", _vp), ("b_qkv", _vp),
        ("norm_q", _vp), ("norm_k", _vp),
        ("w_o", _vp), ("b_o", _vp),
        ("k_cache", _vp), ("v_cache", _vp), ("ld_cache", _i),
        ("local_start", _i), ("local_end", _i), ("attn_lo", _i),
        ("mask_mode", _i), ("block_len", _i), ("window", _i), ("pad_keys", _i),
        ("norm3_w", _vp), ("norm3_b", _vp),
        ("w_cq", _vp), ("b_cq", _vp), ("norm_cq", _vp),
        ("ck", _vp), ("cv", _vp), ("ld_ck", _i), ("ld_cv", _i), ("text_len", _i),
        ("w_co", _vp), ("b_co", _vp),
        ("w_ffn0", _vp), ("b_ffn0", _vp), ("w_ffn2", _vp), ("b_ffn2", _vp),
        ("workspace", _vp), ("workspace_bytes", _sz),
        ("gemm_workspace", _vp), ("gemm_workspace_bytes", _sz),
    ]


# name -> argtypes; every function returns int except where noted
SIGNATURES = {
    "kr_gemm_kernel_id": [_i, _i, _i, _i],
    "kr_gemm_kernel_id_ws": [_i, _i, _i, _i, _i],
    "kr_gemm_ws": [_i, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _f, _vp, _i, _i,
                   _i, _vp, _sz, _vp],
    "kr_gemm": [_i, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _f, _vp, _i, _i,
                _i, _vp],
    "kr_fp8_quantize": [_vp, _i, _i, _i, _vp, _i, _vp, _vp],
    "kr_gemm_fp8": [_i, _vp, _i, _vp, _i, _vp, _f, _vp, _vp, _i, _i, _i, _i, _vp, _i, _vp, _i, _i, _vp, _i, _i, _i, _vp],
    "kr_attn_fwd": [_i, _vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp],
    "kr_t5_attn": [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp, _vp, _vp],
    "kr_ln_modulate": [_vp, _i, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp],
    "kr_qkv_norm_rope": [_vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _i,
                         _i, _i, _i, _i, _i, _i, _f, _vp],
    "kr_qkv_norm_rope_p2p": [_vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _i, _i, _i, _vp,
                             _i, _i, _i, _i, _i, _i, _i, _f, _vp],
    "kr_comm_scatter_rows": [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp],
    "kr_kv_roll": [_vp, _i, _i, _i, _i, _i, _vp],
    "kr_rmsnorm": [_vp, _i, _vp, _i, _vp, _i, _i, _f, _vp],
    "kr_add_modulation": [_vp, _vp, _i, _vp, _i, _i, _i, _vp],
    "kr_activation": [_vp, _vp, _sz, _i, _vp],
    "kr_patchify": [_vp, _l, _l, _l, _l, _vp, _i, _i, _i, _i, _vp],
    "kr_unpatchify_x0": [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "kr_vae_conv3d": [_i, _i, _i, _vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _l, _l,
                      _vp, _l, _l, _vp, _vp, _l, _l, _vp, _i, _vp],
    "kr_vae_rmsnorm_silu": [_i, _vp, _vp, _vp, _l, _i, _i, _vp],
    "kr_vae_upsample2x": [_vp, _vp, _i, _i, _i, _i, _vp],
    "kr_vae_scale_input": [_i, _vp, _l, _l, _l, _l, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp],
    "kr_softmax_rows": [_i, _vp, _l, _vp, _l, _i, _i, _vp],
    "kr_frames_to_rgb8": [_vp, _vp, _i, _i, _i, _vp],
    "kr_dit_block_fwd": [ctypes.POINTER(KrDitBlockParams), _vp],
    "kr_frames_to_jpeg": [_vp, _i, _i, _i, _i, _vp, _l, _vp, _vp, _sz, _vp],
    "kr_rgb8_to_jpeg": [_vp, _i, _i, _i, _i, _vp, _l, _vp, _vp, _sz, _vp],
}

# the quantised attention tier (include/krea_b200_sage.h, kr_sage.cu); every function returns int
SAGE_SIGNATURES = {
    "kr_sage_quantize": [_vp, _i, _vp, _i, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp],
    "kr_sage_attn": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp],
}


def load() -> ctypes.CDLL:
    """Load the shared library (building is the caller's job: ``__graft_entry__.build``)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists():
            raise KreaB200Error(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                f"g.build()'` (there is no CPU / eager fallback)")
        lib = ctypes.CDLL(str(LIB_PATH))
        lib.kr_version.restype = _i
        lib.kr_version.argtypes = []
        lib.kr_last_error.restype = ctypes.c_char_p
        lib.kr_last_error.argtypes = []
        lib.kr_gemm_workspace_bytes.restype = _sz
        lib.kr_gemm_workspace_bytes.argtypes = []
        if hasattr(lib, "kr_dit_block_workspace_bytes"):
            lib.kr_dit_block_workspace_bytes.restype = _sz
            lib.kr_dit_block_workspace_bytes.argtypes = [_i, _i, _i, _i]
        if hasattr(lib, "kr_jpeg_workspace_bytes"):
            lib.kr_jpeg_workspace_bytes.restype = _sz
            lib.kr_jpeg_workspace_bytes.argtypes = [_i, _i, _i]
        for name, argtypes in {**SIGNATURES, **SAGE_SIGNATURES}.items():
            fn = getattr(lib, name, None)
            if fn is None:
                continue   # checked by tests/test_abi.py against the header
            fn.restype = _i
            fn.argtypes = argtypes
        _lib = lib
        return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().kr_last_error()
        raise KreaB200Error(f"{what} failed with code {rc}: {msg.decode(errors='replace') if msg else ''}")
