"""Tensor-level wrappers over the C ABI (``include/krea_b200.h``).

PyTorch is plumbing here: it owns device memory and the current stream; every op below is
one call into libkrea_b200.so.  All ops require CUDA tensors and raise otherwise — there is
no eager / CPU fallback on the product path.
"""
from __future__ import annotations

import ctypes
import math
from typing import NamedTuple, Optional

import torch

from . import _lib

EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_BIAS_RES, EPI_F32, EPI_MUL = 0, 1, 2, 3, 4, 5

_DT = {torch.bfloat16: 0, torch.float16: 1}

# count of kernels launched through this module (bench.py reports it as gpu_launches)
launch_count = 0


def _count(n: int = 1) -> None:
    global launch_count
    launch_count += n


_launch_device = None      # device of the operands of the op being issued (set by _req)


def _stream() -> int:
    """The caller's current stream ON THE OPERANDS' DEVICE (not the process-wide current device)."""
    return torch.cuda.current_stream(_launch_device).cuda_stream


# Optional per-kernel timing (bench.py roofline): CUDA events recorded on the launching stream
# around every launch of a kernel family while enabled.
_prof = None


def profile_begin() -> None:
    global _prof
    _prof = {}


def profile_end() -> dict:
    """{family: {"flops": algorithmic FLOPs, "ms": summed launch durations, "n": launches}}.
    Call after a synchronize."""
    global _prof
    rec, _prof = _prof or {}, None
    out = {}
    for fam, items in rec.items():
        ms = sum(a.elapsed_time(b) for a, b, _ in items)
        out[fam] = {"flops": float(sum(f for _, _, f in items)), "ms": ms, "n": len(items)}
    return out


# kr_gemm_kernel_id -> label used in the per-kernel timing split
_GEMM_KERNELS = {1: "gemm_tn_kernel", 2: "gemm2_tn_kernel", 3: "gemm_sk_kernel", 4: "gemm_flex_kernel"}

# stream-K workspace (kr_gemm_ws): one zero-filled buffer per (device, stream), allocated on first use and
# owned here (the library allocates nothing); set to False to force the data-parallel kernels
stream_k = True
_sk_ws = {}


def _gemm_workspace(device: torch.device, stream: int):
    if not stream_k:
        return None, 0
    key = (device.index, stream)
    ws = _sk_ws.get(key)
    if ws is None:
        n = _lib.load().kr_gemm_workspace_bytes()
        ws = _sk_ws[key] = torch.zeros(n, dtype=torch.uint8, device=device)
    return ws.data_ptr(), ws.numel()


class _Timed:
    def __init__(self, family: str, flops: float, sub: Optional[str] = None):
        self.family, self.flops, self.sub = family, flops, sub

    def __enter__(self):
        if _prof is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record()
        return self

    def __exit__(self, *exc):
        if _prof is not None:
            self.b.record()
            _prof.setdefault(self.family, []).append((self.a, self.b, self.flops))
            if self.sub is not None:
                _prof.setdefault(self.family + "/" + self.sub, []).append((self.a, self.b, self.flops))
        return False


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, name: str, dtype=None) -> None:
    global _launch_device
    if not t.is_cuda:
        raise _lib.KreaB200Error(f"{name} must be a CUDA tensor (no CPU fallback in the product path)")
    if t.device.index != torch.cuda.current_device():
        # kernels and TMA descriptors are issued on the CURRENT device; a model living on another GPU must be
        # driven under torch.cuda.device(...) like the reference server does (release_server.py:741)
        raise _lib.KreaB200Error(f"{name} lives on {t.device} but the current device is cuda:"
                                 f"{torch.cuda.current_device()}; wrap the call in torch.cuda.device({t.device.index})")
    _launch_device = t.device
    if dtype is not None and t.dtype != dtype:
        raise _lib.KreaB200Error(f"{name} must be {dtype}, got {t.dtype}")


def _rows2d(t: torch.Tensor, name: str):
    """View a [..., D] tensor with contiguous last dim and uniform row pitch as (rows, ld)."""
    if t.stride(-1) != 1:
        raise _lib.KreaB200Error(f"{name}: last dimension must be contiguous")
    if t.dim() == 1:
        return 1, t.shape[0]
    if t.dim() == 2:
        return t.shape[0], t.stride(0)
    lead = t.shape[:-1]
    ld = t.stride(-2)
    # leading dims must collapse onto one pitch
    exp = ld
    for size, stride in zip(reversed(lead), reversed(t.stride()[:-1])):
        if size != 1 and stride != exp:
            raise _lib.KreaB200Error(f"{name}: rows are not uniformly strided {t.shape} {t.stride()}")
        exp *= size
    return math.prod(lead), ld


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
         epilogue: int = EPI_BIAS, out: Optional[torch.Tensor] = None,
         residual: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None,
         rows_per_gate: int = 0, alpha: float = 1.0, out2: Optional[torch.Tensor] = None,
         n_split: int = 0, row_offset: int = 0) -> torch.Tensor:
    """out[M,N] = epilogue(a[M,K] @ w[N,K]^T + bias).  gate: [G, N] rows (pitch = stride(0)).
    out2: rows-strided [M, N - n_split] destination of the output columns >= n_split."""
    _req(a, "a"); _req(w, "w", a.dtype)
    M, lda = _rows2d(a, "a")
    K = a.shape[-1]
    N = w.shape[0]
    if w.shape[1] != K or w.stride(1) != 1:
        raise _lib.KreaB200Error(f"gemm: weight shape {tuple(w.shape)} does not match K={K}")
    if out is None:
        odt = torch.float32 if epilogue == EPI_F32 else a.dtype
        out = torch.empty(*a.shape[:-1], N, dtype=odt, device=a.device)
    _, ldc = _rows2d(out, "out")
    ldr = 0
    if residual is not None:
        _req(residual, "residual", a.dtype)
        _, ldr = _rows2d(residual, "residual")
    gs = 0
    if gate is not None:
        _req(gate, "gate", a.dtype)
        gs = gate.stride(0) if gate.dim() >= 2 else 0
    ldc2 = 0
    if out2 is not None:
        _req(out2, "out2", a.dtype)
        _, ldc2 = _rows2d(out2, "out2")
    lib = _lib.load()
    stream = _stream()
    ws_ptr, ws_bytes = _gemm_workspace(a.device, stream)
    with _Timed("gemm", 2.0 * M * N * K,
                sub=_GEMM_KERNELS[lib.kr_gemm_kernel_id_ws(epilogue, M, N, K, 1 if ws_ptr else 0)]
                if _prof is not None else None):
        rc = lib.kr_gemm_ws(_DT[a.dtype], epilogue, a.data_ptr(), lda, w.data_ptr(), w.stride(0),
                            _ptr(bias), out.data_ptr(), ldc, M, N, K, _ptr(residual), ldr, _ptr(gate), gs,
                            rows_per_gate, alpha, _ptr(out2), ldc2, n_split, row_offset, ws_ptr, ws_bytes, stream)
    _lib.check(rc, "kr_gemm_ws")
    _count()
    return out


_block_ws = {}


def dit_block_fwd(x: torch.Tensor, e0: torch.Tensor, modulation: torch.Tensor, rope: torch.Tensor, *,
                  w_qkv, b_qkv, norm_q, norm_k, w_o, b_o, k_cache: torch.Tensor, v_cache: torch.Tensor,
                  local_start: int, local_end: int, attn_lo: int, norm3_w, norm3_b, w_cq, b_cq, norm_cq,
                  ck: torch.Tensor, cv: torch.Tensor, w_co, b_co, w_ffn0, b_ffn0, w_ffn2, b_ffn2, heads: int,
                  rows_per_frame: int, grid_h: int, grid_w: int, start_frame: int, eps_block: float, eps_qk: float,
                  eps_norm3: float, eps_cross: float, block_len: int = 0, window: int = 0, pad_keys: int = 0) -> torch.Tensor:
    """One whole DiT block (kr_dit_block_fwd): x [L, D] bf16 updated in place.  k_cache / v_cache: this layer's caches
    viewed as [rows, D]; rows [local_start, local_end) receive this call's K / V; block_len > 0 selects the recompute
    branch (block-causal rule over rows [0, L)), otherwise the queries attend rows [attn_lo, local_end).
    ck / cv: projected prompt K / V [text_len, D].  The scratch workspace is cached per (device, stream, shape)."""
    _req(x, "x", torch.bfloat16)
    L, ldx = _rows2d(x, "x")
    D = x.shape[-1]
    ffn = w_ffn0.shape[0]
    for name, w, shape in (("w_qkv", w_qkv, (3 * D, D)), ("w_o", w_o, (D, D)), ("w_cq", w_cq, (D, D)),
                           ("w_co", w_co, (D, D)), ("w_ffn0", w_ffn0, (ffn, D)), ("w_ffn2", w_ffn2, (D, ffn))):
        _req(w, name, torch.bfloat16)
        if tuple(w.shape) != shape or not w.is_contiguous():
            raise _lib.KreaB200Error(f"dit_block_fwd: {name} must be contiguous {shape}, got {tuple(w.shape)}")
    for name, t in (("e0", e0), ("modulation", modulation), ("k_cache", k_cache), ("v_cache", v_cache), ("ck", ck),
                    ("cv", cv)):
        _req(t, name, torch.bfloat16)
    _req(rope, "rope", torch.float32)
    F = e0.shape[-3]
    if e0.stride(-1) != 1 or e0.stride(-2) != D or e0.shape[-2] != 6:
        raise _lib.KreaB200Error("dit_block_fwd: e0 must be [frames, 6, D] with contiguous rows")
    _, ld_cache = _rows2d(k_cache, "k_cache")
    if _rows2d(v_cache, "v_cache")[1] != ld_cache:
        raise _lib.KreaB200Error("dit_block_fwd: K and V caches must share their row pitch")
    text_len, ld_ck = _rows2d(ck, "ck")
    _, ld_cv = _rows2d(cv, "cv")
    lib = _lib.load()
    stream = _stream()
    need = lib.kr_dit_block_workspace_bytes(L, D, ffn, F)
    key = (x.device.index, stream, L, D, ffn, F)
    ws = _block_ws.get(key)
    if ws is None:
        if len(_block_ws) > 8:
            _block_ws.clear()
        raw = torch.empty(need + 256, dtype=torch.uint8, device=x.device)
        off = (-raw.data_ptr()) % 256                 # the C side wants 256-byte alignment whatever the allocator gives
        ws = _block_ws[key] = raw[off:off + need]
    gws_ptr, gws_bytes = _gemm_workspace(x.device, stream)
    p = _lib.KrDitBlockParams(
        L=L, D=D, ffn=ffn, heads=heads, head_dim=D // heads, frames=F, rows_per_frame=rows_per_frame,
        grid_h=grid_h, grid_w=grid_w, start_frame=start_frame, cross_attn_norm=0 if norm3_w is None else 1,
        eps_block=eps_block, eps_qk=eps_qk, eps_norm3=eps_norm3, eps_cross=eps_cross,
        x=x.data_ptr(), ldx=ldx, e0=e0.data_ptr(), lde0_frame=e0.stride(-3), modulation=modulation.data_ptr(),
        rope=rope.data_ptr(), w_qkv=w_qkv.data_ptr(), b_qkv=_ptr(b_qkv), norm_q=norm_q.data_ptr(),
        norm_k=norm_k.data_ptr(), w_o=w_o.data_ptr(), b_o=_ptr(b_o), k_cache=k_cache.data_ptr(),
        v_cache=v_cache.data_ptr(), ld_cache=ld_cache, local_start=local_start, local_end=local_end, attn_lo=attn_lo,
        mask_mode=1 if block_len > 0 else 0, block_len=block_len, window=window, pad_keys=pad_keys,
        norm3_w=_ptr(norm3_w), norm3_b=_ptr(norm3_b), w_cq=w_cq.data_ptr(), b_cq=_ptr(b_cq),
        norm_cq=norm_cq.data_ptr(), ck=ck.data_ptr(), cv=cv.data_ptr(), ld_ck=ld_ck, ld_cv=ld_cv, text_len=text_len,
        w_co=w_co.data_ptr(), b_co=_ptr(b_co), w_ffn0=w_ffn0.data_ptr(), b_ffn0=_ptr(b_ffn0),
        w_ffn2=w_ffn2.data_ptr(), b_ffn2=_ptr(b_ffn2), workspace=ws.data_ptr(), workspace_bytes=ws.numel(),
        gemm_workspace=gws_ptr, gemm_workspace_bytes=gws_bytes)
    rc = lib.kr_dit_block_fwd(ctypes.byref(p), stream)
    _lib.check(rc, "kr_dit_block_fwd")
    _count(14)
    return x


_fp8_scratch = {}


def _fp8_cast_scratch(kind: str, x: torch.Tensor):
    """``x`` as [rows, cols] and the (q, scale) buffers its ``kind`` ("tensor", "rows", "blocks" or "i8") cast writes,
    reused per (kind, device, rows, cols); the launches are stream-ordered."""
    rows, _ = _rows2d(x, "x")
    cols = x.shape[-1]
    key = (kind, x.device.index, rows, cols)
    sc = _fp8_scratch.get(key)
    if sc is None:
        scale_shape = {"tensor": (2,), "rows": (rows,), "blocks": (cols // 128, rows), "i8": (rows,)}[kind]
        qtype = torch.int8 if kind == "i8" else torch.uint8
        sc = _fp8_scratch[key] = (torch.empty(rows, cols, dtype=qtype, device=x.device),
                                  torch.empty(scale_shape, dtype=torch.float32, device=x.device))
    return (x if x.dim() == 2 else x.reshape(rows, -1)), *sc


def _fp8_epi_pitches(out: torch.Tensor, residual, gate, out2):
    """Row pitches of an FP8 GEMM's epilogue tensors: (ldc, ldr, gate stride, ldc2), 0 for an absent one."""
    _, ldc = _rows2d(out, "out")
    ldr = _rows2d(residual, "residual")[1] if residual is not None else 0
    gs = gate.stride(0) if gate is not None and gate.dim() >= 2 else 0
    ldc2 = _rows2d(out2, "out2")[1] if out2 is not None else 0
    return ldc, ldr, gs, ldc2


def fp8_quantize(x: torch.Tensor, q: Optional[torch.Tensor] = None, state: Optional[torch.Tensor] = None):
    """Dynamic per-tensor e4m3 cast (torchao Float8DynamicActivation, PerTensor): x [rows, cols] bf16 ->
    (q uint8 bytes [rows, cols], state float32 [2] = [amax, dequantisation scale amax / 448])."""
    _req(x, "x", torch.bfloat16)
    rows, ld = _rows2d(x, "x")
    cols = x.shape[-1]
    if q is None:
        q = torch.empty(rows, cols, dtype=torch.uint8, device=x.device)
    if state is None:
        state = torch.empty(2, dtype=torch.float32, device=x.device)
    lib = _lib.load()
    rc = lib.kr_fp8_quantize(x.data_ptr(), ld, rows, cols, q.data_ptr(), q.stride(0), state.data_ptr(), _stream())
    _lib.check(rc, "kr_fp8_quantize")
    _count(2)
    return q, state


def gemm_fp8(a_q: torch.Tensor, w_q: torch.Tensor, scale_a: torch.Tensor, scale_w: float,
             bias: Optional[torch.Tensor] = None, *, epilogue: int = EPI_BIAS, out: Optional[torch.Tensor] = None,
             residual: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None, rows_per_gate: int = 0,
             out2: Optional[torch.Tensor] = None, n_split: int = 0, row_offset: int = 0,
             fast_accum: bool = False) -> torch.Tensor:
    """out[M,N] (bf16) = epilogue((a_q[M,K] @ w_q[N,K]^T) * scale_a[1] * scale_w + bias); a_q / w_q e4m3 bytes,
    scale_a the ``state`` tensor of :func:`fp8_quantize`.  ``fast_accum`` runs kr_gemm_fp8_fast (accumulation inside
    the tensor core across the whole K, torch._scaled_mm's ``use_fast_accum=True``) on the same operands."""
    _req(a_q, "a_q", torch.uint8); _req(w_q, "w_q", torch.uint8)
    M, K = a_q.shape
    N = w_q.shape[0]
    if out is None:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=a_q.device)
    ldc, ldr, gs, ldc2 = _fp8_epi_pitches(out, residual, gate, out2)
    lib = _lib.load()
    name = "kr_gemm_fp8_fast" if fast_accum else "kr_gemm_fp8"
    with _Timed("gemm_fp8_fast" if fast_accum else "gemm_fp8", 2.0 * M * N * K):
        rc = getattr(lib, name)(epilogue, a_q.data_ptr(), a_q.stride(0), w_q.data_ptr(), w_q.stride(0),
                                scale_a.data_ptr() + 4, scale_w, _ptr(bias), out.data_ptr(), ldc, M, N, K,
                                _ptr(residual), ldr, _ptr(gate), gs, rows_per_gate, _ptr(out2), ldc2, n_split,
                                row_offset, _stream())
    _lib.check(rc, name)
    _count()
    return out


def linear_fp8(x: torch.Tensor, w_q: torch.Tensor, scale_w: float, bias: Optional[torch.Tensor] = None, **kw):
    """Float8 dynamic-activation linear: quantise ``x`` per tensor, then the FP8 GEMM (scratch buffers are reused per
    (device, shape); the launches are stream-ordered)."""
    q, state = fp8_quantize(*_fp8_cast_scratch("tensor", x))
    return gemm_fp8(q, w_q, state, scale_w, bias, **kw)


class Fp8Rows(NamedTuple):
    """A row-quantised activation standing in for the 16-bit tensor it was cast from (torchao PerRow): e4m3 bytes
    ``q`` uint8 [rows, cols], dequantisation scales ``scale`` fp32 [rows], and the ``dtype`` of the source tensor."""
    q: torch.Tensor
    scale: torch.Tensor
    dtype: torch.dtype

    @property
    def shape(self):
        return self.q.shape

    @property
    def device(self):
        return self.q.device


def _rows_out(rows: int, cols: int, device, q: Optional[torch.Tensor], scale: Optional[torch.Tensor],
              qtype: torch.dtype = torch.uint8):
    if q is None:
        q = torch.empty(rows, cols, dtype=qtype, device=device)
    if scale is None:
        scale = torch.empty(rows, dtype=torch.float32, device=device)
    _req(q, "q", qtype); _req(scale, "scale", torch.float32)
    if q.shape[0] < rows or q.shape[-1] < cols or q.stride(-1) != 1 or scale.numel() < rows or not scale.is_contiguous():
        raise _lib.KreaB200Error(f"quantised rows: q must be [>= {rows}, >= {cols}] with contiguous rows and scale "
                                 f"[>= {rows}]")
    return q, scale


def fp8_quantize_rows(x: torch.Tensor, q: Optional[torch.Tensor] = None,
                      scale: Optional[torch.Tensor] = None) -> Fp8Rows:
    """Dynamic per-row e4m3 cast (torchao Float8DynamicActivation, PerRow): x [rows, cols] bf16 (row pitch free) ->
    Fp8Rows(q uint8 [rows, cols], scale fp32 [rows] = amax_r / 448)."""
    _req(x, "x", torch.bfloat16)
    rows, ld = _rows2d(x, "x")
    cols = x.shape[-1]
    q, scale = _rows_out(rows, cols, x.device, q, scale)
    lib = _lib.load()
    rc = lib.kr_fp8_quantize_rows(x.data_ptr(), ld, rows, cols, q.data_ptr(), q.stride(0), scale.data_ptr(), _stream())
    _lib.check(rc, "kr_fp8_quantize_rows")
    _count()
    return Fp8Rows(q, scale, x.dtype)


def ln_modulate_fp8(x: torch.Tensor, *, eps: float, weight: Optional[torch.Tensor] = None,
                    bias: Optional[torch.Tensor] = None, mod: Optional[torch.Tensor] = None,
                    shift_idx: int = 0, scale_idx: int = 1, rows_per_frame: int = 0,
                    out: Optional[torch.Tensor] = None, row_offset: int = 0, q: Optional[torch.Tensor] = None,
                    scale: Optional[torch.Tensor] = None) -> Fp8Rows:
    """:func:`ln_modulate` whose output rows are cast to e4m3 per row in the same kernel (exactly
    :func:`fp8_quantize_rows` of the bf16 output).  The bf16 output is written only when ``out`` is given."""
    return _ln_modulate_q("fp8", x, eps, weight, bias, mod, shift_idx, scale_idx, rows_per_frame, out, row_offset,
                          q, scale)


def gemm_fp8_rowwise(a: Fp8Rows, w_q: torch.Tensor, scale_w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
                     epilogue: int = EPI_BIAS, out: Optional[torch.Tensor] = None,
                     residual: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None,
                     rows_per_gate: int = 0, out2: Optional[torch.Tensor] = None, n_split: int = 0,
                     row_offset: int = 0, fast_accum: bool = False) -> torch.Tensor:
    """out[M,N] (bf16) = epilogue((a.q[M,K] @ w_q[N,K]^T) * a.scale[m] * scale_w[n] + bias); w_q e4m3 bytes,
    scale_w fp32 [N] (torch._scaled_mm with row-wise scales).  ``fast_accum`` runs kr_gemm_fp8_rowwise_fast
    (``use_fast_accum=True``) on the same operands."""
    _req(a.q, "a.q", torch.uint8); _req(a.scale, "a.scale", torch.float32)
    _req(w_q, "w_q", torch.uint8); _req(scale_w, "scale_w", torch.float32)
    M, K = a.q.shape
    N = w_q.shape[0]
    if w_q.shape[1] != K or scale_w.numel() != N or not scale_w.is_contiguous() or a.scale.numel() < M:
        raise _lib.KreaB200Error(f"gemm_fp8_rowwise: w_q {tuple(w_q.shape)} / scale_w {tuple(scale_w.shape)} / "
                                 f"a.scale {tuple(a.scale.shape)} do not match M={M} K={K}")
    if out is None:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=a.q.device)
    ldc, ldr, gs, ldc2 = _fp8_epi_pitches(out, residual, gate, out2)
    lib = _lib.load()
    name = "kr_gemm_fp8_rowwise_fast" if fast_accum else "kr_gemm_fp8_rowwise"
    with _Timed("gemm_fp8_fast" if fast_accum else "gemm_fp8", 2.0 * M * N * K, sub="rowwise"):
        rc = getattr(lib, name)(epilogue, a.q.data_ptr(), a.q.stride(0), w_q.data_ptr(), w_q.stride(0),
                                a.scale.data_ptr(), scale_w.data_ptr(), _ptr(bias), out.data_ptr(), ldc, M, N, K,
                                _ptr(residual), ldr, _ptr(gate), gs, rows_per_gate, _ptr(out2), ldc2, n_split,
                                row_offset, _stream())
    _lib.check(rc, name)
    _count()
    return out


def linear_fp8_rowwise(x, w_q: torch.Tensor, scale_w: torch.Tensor, bias: Optional[torch.Tensor] = None, **kw):
    """Float8 dynamic-activation linear with PerRow granularity: ``x`` is a bf16 activation (cast per row here, into
    scratch reused per (device, rows, cols); the launches are stream-ordered) or an :class:`Fp8Rows` already cast by
    :func:`ln_modulate_fp8` / :func:`fp8_quantize_rows`; then the row-scaled FP8 GEMM."""
    if not isinstance(x, Fp8Rows):
        x = fp8_quantize_rows(*_fp8_cast_scratch("rows", x))
    return gemm_fp8_rowwise(x, w_q, scale_w, bias, **kw)


class Fp8Blocks(NamedTuple):
    """A block-quantised activation standing in for the 16-bit tensor it was cast from (torchao PerBlock [1, 128]):
    e4m3 bytes ``q`` uint8 [rows, cols], dequantisation scales ``scale`` fp32 [cols / 128, ld_s >= rows] stored
    k-block-major (``scale[g, r]`` belongs to channels [128 g, 128 g + 128) of row r), and the source ``dtype``."""
    q: torch.Tensor
    scale: torch.Tensor
    dtype: torch.dtype

    @property
    def shape(self):
        return self.q.shape

    @property
    def device(self):
        return self.q.device


def _blocks_out(rows: int, cols: int, device, q: Optional[torch.Tensor], scale: Optional[torch.Tensor]):
    if cols % 128 != 0:
        raise _lib.KreaB200Error(f"fp8 blocks: cols={cols} is not a multiple of 128")
    if q is None:
        q = torch.empty(rows, cols, dtype=torch.uint8, device=device)
    if scale is None:
        scale = torch.empty(cols // 128, rows, dtype=torch.float32, device=device)
    _req(q, "q", torch.uint8); _req(scale, "scale", torch.float32)
    if (q.shape[0] < rows or q.shape[-1] < cols or q.stride(-1) != 1 or scale.dim() != 2 or
            scale.shape[0] != cols // 128 or scale.shape[1] < rows or scale.stride(-1) != 1):
        raise _lib.KreaB200Error(f"fp8 blocks: q must be [>= {rows}, >= {cols}] with contiguous rows and scale "
                                 f"[{cols // 128}, >= {rows}] with contiguous rows")
    return q, scale


def _ln_modulate_q(cast: str, x: torch.Tensor, eps: float, weight, bias, mod, shift_idx: int, scale_idx: int,
                   rows_per_frame: int, out, row_offset: int, q, scale):
    """The body of :func:`ln_modulate_fp8` (``cast`` "fp8": per-row e4m3), :func:`ln_modulate_fp8_blocks`
    ("fp8_blocks": per-group e4m3) and :func:`ln_modulate_i8` ("i8": per-row s8)."""
    name = "ln_modulate_" + cast
    blocks = cast == "fp8_blocks"
    _req(x, "x", torch.bfloat16)
    rows, ldx = _rows2d(x, "x")
    D = x.shape[-1]
    ldo = 0
    if out is not None:
        _req(out, "out", torch.bfloat16)
        _, ldo = _rows2d(out, "out")
    mod_rows = 0
    if mod is not None:
        _req(mod, "mod", torch.bfloat16)
        if not mod.is_contiguous() or mod.shape[-1] != D:
            raise _lib.KreaB200Error(f"{name}: mod must be contiguous [frames, rows, D]")
        mod_rows = mod.shape[-2]
    if blocks:
        q, scale = _blocks_out(rows, D, x.device, q, scale)
    else:
        q, scale = _rows_out(rows, D, x.device, q, scale, torch.int8 if cast == "i8" else torch.uint8)
    ld_s = (scale.stride(0),) if blocks else ()
    lib = _lib.load()
    rc = getattr(lib, "kr_" + name)(x.data_ptr(), ldx, _ptr(out), ldo, rows, D, eps, _ptr(weight), _ptr(bias),
                                    _ptr(mod), mod_rows, shift_idx, scale_idx, rows_per_frame, row_offset,
                                    q.data_ptr(), q.stride(0), scale.data_ptr(), *ld_s, _stream())
    _lib.check(rc, "kr_" + name)
    _count()
    return {"fp8": Fp8Rows, "fp8_blocks": Fp8Blocks, "i8": I8Rows}[cast](q, scale, x.dtype)


def fp8_quantize_blocks(x: torch.Tensor, q: Optional[torch.Tensor] = None,
                        scale: Optional[torch.Tensor] = None) -> Fp8Blocks:
    """Dynamic per-group e4m3 cast (torchao PerBlock [1, 128]): x [rows, cols] bf16 (row pitch free, cols % 128 == 0)
    -> Fp8Blocks(q uint8 [rows, cols], scale fp32 [cols / 128, rows] = amax / 448 of each 128-channel group)."""
    _req(x, "x", torch.bfloat16)
    rows, ld = _rows2d(x, "x")
    cols = x.shape[-1]
    q, scale = _blocks_out(rows, cols, x.device, q, scale)
    lib = _lib.load()
    rc = lib.kr_fp8_quantize_blocks(x.data_ptr(), ld, rows, cols, q.data_ptr(), q.stride(0), scale.data_ptr(),
                                    scale.stride(0), _stream())
    _lib.check(rc, "kr_fp8_quantize_blocks")
    _count()
    return Fp8Blocks(q, scale, x.dtype)


def ln_modulate_fp8_blocks(x: torch.Tensor, *, eps: float, weight: Optional[torch.Tensor] = None,
                           bias: Optional[torch.Tensor] = None, mod: Optional[torch.Tensor] = None,
                           shift_idx: int = 0, scale_idx: int = 1, rows_per_frame: int = 0,
                           out: Optional[torch.Tensor] = None, row_offset: int = 0, q: Optional[torch.Tensor] = None,
                           scale: Optional[torch.Tensor] = None) -> Fp8Blocks:
    """:func:`ln_modulate` whose output rows are cast to e4m3 per 128-channel group in the same kernel (exactly
    :func:`fp8_quantize_blocks` of the bf16 output).  The bf16 output is written only when ``out`` is given."""
    return _ln_modulate_q("fp8_blocks", x, eps, weight, bias, mod, shift_idx, scale_idx, rows_per_frame, out,
                          row_offset, q, scale)


def gemm_fp8_blockwise(a: Fp8Blocks, w_q: torch.Tensor, scale_w: torch.Tensor, bias: Optional[torch.Tensor] = None,
                       *, epilogue: int = EPI_BIAS, out: Optional[torch.Tensor] = None,
                       residual: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None,
                       rows_per_gate: int = 0, out2: Optional[torch.Tensor] = None, n_split: int = 0,
                       row_offset: int = 0) -> torch.Tensor:
    """out[M,N] = epilogue(sum over 128-wide k-blocks kb of (a.q[:, kb] @ w_q[:, kb]^T) * a.scale[kb, m] *
    scale_w[n / 128, kb] + bias); w_q e4m3 bytes, scale_w fp32 [N/128, K/128] (torch._scaled_mm with BlockWise1x128 /
    BlockWise128x128 scales).  bf16 output, or fp32 with ``epilogue=EPI_F32``."""
    _req(a.q, "a.q", torch.uint8); _req(a.scale, "a.scale", torch.float32)
    _req(w_q, "w_q", torch.uint8); _req(scale_w, "scale_w", torch.float32)
    M, K = a.q.shape
    N = w_q.shape[0]
    if (w_q.shape[1] != K or K % 128 or N % 128 or tuple(scale_w.shape) != (N // 128, K // 128) or
            not scale_w.is_contiguous() or a.scale.dim() != 2 or a.scale.shape[0] != K // 128 or
            a.scale.shape[1] < M or a.scale.stride(-1) != 1):
        raise _lib.KreaB200Error(f"gemm_fp8_blockwise: w_q {tuple(w_q.shape)} / scale_w {tuple(scale_w.shape)} / "
                                 f"a.scale {tuple(a.scale.shape)} do not match M={M} K={K}")
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32 if epilogue == EPI_F32 else torch.bfloat16, device=a.q.device)
    ldc, ldr, gs, ldc2 = _fp8_epi_pitches(out, residual, gate, out2)
    lib = _lib.load()
    with _Timed("gemm_fp8", 2.0 * M * N * K, sub="blockwise"):
        rc = lib.kr_gemm_fp8_blockwise(epilogue, a.q.data_ptr(), a.q.stride(0), w_q.data_ptr(), w_q.stride(0),
                                       a.scale.data_ptr(), a.scale.stride(0), scale_w.data_ptr(), _ptr(bias),
                                       out.data_ptr(), ldc, M, N, K, _ptr(residual), ldr, _ptr(gate), gs,
                                       rows_per_gate, _ptr(out2), ldc2, n_split, row_offset, _stream())
    _lib.check(rc, "kr_gemm_fp8_blockwise")
    _count()
    return out


def linear_fp8_blockwise(x, w_q: torch.Tensor, scale_w: torch.Tensor, bias: Optional[torch.Tensor] = None, **kw):
    """Float8 dynamic-activation linear with PerBlock granularity: ``x`` is a bf16 activation (cast per 128-channel
    group here, into scratch reused per (device, rows, cols); the launches are stream-ordered) or an
    :class:`Fp8Blocks` already cast by :func:`ln_modulate_fp8_blocks` / :func:`fp8_quantize_blocks`; then the
    block-scaled FP8 GEMM."""
    if not isinstance(x, Fp8Blocks):
        x = fp8_quantize_blocks(*_fp8_cast_scratch("blocks", x))
    return gemm_fp8_blockwise(x, w_q, scale_w, bias, **kw)


class I8Rows(NamedTuple):
    """A row-quantised s8 activation standing in for the 16-bit tensor it was cast from (torchao
    Int8DynamicActivation, per token): ``q`` int8 [rows, cols], dequantisation scales ``scale`` fp32 [rows] =
    amax_r / 127, and the ``dtype`` of the source tensor."""
    q: torch.Tensor
    scale: torch.Tensor
    dtype: torch.dtype

    @property
    def shape(self):
        return self.q.shape

    @property
    def device(self):
        return self.q.device


def i8_quantize_rows(x: torch.Tensor, q: Optional[torch.Tensor] = None,
                     scale: Optional[torch.Tensor] = None) -> I8Rows:
    """Dynamic per-row symmetric s8 cast (torchao Int8DynamicActivation): x [rows, cols] bf16 (row pitch free) ->
    I8Rows(q int8 [rows, cols] = clamp(rint(x * (127 / amax_r)), -127, 127), scale fp32 [rows] = amax_r / 127)."""
    _req(x, "x", torch.bfloat16)
    rows, ld = _rows2d(x, "x")
    cols = x.shape[-1]
    q, scale = _rows_out(rows, cols, x.device, q, scale, torch.int8)
    lib = _lib.load()
    rc = lib.kr_i8_quantize_rows(x.data_ptr(), ld, rows, cols, q.data_ptr(), q.stride(0), scale.data_ptr(), _stream())
    _lib.check(rc, "kr_i8_quantize_rows")
    _count()
    return I8Rows(q, scale, x.dtype)


def ln_modulate_i8(x: torch.Tensor, *, eps: float, weight: Optional[torch.Tensor] = None,
                   bias: Optional[torch.Tensor] = None, mod: Optional[torch.Tensor] = None,
                   shift_idx: int = 0, scale_idx: int = 1, rows_per_frame: int = 0,
                   out: Optional[torch.Tensor] = None, row_offset: int = 0, q: Optional[torch.Tensor] = None,
                   scale: Optional[torch.Tensor] = None) -> I8Rows:
    """:func:`ln_modulate` whose output rows are cast to s8 per row in the same kernel (exactly
    :func:`i8_quantize_rows` of the bf16 output).  The bf16 output is written only when ``out`` is given."""
    return _ln_modulate_q("i8", x, eps, weight, bias, mod, shift_idx, scale_idx, rows_per_frame, out, row_offset,
                          q, scale)


def gemm_i8_rowwise(a: I8Rows, w_q: torch.Tensor, scale_w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
                    epilogue: int = EPI_BIAS, out: Optional[torch.Tensor] = None,
                    residual: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None,
                    rows_per_gate: int = 0, out2: Optional[torch.Tensor] = None, n_split: int = 0,
                    row_offset: int = 0) -> torch.Tensor:
    """out[M,N] = epilogue((float(a.q[M,K] @ w_q[N,K]^T) * a.scale[m]) * scale_w[n] + bias), the product summed
    exactly in s32; w_q int8, scale_w fp32 [N].  bf16 output, or fp32 with ``epilogue=EPI_F32``."""
    _req(a.q, "a.q", torch.int8); _req(a.scale, "a.scale", torch.float32)
    _req(w_q, "w_q", torch.int8); _req(scale_w, "scale_w", torch.float32)
    M, K = a.q.shape
    N = w_q.shape[0]
    if w_q.shape[1] != K or scale_w.numel() != N or not scale_w.is_contiguous() or a.scale.numel() < M:
        raise _lib.KreaB200Error(f"gemm_i8_rowwise: w_q {tuple(w_q.shape)} / scale_w {tuple(scale_w.shape)} / "
                                 f"a.scale {tuple(a.scale.shape)} do not match M={M} K={K}")
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32 if epilogue == EPI_F32 else torch.bfloat16, device=a.q.device)
    ldc, ldr, gs, ldc2 = _fp8_epi_pitches(out, residual, gate, out2)
    lib = _lib.load()
    with _Timed("gemm_i8", 2.0 * M * N * K):
        rc = lib.kr_gemm_i8_rowwise(epilogue, a.q.data_ptr(), a.q.stride(0), w_q.data_ptr(), w_q.stride(0),
                                    a.scale.data_ptr(), scale_w.data_ptr(), _ptr(bias), out.data_ptr(), ldc, M, N, K,
                                    _ptr(residual), ldr, _ptr(gate), gs, rows_per_gate, _ptr(out2), ldc2, n_split,
                                    row_offset, _stream())
    _lib.check(rc, "kr_gemm_i8_rowwise")
    _count()
    return out


def linear_i8(x, w_q: torch.Tensor, scale_w: torch.Tensor, bias: Optional[torch.Tensor] = None, **kw):
    """INT8 dynamic-activation linear (torchao Int8DynamicActivationInt8WeightConfig): ``x`` is a bf16 activation
    (cast per row here, into scratch reused per (device, rows, cols); the launches are stream-ordered) or an
    :class:`I8Rows` already cast by :func:`ln_modulate_i8` / :func:`i8_quantize_rows`; then the s8 GEMM."""
    if not isinstance(x, I8Rows):
        x = i8_quantize_rows(*_fp8_cast_scratch("i8", x))
    return gemm_i8_rowwise(x, w_q, scale_w, bias, **kw)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, heads: int,
              out: Optional[torch.Tensor] = None, softmax_scale: Optional[float] = None,
              block_len: int = 0, window: int = 0, pad_keys: int = 0) -> torch.Tensor:
    """q [Lq, heads*128], k/v [Lkv, heads*128] (row pitch free) -> [Lq, heads*128].

    block_len > 0 selects the block-causal mask of get_block_mask (causal_model.py:109-141)."""
    _req(q, "q"); _req(k, "k", q.dtype); _req(v, "v", q.dtype)
    Lq, ldq = _rows2d(q, "q")
    Lkv, ldk = _rows2d(k, "k")
    _, ldv = _rows2d(v, "v")
    hd = q.shape[-1] // heads if q.dim() == 2 else q.shape[-1]
    if hd != 128:
        raise _lib.KreaB200Error(f"attention: head_dim {hd} unsupported (128 only)")
    if out is None:
        out = torch.empty(Lq, heads * 128, dtype=q.dtype, device=q.device)
    _, ldo = _rows2d(out, "out")
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(128)
    lib = _lib.load()
    with _Timed("attention", 4.0 * Lq * Lkv * heads * 128):
        rc = lib.kr_attn_fwd(_DT[q.dtype], q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv,
                             out.data_ptr(), ldo, Lq, Lkv, heads, softmax_scale,
                             1 if block_len > 0 else 0, block_len, window, pad_keys, _stream())
    _lib.check(rc, "kr_attn_fwd")
    _count()
    return out


def sage_buffers(Lq: int, Lkv: int, heads: int, device) -> dict:
    """Fresh buffers of :func:`sage_quantize` (shapes of include/krea_b200.h, kr_sage_quantize)."""
    W, nqb, nkb = heads * 128, (Lq + 15) // 16, (Lkv + 127) // 128
    return dict(
        q_i8=torch.empty(Lq, W, dtype=torch.int8, device=device),
        q_scale=torch.empty(heads, nqb, 8, dtype=torch.float32, device=device),
        k_mean=torch.empty(W, dtype=torch.bfloat16, device=device),
        k_i8=torch.empty(Lkv, W, dtype=torch.int8, device=device),
        k_scale=torch.empty(heads, nkb, 4, dtype=torch.float32, device=device),
        v_t8=torch.empty(W, nkb * 128, dtype=torch.uint8, device=device),
        v_scale=torch.empty(W, dtype=torch.float32, device=device))


def sage_quantize(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, heads: int,
                  buffers: Optional[dict] = None) -> dict:
    """Quantise for :func:`sage_attention`: q [Lq, heads*128], k / v [Lkv, heads*128] bf16 (row pitch free) ->
    dict of q_i8, q_scale, k_mean, k_i8, k_scale, v_t8 (e4m3 bits), v_scale (``buffers`` is filled if given)."""
    _req(q, "q", torch.bfloat16); _req(k, "k", torch.bfloat16); _req(v, "v", torch.bfloat16)
    Lq, ldq = _rows2d(q, "q")
    Lkv, ldk = _rows2d(k, "k")
    _, ldv = _rows2d(v, "v")
    if q.shape[-1] != heads * 128 or k.shape[-1] != heads * 128 or v.shape[-1] != heads * 128:
        raise _lib.KreaB200Error(f"sage_quantize: rows must be heads*128 = {heads * 128} wide (head_dim 128 only)")
    b = buffers if buffers is not None else sage_buffers(Lq, Lkv, heads, q.device)
    lib = _lib.load()
    with _Timed("sage_quantize", 0.0):
        rc = lib.kr_sage_quantize(q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, Lq, Lkv, heads,
                                  b["q_i8"].data_ptr(), b["q_scale"].data_ptr(), b["k_mean"].data_ptr(),
                                  b["k_i8"].data_ptr(), b["k_scale"].data_ptr(), b["v_t8"].data_ptr(),
                                  b["v_scale"].data_ptr(), _stream())
    _lib.check(rc, "kr_sage_quantize")
    _count(3)
    return b


_sage_scratch = {}


def sage_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, *, heads: int,
                   out: Optional[torch.Tensor] = None, softmax_scale: Optional[float] = None) -> torch.Tensor:
    """Quantised attention (the SageAttention sm_90 numerics: INT8 Q/K per thread with smoothed K, e4m3 P.V with fp32
    accumulation), no mask: q [Lq, heads*128], k / v [Lkv, heads*128] bf16 -> bf16 [Lq, heads*128].  The quantised
    buffers are scratch reused per (device, Lq, Lkv, heads); the launches are stream-ordered."""
    _req(q, "q", torch.bfloat16)
    Lq, _ = _rows2d(q, "q")
    Lkv, _ = _rows2d(k, "k")
    key = (q.device.index, Lq, Lkv, heads)
    b = _sage_scratch.get(key)
    if b is None:
        b = _sage_scratch[key] = sage_buffers(Lq, Lkv, heads, q.device)
    sage_quantize(q, k, v, heads=heads, buffers=b)
    if out is None:
        out = torch.empty(Lq, heads * 128, dtype=q.dtype, device=q.device)
    _req(out, "out", torch.bfloat16)
    _, ldo = _rows2d(out, "out")
    if softmax_scale is None:
        softmax_scale = 1.0 / math.sqrt(128)
    lib = _lib.load()
    with _Timed("attention_sage", 4.0 * Lq * Lkv * heads * 128):
        rc = lib.kr_sage_attn(b["q_i8"].data_ptr(), b["q_scale"].data_ptr(), b["k_i8"].data_ptr(),
                              b["k_scale"].data_ptr(), b["v_t8"].data_ptr(), b["v_scale"].data_ptr(), out.data_ptr(),
                              ldo, Lq, Lkv, heads, softmax_scale, _stream())
    _lib.check(rc, "kr_sage_attn")
    _count()
    return out


def t5_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, bias_delta: torch.Tensor,
                 key_mask: Optional[torch.Tensor], *, heads: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """UMT5 self-attention, head_dim 64: q/k/v [L, heads*64] bf16, bias_delta [heads, 2L-1] bf16 (position bias by
    offset k - q), key_mask [L] uint8 or None -> [L, heads*64] (wan/modules/t5.py:86-120 in one launch)."""
    _req(q, "q", torch.bfloat16); _req(k, "k", torch.bfloat16); _req(v, "v", torch.bfloat16)
    _req(bias_delta, "bias_delta", torch.bfloat16)
    L, ldq = _rows2d(q, "q")
    _, ldk = _rows2d(k, "k")
    _, ldv = _rows2d(v, "v")
    if q.shape[-1] != heads * 64 or tuple(bias_delta.shape) != (heads, 2 * L - 1) or not bias_delta.is_contiguous():
        raise _lib.KreaB200Error("t5_attention: need head_dim 64 and a contiguous bias_delta [heads, 2L-1]")
    if key_mask is not None:
        _req(key_mask, "key_mask", torch.uint8)
    if out is None:
        out = torch.empty(L, heads * 64, dtype=q.dtype, device=q.device)
    _, ldo = _rows2d(out, "out")
    lib = _lib.load()
    with _Timed("t5_attention", 4.0 * L * L * heads * 64):
        rc = lib.kr_t5_attn(q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, out.data_ptr(), ldo, L, heads,
                            bias_delta.data_ptr(), _ptr(key_mask), _stream())
    _lib.check(rc, "kr_t5_attn")
    _count()
    return out


def ln_modulate(x: torch.Tensor, *, eps: float, weight: Optional[torch.Tensor] = None,
                bias: Optional[torch.Tensor] = None, mod: Optional[torch.Tensor] = None,
                shift_idx: int = 0, scale_idx: int = 1, rows_per_frame: int = 0,
                out: Optional[torch.Tensor] = None, row_offset: int = 0) -> torch.Tensor:
    """LayerNorm over the last dim (+affine) (+ x*(1+mod[f,scale_idx]) + mod[f,shift_idx])."""
    _req(x, "x", torch.bfloat16)
    rows, ldx = _rows2d(x, "x")
    D = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    _, ldo = _rows2d(out, "out")
    mod_rows = 0
    if mod is not None:
        _req(mod, "mod", torch.bfloat16)
        if not mod.is_contiguous() or mod.shape[-1] != D:
            raise _lib.KreaB200Error("ln_modulate: mod must be contiguous [frames, rows, D]")
        mod_rows = mod.shape[-2]
    lib = _lib.load()
    rc = lib.kr_ln_modulate(x.data_ptr(), ldx, out.data_ptr(), ldo, rows, D, eps, _ptr(weight),
                            _ptr(bias), _ptr(mod), mod_rows, shift_idx, scale_idx, rows_per_frame,
                            row_offset, _stream())
    _lib.check(rc, "kr_ln_modulate")
    _count()
    return out


def qkv_norm_rope(q, k, v, wq, wk, q_out, k_out, v_out, rope, *, head_dim: int, grid_h: int,
                  grid_w: int, start_frame: int, eps: float, row_offset: int = 0) -> None:
    """RMSNorm(q), RMSNorm(k), RoPE, write q_out / K-cache slot / V-cache slot (row views)."""
    _req(q, "q", torch.bfloat16)
    rows, ldq = _rows2d(q, "q")
    _, ldk = _rows2d(k, "k")
    D = q.shape[-1]
    _, ldqo = _rows2d(q_out, "q_out")
    _, ldko = _rows2d(k_out, "k_out")
    ldv = ldvo = 0
    if v is not None:
        _, ldv = _rows2d(v, "v")
        _, ldvo = _rows2d(v_out, "v_out")
    lib = _lib.load()
    rc = lib.kr_qkv_norm_rope(q.data_ptr(), ldq, k.data_ptr(), ldk, _ptr(v), ldv, wq.data_ptr(),
                              wk.data_ptr(), q_out.data_ptr(), ldqo, k_out.data_ptr(), ldko,
                              _ptr(v_out), ldvo, _ptr(rope), rows, D, head_dim, grid_h, grid_w,
                              start_frame, row_offset, eps, _stream())
    _lib.check(rc, "kr_qkv_norm_rope")
    _count()


def qkv_norm_rope_p2p(q, k, v, wq, wk, q_peers, ldqo: int, k_peers, ldko: int, v_peers, ldvo: int, world: int,
                      peer_cols: int, rope, *, head_dim: int, grid_h: int, grid_w: int, start_frame: int,
                      eps: float, row_offset: int = 0) -> None:
    """``qkv_norm_rope`` whose stores are the rows->heads exchange of the multi-GPU mode: ``*_peers`` are ctypes
    arrays of ``world`` device pointers (this rank's first row inside every rank's q buffer / K slot / V slot)."""
    _req(q, "q", torch.bfloat16)
    rows, ldq = _rows2d(q, "q")
    _, ldk = _rows2d(k, "k")
    _, ldv = _rows2d(v, "v")
    lib = _lib.load()
    rc = lib.kr_qkv_norm_rope_p2p(q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, wq.data_ptr(),
                                  wk.data_ptr(), q_peers, ldqo, k_peers, ldko, v_peers, ldvo, world, peer_cols,
                                  _ptr(rope), rows, q.shape[-1], head_dim, grid_h, grid_w, start_frame,
                                  row_offset, eps, _stream())
    _lib.check(rc, "kr_qkv_norm_rope_p2p")
    _count()


def comm_scatter_rows(src: torch.Tensor, dst_peers, ld_dst: int, rows_per_peer: int, world: int) -> None:
    """rows [r*rows_per_peer, ...) of ``src`` [rows, cols] -> rank r's buffer ``dst_peers[r]`` (row pitch ld_dst)."""
    _req(src, "src")
    rows, ld = _rows2d(src, "src")
    lib = _lib.load()
    rc = lib.kr_comm_scatter_rows(src.data_ptr(), ld, dst_peers, ld_dst, rows, src.shape[-1], rows_per_peer, world,
                                  _stream())
    _lib.check(rc, "kr_comm_scatter_rows")
    _count()


def kv_roll(cache: torch.Tensor, dst_row: int, src_row: int, rows: int) -> None:
    """In-place ``cache[dst_row:dst_row+rows] = cache[src_row:src_row+rows]`` (dst_row <= src_row, overlap allowed) on a
    [rows, width] 16-bit cache view — the eviction memmove of causal_model.py:363-373 without the clone."""
    _req(cache, "cache")
    n, ld = _rows2d(cache, "cache")
    if src_row + rows > n:
        raise _lib.KreaB200Error(f"kv_roll: rows [{src_row}, {src_row + rows}) exceed the cache ({n} rows)")
    lib = _lib.load()
    rc = lib.kr_kv_roll(cache.data_ptr(), ld, cache.shape[-1], dst_row, src_row, rows, _stream())
    _lib.check(rc, "kr_kv_roll")
    _count()


def rmsnorm(x: torch.Tensor, weight: torch.Tensor, eps: float,
            out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, "x", torch.bfloat16)
    rows, ldx = _rows2d(x, "x")
    D = x.shape[-1]
    if out is None:
        out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    _, ldo = _rows2d(out, "out")
    lib = _lib.load()
    rc = lib.kr_rmsnorm(x.data_ptr(), ldx, out.data_ptr(), ldo, weight.data_ptr(), rows, D, eps,
                        _stream())
    _lib.check(rc, "kr_rmsnorm")
    _count()
    return out


def add_modulation(modulation: torch.Tensor, e0: torch.Tensor,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """modulation [1, R, D] + e0 [F, R, D] -> [F, R, D] (bf16)."""
    _req(modulation, "modulation", torch.bfloat16); _req(e0, "e0", torch.bfloat16)
    F, R, D = e0.shape[-3], e0.shape[-2], e0.shape[-1]
    if e0.stride(-1) != 1 or e0.stride(-2) != D:
        raise _lib.KreaB200Error("add_modulation: e0 rows must be contiguous")
    if out is None:
        out = torch.empty(F, R, D, dtype=e0.dtype, device=e0.device)
    lib = _lib.load()
    rc = lib.kr_add_modulation(modulation.data_ptr(), e0.data_ptr(), e0.stride(-3), out.data_ptr(),
                               F, R, D, _stream())
    _lib.check(rc, "kr_add_modulation")
    _count()
    return out


def activation(x: torch.Tensor, kind: str) -> torch.Tensor:
    _req(x, "x", torch.bfloat16)
    if not x.is_contiguous():
        raise _lib.KreaB200Error("activation: tensor must be contiguous")
    y = torch.empty_like(x)
    lib = _lib.load()
    rc = lib.kr_activation(x.data_ptr(), y.data_ptr(), x.numel(), {"silu": 0, "gelu": 1}[kind],
                           _stream())
    _lib.check(rc, "kr_activation")
    _count()
    return y


def patchify(x: torch.Tensor) -> torch.Tensor:
    """x [C, F, H, W] (any strides) -> [F*(H/2)*(W/2), 4C] bf16, Conv3d(1,2,2) im2col."""
    _req(x, "x", torch.bfloat16)
    C, F, H, W = x.shape
    out = torch.empty(F * (H // 2) * (W // 2), C * 4, dtype=x.dtype, device=x.device)
    lib = _lib.load()
    rc = lib.kr_patchify(x.data_ptr(), x.stride(0), x.stride(1), x.stride(2), x.stride(3),
                         out.data_ptr(), C, F, H, W, _stream())
    _lib.check(rc, "kr_patchify")
    _count()
    return out


def unpatchify_x0(head_out: torch.Tensor, xt: Optional[torch.Tensor], sigma: Optional[torch.Tensor],
                  C: int, F: int, H: int, W: int):
    """head_out [F*h*w, 4C] -> (flow [F,C,H,W], x0 [F,C,H,W] or None)."""
    _req(head_out, "head_out", torch.bfloat16)
    flow = torch.empty(F, C, H, W, dtype=head_out.dtype, device=head_out.device)
    x0 = None
    if xt is not None:
        _req(xt, "xt", torch.bfloat16); _req(sigma, "sigma", torch.float64)
        if not xt.is_contiguous():
            raise _lib.KreaB200Error("unpatchify_x0: xt must be contiguous [F,C,H,W]")
        x0 = torch.empty_like(flow)
    lib = _lib.load()
    rc = lib.kr_unpatchify_x0(head_out.data_ptr(), head_out.stride(0), _ptr(xt), _ptr(sigma),
                              flow.data_ptr(), _ptr(x0), C, F, H, W, _stream())
    _lib.check(rc, "kr_unpatchify_x0")
    _count()
    return flow, x0


# ---------------------------------------------------------------------------------------------
# causal 3D VAE decoder ops (channels-last activations [frames, H, W, C])
# ---------------------------------------------------------------------------------------------
def vae_conv(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], *, n: int, cout: int,
             T: int, taps, tile, out_raw: Optional[torch.Tensor] = None,
             out_norm: Optional[torch.Tensor] = None, gamma: Optional[torch.Tensor] = None,
             residual: Optional[torch.Tensor] = None, out_pix: Optional[torch.Tensor] = None,
             raw_frame_stride: Optional[int] = None, sub2: bool = False) -> None:
    """x [t_in, H, W, cin] (t_in >= T + kt - 1, cached frames in front); weight [rows, taps*cin].

    out_raw / out_norm / residual: channels-last frame stacks [>=T, H, W, C]; ``raw_frame_stride``
    overrides the frame stride of out_raw (time_conv's channel->time interleave)."""
    _req(x, "x"); _req(weight, "weight", x.dtype)
    t_in, H, W, cin = x.shape
    if not x.is_contiguous():
        raise _lib.KreaB200Error("vae_conv: input must be contiguous [frames, H, W, C]")
    kt, kh, kw = taps
    tw, th = tile

    def strides(t):
        if t is None:
            return None, 0, 0
        wo = W // 2 if sub2 else W
        if t.stride(-1) != 1 or t.stride(-3) != wo * t.stride(-2):
            raise _lib.KreaB200Error("vae_conv: outputs must be channels-last with dense rows")
        return t.data_ptr(), t.stride(-2), t.stride(0)

    rp, rpix, rfr = strides(out_raw)
    if raw_frame_stride is not None:
        rfr = raw_frame_stride
    npr, npix, nfr = strides(out_norm)
    sp, spix, sfr = strides(residual)
    lib = _lib.load()
    _fl = 2.0 * T * H * W * n * cin * kt * kh * kw
    with _Timed("vae_conv", _fl):
      rc = lib.kr_vae_conv3d(_DT[x.dtype], cin, n, x.data_ptr(), t_in, weight.data_ptr(), weight.shape[0],
                           _ptr(bias), cout, T, H, W, tw, th, kt, kh, kw, rp, rpix, rfr, npr, npix, nfr,
                           _ptr(gamma), sp, spix, sfr, _ptr(out_pix), 1 if sub2 else 0, _stream())
    _lib.check(rc, "kr_vae_conv3d")
    _count()


def vae_conv_fp8(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], *, n: int, cout: int, T: int,
                 taps, tile, w_scale: Optional[torch.Tensor] = None, in_scale: Optional[float] = None,
                 out_raw: Optional[torch.Tensor] = None, out_norm: Optional[torch.Tensor] = None,
                 norm_scale: Optional[float] = None, gamma: Optional[torch.Tensor] = None,
                 residual: Optional[torch.Tensor] = None, out_pix: Optional[torch.Tensor] = None,
                 sub2: bool = False) -> None:
    """The FP8 tier's conv (kr_vae_conv_fp8): ``vae_conv`` with an e4m3 input and weights when ``x`` is
    ``float8_e4m3fn`` (``weight`` e4m3 [rows, taps*cin] with fp32 channel scales ``w_scale`` [n], ``in_scale`` the
    activation scale s of ``x``), or with fp16 operands otherwise; ``out_norm`` (``float8_e4m3fn``) receives
    e4m3(SiLU(RMS_norm) * ``norm_scale``).  ``sub2``: the encoder's stride-2 conv (kr_vae_conv_fp8_sub2, fp16 operands;
    outputs H/2 x W/2), as in ``vae_conv``."""
    _req(x, "x")
    in_fp8 = x.dtype == torch.float8_e4m3fn
    if not in_fp8 and x.dtype != torch.float16:
        raise _lib.KreaB200Error(f"vae_conv_fp8: input must be float8_e4m3fn or float16, got {x.dtype}")
    _req(weight, "weight", x.dtype)
    if in_fp8:
        if w_scale is None or in_scale is None:
            raise _lib.KreaB200Error("vae_conv_fp8: e4m3 input needs w_scale and in_scale")
        _req(w_scale, "w_scale", torch.float32)
        if w_scale.numel() < n or not w_scale.is_contiguous():
            raise _lib.KreaB200Error(f"vae_conv_fp8: w_scale must be a contiguous [>= {n}] fp32 vector")
    if out_norm is not None:
        _req(out_norm, "out_norm", torch.float8_e4m3fn)
        if norm_scale is None:
            raise _lib.KreaB200Error("vae_conv_fp8: an e4m3 out_norm needs norm_scale")
    for name, t in (("out_raw", out_raw), ("residual", residual), ("bias", bias), ("gamma", gamma)):
        if t is not None and t.dtype != torch.float16:
            raise _lib.KreaB200Error(f"vae_conv_fp8: {name} must be float16, got {t.dtype}")
    t_in, H, W, cin = x.shape
    if not x.is_contiguous():
        raise _lib.KreaB200Error("vae_conv_fp8: input must be contiguous [frames, H, W, C]")
    kt, kh, kw = taps
    tw, th = tile

    def strides(t):
        if t is None:
            return None, 0, 0
        if t.stride(-1) != 1 or t.stride(-3) != (W // 2 if sub2 else W) * t.stride(-2):
            raise _lib.KreaB200Error("vae_conv_fp8: outputs must be channels-last with dense rows")
        return t.data_ptr(), t.stride(-2), t.stride(0)

    rp, rpix, rfr = strides(out_raw)
    npr, npix, nfr = strides(out_norm)
    sp, spix, sfr = strides(residual)
    lib = _lib.load()
    _fl = 2.0 * T * H * W * n * cin * kt * kh * kw
    with _Timed("vae_conv", _fl, "fp8" if in_fp8 else None):
        fn = lib.kr_vae_conv_fp8_sub2 if sub2 else lib.kr_vae_conv_fp8
        rc = fn(1 if in_fp8 else 0, cin, n, x.data_ptr(), t_in, weight.data_ptr(), _ptr(w_scale),
                float(in_scale or 0.0), weight.shape[0], _ptr(bias), cout, T, H, W, tw, th, kt, kh, kw,
                rp, rpix, rfr, npr, npix, nfr, float(norm_scale or 0.0), _ptr(gamma), sp, spix, sfr,
                _ptr(out_pix), _stream())
    _lib.check(rc, "kr_vae_conv_fp8_sub2" if sub2 else "kr_vae_conv_fp8")
    _count()


def vae_rmsnorm_silu_fp8(x: torch.Tensor, gamma: torch.Tensor, out: torch.Tensor, q_scale: float) -> torch.Tensor:
    """e4m3(RMS_norm(x) * sqrt(C) * gamma -> SiLU, then * q_scale) into ``out`` (``float8_e4m3fn``); x fp16."""
    _req(x, "x", torch.float16)
    _req(out, "out", torch.float8_e4m3fn)
    if not (x.is_contiguous() and out.is_contiguous()) or out.shape != x.shape:
        raise _lib.KreaB200Error("vae_rmsnorm_silu_fp8: tensors must be contiguous and of the same shape")
    C = x.shape[-1]
    lib = _lib.load()
    rc = lib.kr_vae_rmsnorm_silu_fp8(x.data_ptr(), out.data_ptr(), gamma.data_ptr(), x.numel() // C, C,
                                     float(q_scale), _stream())
    _lib.check(rc, "kr_vae_rmsnorm_silu_fp8")
    _count()
    return out


def vae_rmsnorm_silu(x: torch.Tensor, gamma: torch.Tensor, out: torch.Tensor, silu: bool = True) -> torch.Tensor:
    _req(x, "x")
    if not (x.is_contiguous() and out.is_contiguous()):
        raise _lib.KreaB200Error("vae_rmsnorm_silu: tensors must be contiguous")
    C = x.shape[-1]
    lib = _lib.load()
    rc = lib.kr_vae_rmsnorm_silu(_DT[x.dtype], x.data_ptr(), out.data_ptr(), gamma.data_ptr(),
                                 x.numel() // C, C, 1 if silu else 0, _stream())
    _lib.check(rc, "kr_vae_rmsnorm_silu")
    _count()
    return out


def vae_upsample2x(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _req(x, "x")
    T, H, W, C = x.shape
    if not (x.is_contiguous() and out.is_contiguous()):
        raise _lib.KreaB200Error("vae_upsample2x: tensors must be contiguous")
    lib = _lib.load()
    rc = lib.kr_vae_upsample2x(x.data_ptr(), out.data_ptr(), T, H, W, C, _stream())
    _lib.check(rc, "kr_vae_upsample2x")
    _count()
    return out


def vae_scale_input(z: torch.Tensor, mean, inv_std, w2, b2, out: torch.Tensor) -> torch.Tensor:
    """z [T, 16, H, W] (any strides) -> out [T, H, W, 64] channels-last, channels >= 16 zero."""
    _req(z, "z")
    T, C, H, W = z.shape
    lib = _lib.load()
    rc = lib.kr_vae_scale_input(_DT[z.dtype], z.data_ptr(), z.stride(0), z.stride(1), z.stride(2),
                                z.stride(3), mean.data_ptr(), inv_std.data_ptr(), w2.data_ptr(),
                                b2.data_ptr(), out.data_ptr(), T, H, W, _stream())
    _lib.check(rc, "kr_vae_scale_input")
    _count()
    return out


def softmax_rows(s: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    _req(s, "s", torch.float32)
    rows, cols = s.shape
    lib = _lib.load()
    rc = lib.kr_softmax_rows(_DT[out.dtype], s.data_ptr(), s.stride(0), out.data_ptr(), out.stride(0),
                             rows, cols, _stream())
    _lib.check(rc, "kr_softmax_rows")
    _count()
    return out


def frames_to_rgb8(pixels: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Decoder output fp32 [..., T, 3, H, W] in [-1, 1] -> uint8 [..., T, H, W, 3] (PIL 'RGB' layout), the bytes
    the reference produces on the host with add_(1).mul_(0.5).clamp_(0, 1) + to_pil_image
    (release_server.py:979-983)."""
    _req(pixels, "pixels", torch.float32)
    if pixels.dim() < 4 or pixels.shape[-3] != 3 or not pixels.is_contiguous():
        raise _lib.KreaB200Error("frames_to_rgb8: expected contiguous fp32 [..., T, 3, H, W]")
    lead, (H, W) = pixels.shape[:-3], pixels.shape[-2:]
    T = 1
    for d in lead:
        T *= int(d)
    if out is None:
        out = torch.empty(*lead, H, W, 3, dtype=torch.uint8, device=pixels.device)
    elif out.dtype != torch.uint8 or not out.is_contiguous() or out.numel() != T * H * W * 3:
        raise _lib.KreaB200Error("frames_to_rgb8: out must be contiguous uint8 [..., T, H, W, 3]")
    lib = _lib.load()
    rc = lib.kr_frames_to_rgb8(pixels.data_ptr(), out.data_ptr(), T, H, W, _stream())
    _lib.check(rc, "kr_frames_to_rgb8")
    _count()
    return out


_jpeg_ws = {}


def frames_to_jpeg(pixels: torch.Tensor, quality: int = 90, *, cap: Optional[int] = None,
                   out: Optional[torch.Tensor] = None, sizes: Optional[torch.Tensor] = None):
    """Decoder output fp32 [..., T, 3, H, W] in [-1, 1] (or RGB bytes uint8 [..., T, H, W, 3]) -> one baseline JPEG
    file per frame, byte-identical to the reference's host-side
    ``TF.to_pil_image(frames[0, idx], "RGB").save(io, format='JPEG', quality=90)`` (release_server.py:973), encoded
    on the device.  Returns ``(out uint8 [T, cap], sizes int32 [T])``: file f is ``out[f, :sizes[f]]``; a negative
    size means the file needs ``-sizes[f]`` bytes and did not fit into ``cap`` (default: the raw RGB size).
    The workspace (coefficients, bit offsets, bit stream) is cached per (device, stream, shape)."""
    if pixels.dtype == torch.float32:
        _req(pixels, "pixels", torch.float32)
        if pixels.dim() < 4 or pixels.shape[-3] != 3 or not pixels.is_contiguous():
            raise _lib.KreaB200Error("frames_to_jpeg: expected contiguous fp32 [..., T, 3, H, W]")
        lead, (H, W) = pixels.shape[:-3], pixels.shape[-2:]
        fn = "kr_frames_to_jpeg"
    else:
        _req(pixels, "pixels", torch.uint8)
        if pixels.dim() < 4 or pixels.shape[-1] != 3 or not pixels.is_contiguous():
            raise _lib.KreaB200Error("frames_to_jpeg: expected contiguous uint8 [..., T, H, W, 3]")
        lead, (H, W) = pixels.shape[:-3], pixels.shape[-3:-1]
        fn = "kr_rgb8_to_jpeg"
    T = 1
    for d in lead:
        T *= int(d)
    H, W = int(H), int(W)
    lib = _lib.load()
    need = lib.kr_jpeg_workspace_bytes(T, H, W)
    if need == 0:
        raise _lib.KreaB200Error(f"frames_to_jpeg: {T} frames of {H}x{W} unsupported (H and W must be multiples of 16)")
    if cap is None:
        cap = (H * W * 3 + 4096 + 3) // 4 * 4
    if out is None:
        out = torch.empty(T, cap, dtype=torch.uint8, device=pixels.device)
    elif out.dtype != torch.uint8 or not out.is_contiguous() or tuple(out.shape) != (T, cap):
        raise _lib.KreaB200Error("frames_to_jpeg: out must be contiguous uint8 [T, cap]")
    if sizes is None:
        sizes = torch.empty(T, dtype=torch.int32, device=pixels.device)
    elif sizes.dtype != torch.int32 or not sizes.is_contiguous() or sizes.numel() != T:
        raise _lib.KreaB200Error("frames_to_jpeg: sizes must be contiguous int32 [T]")
    _req(out, "out"); _req(sizes, "sizes")
    stream = _stream()
    key = (pixels.device.index, stream, T, H, W)
    ws = _jpeg_ws.get(key)
    if ws is None:
        if len(_jpeg_ws) > 8:
            _jpeg_ws.clear()
        ws = _jpeg_ws[key] = torch.empty(need, dtype=torch.uint8, device=pixels.device)
    rc = getattr(lib, fn)(pixels.data_ptr(), T, H, W, int(quality), out.data_ptr(), cap, sizes.data_ptr(),
                          ws.data_ptr(), ws.numel(), stream)
    _lib.check(rc, fn)
    _count(4)
    return out, sizes


def jpeg_files(out: torch.Tensor, sizes: torch.Tensor) -> list:
    """Host-side convenience: the JPEG files of :func:`frames_to_jpeg` as ``bytes`` objects (one small device->host
    read of the sizes, then only the used prefix of every file crosses PCIe)."""
    n = sizes.cpu()
    if int(n.min()) <= 0:
        raise _lib.KreaB200Error(f"frames_to_jpeg: a file did not fit its buffer (sizes {n.tolist()})")
    m = int(n.max())
    host = out[:, :m].cpu()
    return [host[i, :int(n[i])].numpy().tobytes() for i in range(host.shape[0])]
