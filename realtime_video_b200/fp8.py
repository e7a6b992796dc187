"""FP8 (e4m3) DiT linears — this package's counterpart of the reference's ``enable_fp8`` switch (release_server.py:179-182):

    from torchao.quantization.quant_api import quantize_, Float8DynamicActivationFloat8WeightConfig, PerTensor
    quantize_(transformer, Float8DynamicActivationFloat8WeightConfig(granularity=PerTensor()))

torchao turns every ``nn.Linear`` into: per-tensor dynamic e4m3 cast of the input (scale = 448 / amax), e4m3 weight
with its own per-tensor scale, ``torch._scaled_mm`` with fp32 accumulation and bf16 output.  :func:`quantize_` does the
same to the drop-in transformer: it attaches ``(w_q bytes, scale_w)`` to the Linear modules of the DiT blocks and the
block schedule (realtime_video_b200/dit.py ``_linear``) then runs ``kr_fp8_quantize`` + ``kr_gemm_fp8``
(e4m3 wgmma, the bf16 GEMM's fused epilogues).  The embedding / head linears (0.04 % of the FLOPs) stay
bf16.  ``realtime_video_b200.dropin`` serves this module as ``torchao.quantization.quant_api`` so the server's own three
lines above work unchanged.

``granularity=PerRow()`` (or ``[PerRow(), PerRow()]``) is torchao's row-wise variant: one scale per activation row
(token) and one per weight output channel, so one outlier sets the scale of its own row only, and the scales do not
depend on how the rows are split across GPUs.  The block schedule then runs ``kr_gemm_fp8_rowwise`` fed by
``kr_ln_modulate_fp8`` (the LayerNorm writes e4m3 bytes and row scales directly) or ``kr_fp8_quantize_rows``.

``mm_config=Float8MMConfig(use_fast_accum=True)`` selects fast accumulation: the e4m3 wgmma accumulates in place across
the whole K (``kr_gemm_fp8_fast`` / ``kr_gemm_fp8_rowwise_fast``, a 128 x 256 tile with MMAs kept in flight), which is
what ``torch._scaled_mm(use_fast_accum=True)`` does and what torchao's config asks for when the caller passes no
``mm_config`` (from torchao's published source; torchao is not in the image, so like the rest of the torchao parity
this is unpinned).  This is the one place the default here differs from torchao's: ``mm_config=None`` keeps the
promoted accumulation (every 128-wide k-block's partial sum is added to fp32 registers), because the tensor core's
accumulator keeps fewer mantissa bits than fp32 and the promoted kernel is the one every earlier result was taken
with.  ``KR_FP8_FAST_ACCUM=1`` in the environment makes ``quantize_`` calls that pass no ``mm_config`` choose fast
accumulation, so the reference's unmodified lines reach it.  Weights and scales are the same bytes in both modes.

``granularity=[PerBlock([1, 128]), PerBlock([128, 128])]`` is block scaling (the DeepSeek-V3 FP8 recipe; torchao's
``PerBlock``): one scale per 1 x 128 group of an activation row and one per 128 x 128 block of the weight, so a
channel that is large in every token sets the scale of its own 128-channel group instead of every row's.  The block
schedule then runs ``kr_gemm_fp8_blockwise`` (each 128-wide k-block's partial is multiplied by its two scales when it is
promoted to fp32) fed by ``kr_ln_modulate_fp8_blocks`` or ``kr_fp8_quantize_blocks``.  Block scales need a partial sum
per k-block, so this granularity exists only with promoted accumulation: ``Float8MMConfig(use_fast_accum=True)`` with
``PerBlock`` raises ``NotImplementedError``, and ``KR_FP8_FAST_ACCUM=1`` does not apply to it.

``Int8DynamicActivationInt8WeightConfig()`` is torchao's W8A8 INT8 config: symmetric per-token s8 activations
(q = clamp(rint(x * (127 / amax_r)), -127, 127), scale amax_r / 127), symmetric per-output-channel s8 weights
(q = clamp(rint(w / s_n), -128, 127), s_n = amax_n / 127.5), and an s8 tensor-core GEMM whose s32 sums are exact.  The
block schedule then runs ``kr_gemm_i8_rowwise`` (128 x 256 tile, in-place s32 accumulation, the bf16 GEMM's epilogues
after v = (float(acc) * s_r) * s_n) fed by ``kr_ln_modulate_i8`` or ``kr_i8_quantize_rows``; oracle/int8_oracle.py
restates it.  Against e4m3 PerRow it trades accuracy on heavy tails and channel outliers (a uniform grid of 255 steps)
for accuracy on bounded activations (3 mantissa bits); see DESIGN.md section 5.  INT8 and FP8 attachments exclude each
other: quantising a module with one tier replaces the other's.

Numerics are a separate tier from the bf16 headline: e4m3 has 3 mantissa bits; tests state the tolerance against the
fp8 oracle (same quantisation, fp32 matmul) and against the bf16 path.
"""
from __future__ import annotations

import enum
import os
from dataclasses import dataclass

import torch
from torch import nn

E4M3_MAX = 448.0


class PerTensor:
    """Granularity marker (torchao.quantization.PerTensor)."""


class PerRow:
    """Granularity marker (torchao.quantization.PerRow): per-row activation scales, per-output-channel weight scales."""


BLOCK = 128


class PerBlock:
    """Granularity marker (torchao.quantization.PerBlock): one scale per ``block_size`` block.  Accepted only as the
    pair ``[PerBlock([1, 128]), PerBlock([128, 128])]`` (1 x 128 activation groups, 128 x 128 weight blocks)."""

    def __init__(self, block_size):
        self.block_size = tuple(int(b) for b in block_size)

    def __eq__(self, other):
        return isinstance(other, PerBlock) and other.block_size == self.block_size

    def __hash__(self):
        return hash(("PerBlock", self.block_size))

    def __repr__(self):
        return f"PerBlock({list(self.block_size)})"


@dataclass(frozen=True)
class Float8MMConfig:
    """torchao.float8.inference.Float8MMConfig, field for field.  ``use_fast_accum=True`` runs the FP8 GEMM that
    accumulates inside the tensor core across the whole K; ``False`` the one that promotes every 128-wide k-block to
    fp32.  ``emulate`` and ``pad_inner_dim`` are not implemented (K % 16 == 0 holds for every DiT block linear)."""
    emulate: bool = False
    use_fast_accum: bool = False
    pad_inner_dim: bool = False

    def __post_init__(self):
        if self.emulate or self.pad_inner_dim:
            raise NotImplementedError("Float8MMConfig: emulate=True / pad_inner_dim=True are not implemented")


def _fast_accum_default() -> bool:
    """The A/B switch: ``KR_FP8_FAST_ACCUM=1`` makes quantize_ calls without an mm_config choose fast accumulation."""
    return os.environ.get("KR_FP8_FAST_ACCUM", "0") not in ("", "0")


class Float8DynamicActivationFloat8WeightConfig:
    """``granularity``: ``PerTensor()`` or ``PerRow()``, alone or as an (activation, weight) pair of the same kind, or
    exactly the pair ``[PerBlock([1, 128]), PerBlock([128, 128])]``.  ``mm_config``: a :class:`Float8MMConfig`, or None
    for promoted accumulation (torchao's None means ``use_fast_accum=True``; see the module docstring) unless
    ``KR_FP8_FAST_ACCUM=1``.  ``PerBlock`` is promoted only: ``use_fast_accum=True`` with it raises."""

    def __init__(self, granularity=None, mm_config=None, **unused):
        if mm_config is not None and not isinstance(mm_config, Float8MMConfig):
            raise TypeError(f"mm_config must be a Float8MMConfig or None, got {type(mm_config).__name__}")
        self.mm_config = mm_config
        g = PerTensor() if granularity is None else granularity
        if isinstance(g, PerBlock) or (isinstance(g, (list, tuple)) and any(isinstance(x, PerBlock) for x in g)):
            self.granularity = self._per_block(g)
            if mm_config is not None and mm_config.use_fast_accum:
                raise NotImplementedError(
                    "PerBlock with Float8MMConfig(use_fast_accum=True) is not implemented: block scales are applied "
                    "to each 128-wide k-block's partial sum when it is promoted to fp32, and fast accumulation keeps "
                    "no such partial")
            return
        if isinstance(g, (list, tuple)):
            if len(g) != 2:
                raise ValueError(f"granularity pair must have two entries, got {len(g)}")
            if type(g[0]) is not type(g[1]):
                raise ValueError("activation and weight granularity must be of the same kind, got "
                                 f"{type(g[0]).__name__} and {type(g[1]).__name__}")
            g = g[0]
        if not isinstance(g, (PerTensor, PerRow)):
            raise NotImplementedError(f"granularity {type(g).__name__} is not implemented (PerTensor or PerRow)")
        self.granularity = g

    @staticmethod
    def _per_block(g):
        if not isinstance(g, (list, tuple)) or len(g) != 2:
            raise ValueError("PerBlock granularity is an (activation, weight) pair: "
                             "[PerBlock([1, 128]), PerBlock([128, 128])]")
        if not all(isinstance(x, PerBlock) for x in g):
            raise ValueError("activation and weight granularity must be of the same kind, got "
                             f"{type(g[0]).__name__} and {type(g[1]).__name__}")
        if g[0].block_size != (1, BLOCK) or g[1].block_size != (BLOCK, BLOCK):
            raise NotImplementedError(f"PerBlock block sizes {list(g[0].block_size)} / {list(g[1].block_size)} are "
                                      f"not implemented (activation [1, {BLOCK}], weight [{BLOCK}, {BLOCK}])")
        return g[0]


class MappingType(enum.Enum):
    """torchao.quantization.quant_primitives.MappingType: how a quantised range maps onto the real line."""
    SYMMETRIC = enum.auto()
    SYMMETRIC_NO_CLIPPING_ERR = enum.auto()
    ASYMMETRIC = enum.auto()


class PlainLayout:
    """torchao's default tensor layout (torchao.dtypes.PlainLayout): the quantised weight stored as a dense [N, K]."""


I8_MAX_K = 132104   # 127 * 128 * K < 2^31: the s32 sums of the INT8 GEMM cannot overflow


class Int8DynamicActivationInt8WeightConfig:
    """torchao's W8A8 INT8 config: per-token symmetric s8 activations, per-channel symmetric s8 weights.  Only the
    defaults are implemented: ``layout`` None or :class:`PlainLayout`, ``act_mapping_type`` ``MappingType.SYMMETRIC``
    and ``weight_only_decode=False`` (anything else raises ``NotImplementedError``).  ``set_inductor_config`` is
    accepted and has nothing to configure here."""

    def __init__(self, layout=None, act_mapping_type=MappingType.SYMMETRIC, weight_only_decode=False,
                 set_inductor_config=True):
        if layout is not None and type(layout) is not PlainLayout:
            raise NotImplementedError(f"Int8DynamicActivationInt8WeightConfig: layout {type(layout).__name__} is not "
                                      "implemented (PlainLayout)")
        if act_mapping_type is not MappingType.SYMMETRIC:
            raise NotImplementedError(f"Int8DynamicActivationInt8WeightConfig: act_mapping_type {act_mapping_type} "
                                      "is not implemented (MappingType.SYMMETRIC)")
        if weight_only_decode:
            raise NotImplementedError("Int8DynamicActivationInt8WeightConfig: weight_only_decode=True is not "
                                      "implemented")
        self.layout = layout
        self.act_mapping_type = act_mapping_type
        self.weight_only_decode = weight_only_decode
        self.set_inductor_config = set_inductor_config


@torch.no_grad()
def quantize_weight(w: torch.Tensor):
    """w [N, K] -> (e4m3 bytes as uint8 [N, K], dequantisation scale amax / 448): w_q = sat(w * 448 / amax)."""
    amax = w.detach().abs().max().float().clamp(min=1e-12)
    q = (w.detach().float() * (E4M3_MAX / amax)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8).contiguous(), float(amax / E4M3_MAX)


@torch.no_grad()
def quantize_weight_rows(w: torch.Tensor):
    """w [N, K] -> (e4m3 bytes as uint8 [N, K], fp32 [N] dequantisation scales amax_n / 448), one per output
    channel: w_q[n] = sat(w[n] * 448 / amax_n)."""
    amax = w.detach().float().abs().amax(dim=1, keepdim=True).clamp(min=1e-12)
    mul = torch.full_like(amax, E4M3_MAX) / amax          # a true division, as in the kernels
    q = (w.detach().float() * mul).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8).contiguous(), (amax / E4M3_MAX).squeeze(1).contiguous()


@torch.no_grad()
def quantize_weight_blocks(w: torch.Tensor):
    """w [N, K] (N, K multiples of 128) -> (e4m3 bytes as uint8 [N, K], fp32 [N/128, K/128] dequantisation scales
    amax_b / 448), one per 128 x 128 block: w_q[b] = sat(w[b] * 448 / amax_b), a true division as in
    :func:`quantize_weight_rows`; an all-zero block gets amax 1e-12."""
    N, K = w.shape
    if N % BLOCK or K % BLOCK:
        raise ValueError(f"quantize_weight_blocks: [{N}, {K}] is not a whole number of {BLOCK} x {BLOCK} blocks")
    wb = w.detach().float().reshape(N // BLOCK, BLOCK, K // BLOCK, BLOCK)
    amax = wb.abs().amax(dim=(1, 3), keepdim=True).clamp(min=1e-12)
    mul = torch.full_like(amax, E4M3_MAX) / amax
    q = (wb * mul).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).reshape(N, K)
    return q.view(torch.uint8).contiguous(), (amax / E4M3_MAX).reshape(N // BLOCK, K // BLOCK).contiguous()


@torch.no_grad()
def quantize_weight_int8_rows(w: torch.Tensor):
    """w [N, K] -> (int8 [N, K], fp32 [N] dequantisation scales s_n = amax_n / 127.5), symmetric over [-128, 127]:
    w_q[n] = clamp(rint(w[n] / s_n), -128, 127) (round half to even).  An all-zero channel gets the scale
    torch.finfo(float32).eps (torchao's floor), so it quantises to zeros."""
    amax = w.detach().float().abs().amax(dim=1, keepdim=True)
    scale = (amax / 127.5).clamp(min=torch.finfo(torch.float32).eps)
    q = torch.round(w.detach().float() / scale).clamp(-128, 127).to(torch.int8)
    return q.contiguous(), scale.squeeze(1).contiguous()


def is_int8(lin: nn.Module) -> bool:
    """True when :func:`quantize_` attached INT8 weights to ``lin``."""
    return hasattr(lin, "_kr_i8")


def is_rowwise(lin: nn.Module) -> bool:
    """True when :func:`quantize_` attached per-row (PerRow) FP8 weights to ``lin``."""
    return isinstance(getattr(lin, "_kr_fp8_granularity", None), PerRow)


def is_blockwise(lin: nn.Module) -> bool:
    """True when :func:`quantize_` attached block-scaled (PerBlock) FP8 weights to ``lin``."""
    return isinstance(getattr(lin, "_kr_fp8_granularity", None), PerBlock)


def is_fast_accum(lin: nn.Module) -> bool:
    """True when :func:`quantize_` chose fast accumulation (``Float8MMConfig(use_fast_accum=True)``) for ``lin``."""
    return getattr(lin, "_kr_fp8_fast_accum", False)


@torch.no_grad()
def quantize_(module: nn.Module, config=None, filter_fn=None) -> nn.Module:
    """In-place, like torchao's: every ``nn.Linear`` inside the DiT blocks of ``module`` (a WanDiffusionWrapper, a
    CausalWanModel or any container of CausalWanAttentionBlock) gets FP8 weights.  The bf16 weights stay in place
    (state_dict unchanged); call ``dequantize_`` to go back.  PerTensor attaches ``(w_q, scale_w float)``, PerRow
    ``(w_q, scale_w fp32 [N])``, PerBlock ``(w_q, scale_w fp32 [N/128, K/128])`` (only to Linears with K % 128 == 0)
    on the weight's device.  The accumulation mode of ``config.mm_config`` is recorded
    beside them; the weights and scales do not depend on it.  :class:`Int8DynamicActivationInt8WeightConfig` attaches
    ``(w_q int8, scale_w fp32 [N])`` instead (only to Linears with K <= 132104).  Either replaces what an earlier call
    with the other tier attached."""
    if isinstance(config, Int8DynamicActivationInt8WeightConfig):
        return _quantize_int8(module, filter_fn)
    if config is not None and not isinstance(config, Float8DynamicActivationFloat8WeightConfig):
        raise NotImplementedError(f"unsupported quantisation config {type(config).__name__}")
    gran = config.granularity if config is not None else PerTensor()
    blocks = isinstance(gran, PerBlock)
    quant = quantize_weight_blocks if blocks else quantize_weight_rows if isinstance(gran, PerRow) else quantize_weight
    mm = config.mm_config if config is not None else None
    # PerBlock is promoted only (the config rejects use_fast_accum=True); the environment switch does not apply to it
    fast = False if blocks else _fast_accum_default() if mm is None else mm.use_fast_accum
    from .dit import CausalWanAttentionBlock
    n = 0
    for blk in module.modules():
        if not isinstance(blk, CausalWanAttentionBlock):
            continue
        for name, lin in blk.named_modules():
            if isinstance(lin, nn.Linear) and lin.weight.shape[0] % 256 == 0 and lin.weight.shape[1] % 16 == 0 and \
                    (not blocks or lin.weight.shape[1] % BLOCK == 0) and (filter_fn is None or filter_fn(lin, name)):
                _detach(lin, _I8_ATTRS)
                lin._kr_fp8 = quant(lin.weight)
                lin._kr_fp8_granularity = gran
                if fast:
                    lin._kr_fp8_fast_accum = True
                elif hasattr(lin, "_kr_fp8_fast_accum"):
                    del lin._kr_fp8_fast_accum
                n += 1
    if n == 0:
        raise ValueError("quantize_: no DiT block linears found in the module")
    return module


_FP8_ATTRS = ("_kr_fp8", "_kr_fp8_granularity", "_kr_fp8_fast_accum")
_I8_ATTRS = ("_kr_i8",)


def _detach(lin: nn.Module, attrs) -> None:
    for attr in attrs:
        if hasattr(lin, attr):
            delattr(lin, attr)


def _quantize_int8(module: nn.Module, filter_fn) -> nn.Module:
    from .dit import CausalWanAttentionBlock
    n = 0
    for blk in module.modules():
        if not isinstance(blk, CausalWanAttentionBlock):
            continue
        for name, lin in blk.named_modules():
            N, K = lin.weight.shape if isinstance(lin, nn.Linear) else (0, 0)
            if isinstance(lin, nn.Linear) and N % 256 == 0 and K % 16 == 0 and K <= I8_MAX_K and \
                    (filter_fn is None or filter_fn(lin, name)):
                _detach(lin, _FP8_ATTRS)
                lin._kr_i8 = quantize_weight_int8_rows(lin.weight)
                n += 1
    if n == 0:
        raise ValueError("quantize_: no DiT block linears found in the module")
    return module


def dequantize_(module: nn.Module) -> nn.Module:
    for lin in module.modules():
        if isinstance(lin, nn.Linear):
            _detach(lin, _FP8_ATTRS + _I8_ATTRS)
    return module
