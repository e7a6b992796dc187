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

Numerics are a separate tier from the bf16 headline: e4m3 has 3 mantissa bits; tests state the tolerance against the
fp8 oracle (same quantisation, fp32 matmul) and against the bf16 path.
"""
from __future__ import annotations

import torch
from torch import nn

E4M3_MAX = 448.0


class PerTensor:
    """Granularity marker (torchao.quantization.PerTensor)."""


class Float8DynamicActivationFloat8WeightConfig:
    def __init__(self, granularity=None, **unused):
        if granularity is not None and not isinstance(granularity, PerTensor):
            raise NotImplementedError("only the per-tensor granularity the reference server uses is implemented")
        self.granularity = granularity or PerTensor()


@torch.no_grad()
def quantize_weight(w: torch.Tensor):
    """w [N, K] -> (e4m3 bytes as uint8 [N, K], dequantisation scale amax / 448): w_q = sat(w * 448 / amax)."""
    amax = w.detach().abs().max().float().clamp(min=1e-12)
    q = (w.detach().float() * (E4M3_MAX / amax)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return q.view(torch.uint8).contiguous(), float(amax / E4M3_MAX)


@torch.no_grad()
def quantize_(module: nn.Module, config=None, filter_fn=None) -> nn.Module:
    """In-place, like torchao's: every ``nn.Linear`` inside the DiT blocks of ``module`` (a WanDiffusionWrapper, a
    CausalWanModel or any container of CausalWanAttentionBlock) gets FP8 weights.  The bf16 weights stay in place
    (state_dict unchanged); call ``dequantize_`` to go back."""
    if config is not None and not isinstance(config, Float8DynamicActivationFloat8WeightConfig):
        raise NotImplementedError(f"unsupported quantisation config {type(config).__name__}")
    from .dit import CausalWanAttentionBlock
    n = 0
    for blk in module.modules():
        if not isinstance(blk, CausalWanAttentionBlock):
            continue
        for name, lin in blk.named_modules():
            if isinstance(lin, nn.Linear) and lin.weight.shape[0] % 256 == 0 and lin.weight.shape[1] % 16 == 0 and \
                    (filter_fn is None or filter_fn(lin, name)):
                lin._kr_fp8 = quantize_weight(lin.weight)
                n += 1
    if n == 0:
        raise ValueError("quantize_: no DiT block linears found in the module")
    return module


def dequantize_(module: nn.Module) -> nn.Module:
    for lin in module.modules():
        if isinstance(lin, nn.Linear) and hasattr(lin, "_kr_fp8"):
            del lin._kr_fp8
    return module
