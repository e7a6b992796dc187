"""FP8 (e4m3) tier of the VAE decoder (``VAEDecoderWrapper.quant = "fp8"``), restated in fp32 torch.

The convs whose input is a normalised tensor — ``residual.2`` / ``residual.6`` of every ResidualBlock and ``head.2`` —
read e4m3 activations and per-output-channel e4m3 weights:

  s      = 448 / max(sqrt(C) * max|gamma|, 0.28)          static activation scale of the conv's input (gamma of the
                                                          RMS_norm in front of it, C its channels)
  x_q    = e4m3(x * s)                                     x = SiLU(RMS_norm(y) * sqrt(C) * gamma): |x| <= sqrt(C)
                                                          max|gamma| (|SiLU(z)| <= max(|z|, 0.2785)), so x_q never
                                                          saturates
  w_q, ws = e4m3(w / ws[o]), ws[o] = amax_o / 448          per output channel (1 for an all-zero channel)
  out    = (sum x_q * w_q) * (1 / s) * ws[o] + bias

Every other conv, the norms and the attention block stay in fp32 here (fp16 in the product)."""
from __future__ import annotations

import math

import torch

from oracle.vae_oracle import VAEDecoderOracle

E4M3_MAX = 448.0
SILU_NEG_BOUND = 0.28
FP8_CONV_SUFFIXES = (".residual.2", ".residual.6", "decoder.head.2")


def input_scale(gamma: torch.Tensor) -> float:
    """s = 448 / max(sqrt(C) max|gamma|, 0.28) as an fp32 number."""
    bound = max(math.sqrt(gamma.numel()) * gamma.detach().float().abs().max().item(), SILU_NEG_BOUND)
    return float(torch.tensor(E4M3_MAX / bound, dtype=torch.float32).item())


def quantize_weight(w: torch.Tensor):
    """w [cout, ...] -> (e4m3 w_q of the same shape, fp32 scales [cout]) with w ~ w_q * scale."""
    w2 = w.detach().float().reshape(w.shape[0], -1)
    amax = w2.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    w_q = (w2 / scale[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)
    return w_q.reshape(w.shape), scale


def fake_quant_weight(w: torch.Tensor) -> torch.Tensor:
    w_q, scale = quantize_weight(w)
    return w_q.float() * scale.view(-1, *([1] * (w.dim() - 1)))


def fake_quant_input(x: torch.Tensor, s: float) -> torch.Tensor:
    """e4m3(x * s) / s, the value the conv's GEMM sees."""
    return (x.float() * s).to(torch.float8_e4m3fn).float() * (1.0 / s)


def gamma_of(name: str) -> str:
    """State-dict key of the gamma of the RMS_norm that produces the input of FP8 conv ``name``."""
    if name.endswith(".residual.2"):
        return name[:-len("residual.2")] + "residual.0.gamma"
    if name.endswith(".residual.6"):
        return name[:-len("residual.6")] + "residual.3.gamma"
    return "decoder.head.0.gamma"


class VAEDecoderFp8Oracle(VAEDecoderOracle):
    """VAEDecoderOracle with the FP8 convs' inputs and weights fake-quantised (the feature cache keeps the quantised
    input frames, as the product's e4m3 conv-input buffers do)."""

    def __init__(self, params):
        p = dict(params)
        self.scales = {}
        for k in list(p):
            if k.endswith(".weight") and k[:-len(".weight")].endswith(FP8_CONV_SUFFIXES):
                name = k[:-len(".weight")]
                p[k] = fake_quant_weight(p[k])
                self.scales[name] = input_scale(p[gamma_of(name)])
        super().__init__(p)

    def _cached_conv(self, name, x, cache, idx):
        if name in self.scales:
            x = fake_quant_input(x, self.scales[name])
        return super()._cached_conv(name, x, cache, idx)
