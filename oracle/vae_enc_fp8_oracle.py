"""FP8 (e4m3) tier of the VAE encoder (``VAEEncoderWrapper.quant = "fp8"``), restated in fp32 torch.

Same scheme as the decoder's tier (oracle/vae_fp8_oracle.py): the convs whose input is a normalised tensor —
``residual.2`` / ``residual.6`` of every encoder ResidualBlock and ``encoder.head.2`` — read e4m3(x * s) of their input,
s = 448 / max(sqrt(C) * max|gamma|, 0.28) from the gamma of the RMS_norm in front of them, and per-output-channel e4m3
weights.  conv1 on raw pixels, the stride-2 convs, the time_convs, the shortcuts, the middle attention block and
WanVAE_.conv1 stay in fp32 here (fp16 in the product)."""
from __future__ import annotations

from oracle.vae_fp8_oracle import fake_quant_input, fake_quant_weight, input_scale
from oracle.vae_oracle import VAEDecoderOracle, VAEEncoderOracle

FP8_CONV_SUFFIXES = (".residual.2", ".residual.6", "encoder.head.2")


def gamma_of(name: str) -> str:
    """State-dict key of the gamma of the RMS_norm that produces the input of FP8 conv ``name``."""
    if name.endswith(".residual.2"):
        return name[:-len("residual.2")] + "residual.0.gamma"
    if name.endswith(".residual.6"):
        return name[:-len("residual.6")] + "residual.3.gamma"
    return "encoder.head.0.gamma"


class _Fp8CachedConvs(VAEDecoderOracle):
    """The causal-conv / res / attention restatements with the inputs of the convs in ``scales`` fake-quantised (the
    feature cache keeps the quantised input frames, as the product's e4m3 conv-input buffers do)."""

    def __init__(self, params, scales):
        super().__init__(params)
        self.scales = scales

    def _cached_conv(self, name, x, cache, idx):
        if name in self.scales:
            x = fake_quant_input(x, self.scales[name])
        return super()._cached_conv(name, x, cache, idx)


class VAEEncoderFp8Oracle(VAEEncoderOracle):
    """VAEEncoderOracle with the FP8 convs' inputs and weights fake-quantised; ``quant=False`` leaves every conv
    unquantised (then it is VAEEncoderOracle)."""

    def __init__(self, params, quant: bool = True):
        p = dict(params)
        scales = {}
        if quant:
            for k in list(p):
                if k.endswith(".weight") and k[:-len(".weight")].endswith(FP8_CONV_SUFFIXES):
                    name = k[:-len(".weight")]
                    p[k] = fake_quant_weight(p[k])
                    scales[name] = input_scale(p[gamma_of(name)])
        super().__init__(p)
        self.scales = scales
        self.dec = _Fp8CachedConvs(p, scales)
