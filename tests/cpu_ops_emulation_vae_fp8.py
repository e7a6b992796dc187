"""fp32 torch stand-ins of tests/cpu_ops_emulation.py plus the FP8 VAE entry points — TEST INFRASTRUCTURE for
tests/test_vae_fp8_cpu.py, which monkeypatches ``vae.ops`` with this module.  Contracts: include/krea_b200_vae_fp8.h
kr_vae_conv_fp8 / kr_vae_rmsnorm_silu_fp8."""
from __future__ import annotations

import torch

from tests.cpu_ops_emulation import *  # noqa: F401,F403  (every stand-in the decoder schedule calls)
from tests.cpu_ops_emulation import _rms, vae_conv

E4M3 = torch.float8_e4m3fn


def _e4m3(v16: torch.Tensor, s: float) -> torch.Tensor:
    """e4m3(v * s) of the 16-bit value v, scaled in fp32."""
    return (v16.float() * s).to(E4M3)


def vae_conv_fp8(x, weight, bias, *, n, cout, T, taps, tile, w_scale=None, in_scale=None, out_raw=None,
                 out_norm=None, norm_scale=None, gamma=None, residual=None, out_pix=None):
    """kr_vae_conv_fp8: e4m3 operands (x e4m3) dequantised as acc * (1/s) * w_scale[c], or fp16 operands; out_norm
    as e4m3 bytes of the fp16 SiLU(RMS_norm) value times norm_scale."""
    if x.dtype == E4M3:
        xf = x.float()
        wf = weight.float() * (w_scale.float()[:weight.shape[0], None] * (1.0 / in_scale))
    else:
        xf, wf = x, weight
    norm16 = None
    if out_norm is not None:
        norm16 = torch.empty(out_norm.shape, dtype=torch.float16)
    vae_conv(xf, wf, bias, n=n, cout=cout, T=T, taps=taps, tile=tile, out_raw=out_raw, out_norm=norm16, gamma=gamma,
             residual=residual, out_pix=out_pix)
    if out_norm is not None:
        out_norm[:T].copy_(_e4m3(norm16[:T], norm_scale))


def vae_rmsnorm_silu_fp8(x, gamma, out, q_scale):
    out.copy_(_e4m3(_rms(x.float(), gamma).to(torch.float16), q_scale))
    return out
