"""fp32 torch stand-ins of tests/cpu_ops_emulation_vae_fp8.py with the encoder's stride-2 entry point — TEST
INFRASTRUCTURE for tests/test_vae_enc_fp8_cpu.py, which monkeypatches ``vae.ops`` with this module.  Contract:
include/krea_b200_vae_fp8.h kr_vae_conv_fp8 / kr_vae_conv_fp8_sub2."""
from __future__ import annotations

import torch

from tests.cpu_ops_emulation_vae_fp8 import *  # noqa: F401,F403  (every stand-in the encoder schedule calls)
from tests.cpu_ops_emulation_vae_fp8 import E4M3, _e4m3
from tests.cpu_ops_emulation import vae_conv


def vae_conv_fp8(x, weight, bias, *, n, cout, T, taps, tile, w_scale=None, in_scale=None, out_raw=None,
                 out_norm=None, norm_scale=None, gamma=None, residual=None, out_pix=None, sub2=False):
    """kr_vae_conv_fp8 (sub2 = False) / kr_vae_conv_fp8_sub2 (sub2 = True, fp16 operands only): e4m3 operands
    dequantised as acc * (1/s) * w_scale[c], or fp16 operands; out_norm as e4m3 bytes of the fp16 SiLU(RMS_norm) value
    times norm_scale."""
    if x.dtype == E4M3:
        assert not sub2, "kr_vae_conv_fp8_sub2 takes fp16 operands"
        xf = x.float()
        wf = weight.float() * (w_scale.float()[:weight.shape[0], None] * (1.0 / in_scale))
    else:
        xf, wf = x, weight
    norm16 = None if out_norm is None else torch.empty(out_norm.shape, dtype=torch.float16)
    vae_conv(xf, wf, bias, n=n, cout=cout, T=T, taps=taps, tile=tile, out_raw=out_raw, out_norm=norm16, gamma=gamma,
             residual=residual, out_pix=out_pix, sub2=sub2)
    if out_norm is not None:
        out_norm[:T].copy_(_e4m3(norm16[:T], norm_scale))
