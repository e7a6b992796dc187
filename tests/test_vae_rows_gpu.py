"""Per-kernel GPU parity of the VAE row kernels of ``kr_vae.cu`` in fp16 and bf16 against the float64 restatements
of ``tests/kernel_refs.py``, per element:

  * ``vae_rmsnorm_silu``: RMS_norm (F.normalize over C * sqrt(C) * gamma, vae.py:39-54) then SiLU, rounded to 16 bits
    where the reference's eager ops round: the norm, x / norm, * sqrt(C), * gamma, SiLU.  The kernel computes the
    same in fp32, so it differs by <= 1 ulp of the rounded restatement, and only rarely: at most FRAC of the
    elements are not bit-identical (measured on an H100: <= 2.3e-4 in fp16, 0 in bf16).  All-zero pixels give 0, and a
    norm that overflows fp16 gives 0 as the reference's fp16 division by inf does;
  * ``vae_upsample2x``: bit-exact nearest 2x;
  * ``vae_scale_input``: a strided z, one 16-bit rounding per reference op, a 16-term fp32 dot product (bound:
    1 ulp + 16 * 2^-24 * sum |w x|), channels 16-63 exactly 0;
  * ``softmax_rows``: fp32 scores with a row pitch larger than the row, <= 1 ulp of the rounded float64 softmax;
    the padding columns of the output keep their sentinel."""
import pytest
import torch

from tests import kernel_refs as R

pytestmark = pytest.mark.gpu
DTYPES = [torch.float16, torch.bfloat16]
FRAC = 2e-3


def _ops():
    from realtime_video_b200 import ops
    return ops


def _ulps(got, ref, dtype):
    d = (got.double() - ref.double()).abs()
    return float((d / R.ulp(ref, dtype)).max()), float((d != 0).double().mean())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [96, 192, 384, 100])
def test_vae_rmsnorm_silu(C, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(C)
    x = (torch.randn(2, 24, 40, C, device="cuda", generator=g) * 3).to(dtype)
    x[0, 0, 0] = 0                                          # an all-zero pixel
    gamma = (1 + 0.3 * torch.randn(C, device="cuda", generator=g)).to(dtype)
    out = torch.empty_like(x)
    ops.vae_rmsnorm_silu(x, gamma, out)
    ref, exact = R.vae_rmsnorm_silu(x, gamma, dtype)
    worst, frac = _ulps(out, ref, dtype)
    assert worst <= 1 and frac <= FRAC, (worst, frac)
    assert float(out[0, 0, 0].abs().max()) == 0
    print(f"vae_rmsnorm_silu C={C} {dtype}: max {worst:.2f} ulp, {frac:.2e} not identical")


def test_vae_rmsnorm_silu_fp16_norm_overflow():
    """||x|| > 65504 rounds to inf in fp16: x / inf = 0 for every channel, then SiLU(0) = 0."""
    ops = _ops()
    C = 192
    x = torch.full((4, C), 6000.0, device="cuda").half()
    gamma = torch.ones(C, device="cuda").half()
    out = torch.empty_like(x)
    ops.vae_rmsnorm_silu(x, gamma, out)
    ref, _ = R.vae_rmsnorm_silu(x, gamma, torch.float16)
    assert float(ref.abs().max()) == 0 and torch.equal(out, ref.half())


@pytest.mark.parametrize("dtype", DTYPES)
def test_vae_upsample2x(dtype):
    ops = _ops()
    x = torch.randn(3, 12, 20, 96, device="cuda").to(dtype)
    out = torch.empty(3, 24, 40, 96, device="cuda", dtype=dtype)
    ops.vae_upsample2x(x, out)
    assert torch.equal(out, x.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))


@pytest.mark.parametrize("dtype", DTYPES)
def test_vae_scale_input(dtype):
    ops = _ops()
    T, H, W = 3, 30, 52
    g = torch.Generator(device="cuda").manual_seed(7)
    base = torch.randn(H, T, W, 16, device="cuda", generator=g).to(dtype)
    z = base.permute(1, 3, 0, 2)                                # [T, 16, H, W], no dimension contiguous in order
    mean = (0.5 * torch.randn(16, device="cuda", generator=g)).to(dtype)
    inv_std = (0.5 + torch.rand(16, device="cuda", generator=g)).to(dtype)
    w2 = (torch.randn(16, 16, device="cuda", generator=g) / 4).to(dtype)
    b2 = (0.1 * torch.randn(16, device="cuda", generator=g)).to(dtype)
    out = torch.full((T, H, W, 64), 9.0, device="cuda", dtype=dtype)
    ops.vae_scale_input(z, mean, inv_std, w2, b2, out)
    zz = z.permute(0, 2, 3, 1).double()                         # [T, H, W, 16]
    xs = R.r16(R.r16(zz / inv_std.double(), dtype) + mean.double(), dtype)
    exact = xs @ w2.double().t() + b2.double()
    ref = R.r16(exact, dtype)
    tol = R.ulp(ref, dtype) + 16 * 2.0 ** -24 * ((xs.abs() @ w2.double().abs().t()) + b2.double().abs())
    assert bool(((out[..., :16].double() - ref).abs() <= tol).all())
    assert bool((out[..., 16:] == 0).all())


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("cols", [300, 1560])
def test_softmax_rows(cols, dtype):
    ops = _ops()
    rows = 257
    sb = torch.randn(rows, cols + 40, device="cuda") * 4
    s = sb[:, :cols]
    ob = torch.full((rows, cols + 24), 7.0, device="cuda", dtype=dtype)
    ops.softmax_rows(s, ob[:, :cols])
    ref = R.r16(R.softmax_rows(s), dtype)
    worst, frac = _ulps(ob[:, :cols], ref, dtype)
    assert worst <= 1, (worst, frac)
    assert bool((ob[:, cols:] == 7.0).all())
    print(f"softmax_rows cols={cols} {dtype}: max {worst:.2f} ulp, {frac:.2e} not identical")
