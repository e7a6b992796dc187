"""GPU parity: sm_90a VAE decoder (through the C ABI) vs golden outputs of the reference
VAEDecoderWrapper and vs the CPU oracle.

Tolerance (stated): the product path stores activations in fp16 (the server's VAE dtype,
release_server.py:196) with fp32 accumulation; goldens are the reference in fp32.  Pixels live
in [-1, 1]; we require rel-L2 <= 2e-2 and mean |d| <= 6e-3 per call (33 convolutions deep).
"""
import pytest
import torch

from oracle.vae_oracle import synthetic_vae_params
from tests import kernel_refs as R
from tests.golden_io import load_npz, rel_l2

pytestmark = pytest.mark.gpu


def build(dtype=torch.float16):
    from realtime_video_b200.vae import VAEDecoderWrapper
    m = VAEDecoderWrapper()
    missing = m.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    assert not missing.unexpected_keys and set(missing.missing_keys) <= {"mean", "std"}
    return m.to(device="cuda", dtype=dtype).eval()


@pytest.mark.parametrize("tag,sub", [("s8x12", 1), ("s16x24", 2)])
def test_decoder_vs_reference_golden(tag, sub):
    g = load_npz("vae_small.npz")
    m = build()
    cache = [None] * 55
    frames = [9, 12, 4]
    with torch.no_grad():
        for call in range(3):
            z = g[f"{tag}/z{call}"].cuda().half()
            px, cache = m(z, *cache)
            assert px.dtype == torch.float32 and px.shape[1] == frames[call]
            assert float(px.max()) <= 1.0 and float(px.min()) >= -1.0
            ref = g[f"{tag}/px{call}"]
            got = px[..., ::sub, ::sub].cpu()
            r = rel_l2(got, ref)
            mad = (got - ref).abs().mean().item()
            assert r < 2e-2 and mad < 6e-3, f"{tag} call {call}: rel_l2={r:.3e} mean|d|={mad:.3e}"


def test_reset_and_cache_roundtrip():
    """Passing [None]*55 restarts the stream; passing the returned cache continues it."""
    g = load_npz("vae_small.npz")
    m = build()
    z0 = g["s8x12/z0"].cuda().half()
    with torch.no_grad():
        a, cache = m(z0, *([None] * 55))
        b, _ = m(g["s8x12/z1"].cuda().half(), *cache)
        a2, cache2 = m(z0, *([None] * 55))
        b2, _ = m(g["s8x12/z1"].cuda().half(), *[c.clone() if c is not None else None for c in cache2])
    assert torch.equal(a, a2) and torch.equal(b, b2)


def test_conv_kernel_vs_torch_conv3d():
    """One causal conv per channel configuration against F.conv3d (fp32) on the same fp16 data."""
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import _prep_conv, _tile_for
    import torch.nn.functional as F
    torch.manual_seed(0)
    for (cin, cout, taps, H, W, T) in [(96, 96, (3, 3, 3), 20, 28, 3), (192, 192, (3, 3, 3), 12, 20, 2),
                                       (384, 384, (3, 3, 3), 10, 14, 1), (192, 384, (1, 1, 1), 9, 17, 2),
                                       (384, 192, (1, 3, 3), 16, 16, 2), (192, 96, (1, 3, 3), 24, 40, 1),
                                       (384, 384, (3, 1, 1), 8, 12, 2)]:
        kt, kh, kw = taps
        w = (torch.randn(cout, cin, kt, kh, kw) / (cin * kt * kh * kw) ** 0.5).half()
        b = (torch.randn(cout) * 0.1).half()
        x = torch.randn(T + kt - 1, H, W, cin).half()
        ref = F.conv3d(F.pad(x.float().permute(3, 0, 1, 2)[None], (kw // 2, kw // 2, kh // 2, kh // 2, 0, 0)),
                       w.float(), b.float())[0].permute(1, 2, 3, 0)            # [T, H, W, cout]
        c = _prep_conv(w, b, torch.float16, "cuda")
        out = torch.empty(T, H, W, cout, dtype=torch.float16, device="cuda")
        ops.vae_conv(x.cuda().contiguous(), c.weight, c.bias, n=c.n, cout=c.cout, T=T, taps=taps,
                     tile=_tile_for(H, W), out_raw=out)
        r = rel_l2(out, ref)
        assert r < 2e-3, f"conv {cin}->{cout} taps {taps}: rel_l2={r:.3e}"
        if c.n != cout:
            continue
        # fused epilogue: out_raw = r16(res + r16(conv + bias)), out_norm = SiLU(RMS_norm(out_raw) * sqrt(C) * gamma).
        # The conv sum differs from fp32 torch only in its order (<= 1 ulp of r16(conv)); the norm is checked on the
        # kernel's own raw output, so it must match the rounded restatement to 1 ulp with few non-identical elements.
        res = torch.randn(T, H, W, cout, device="cuda").half()
        gam = (1 + 0.3 * torch.randn(cout, device="cuda")).half()
        raw2 = torch.empty(T, H, W, cout, dtype=torch.float16, device="cuda")
        nrm = torch.empty_like(raw2)
        ops.vae_conv(x.cuda().contiguous(), c.weight, c.bias, n=c.n, cout=c.cout, T=T, taps=taps,
                     tile=_tile_for(H, W), out_raw=raw2, out_norm=nrm, gamma=gam, residual=res)
        y = R.r16(ref.double().cuda(), torch.float16)
        want = R.r16(res.double() + y, torch.float16)
        d = (raw2.double() - want).abs()
        assert bool((d <= R.ulp(y, torch.float16) + R.ulp(want, torch.float16)).all()), (cin, cout, taps)
        frac = float((d != 0).double().mean())
        assert frac <= 2e-2, (cin, cout, taps, frac)
        nref, _ = R.vae_rmsnorm_silu(raw2, gam, torch.float16)
        dn = (nrm.double() - nref).abs()
        worst_n = float((dn / R.ulp(nref, torch.float16)).max())
        frac_n = float((dn != 0).double().mean())
        assert worst_n <= 1 and frac_n <= 2e-2, (cin, cout, taps, worst_n, frac_n)
        print(f"conv {cin}->{cout} taps {taps}: residual {frac:.2e} not identical; norm {worst_n:.2f} ulp, "
              f"{frac_n:.2e} not identical")


def test_single_frame_wrapper_vs_reference_golden():
    """demo_utils.vae.VAEDecoderWrapperSingle semantics (4 frames even for the first latent)."""
    from realtime_video_b200.vae import VAEDecoderWrapperSingle
    g = load_npz("vae_small.npz")
    m = VAEDecoderWrapperSingle()
    m.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    m = m.to(device="cuda", dtype=torch.float16).eval()
    h, w = 8, 12
    shapes = [(16, h, w)] + [(384, h, w)] * 11 + [(192, 2 * h, 2 * w)] + [(384, 2 * h, 2 * w)] * 6 \
        + [(192, 4 * h, 4 * w)] * 6 + [(96, 8 * h, 8 * w)] * 7
    cache = [torch.zeros(1, c, 2, hh, ww, device="cuda", dtype=torch.float16) for (c, hh, ww) in shapes]
    with torch.no_grad():
        for i in range(3):
            z = g[f"single8x12/z{i}"].cuda().half()
            px, cache = m(z, torch.tensor(i == 0, device="cuda"), *cache)
            assert px.shape == (1, 4, 3, 64, 96) and px.dtype == torch.float16 and len(cache) == 32
            ref = g[f"single8x12/px{i}"]
            r = rel_l2(px.float().cpu(), ref)
            assert r < 2e-2, f"single frame {i}: rel_l2={r:.3e}"


@pytest.mark.parametrize("tag", ["enc64x96", "enc128x192"])
def test_encoder_first_frame_vs_reference_golden(tag):
    """First-frame re-encode (release_server.py:571-576): fp16 engine vs the fp32 reference.
    Tolerance: rel-L2 <= 2e-2 on the scaled latent."""
    from realtime_video_b200.vae import VAEEncoderWrapper
    g = load_npz("vae_small.npz")
    m = VAEEncoderWrapper()
    m.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
    m = m.to(device="cuda", dtype=torch.float16).eval()
    with torch.no_grad():
        mu, cache = m(g[f"{tag}/x"].cuda().half(), [None] * 55)
    ref = g[f"{tag}/mu"]
    assert mu.shape == ref.shape
    r = rel_l2(mu, ref)
    assert r < 2e-2, f"{tag}: rel_l2={r:.3e}"


def test_encoder_streaming_vs_reference_golden():
    """Streaming encode (SURVEY.md 8f.1): 1 + 4 + 4 frames on a fresh cache, then 4 + 4 and 4 frames with
    stream=True on the carried cache (release_server.py:518-538), fp16 engine vs the fp32 reference
    VAEEncoderWrapper (tests/golden/make_vae_encoder_stream_goldens.py).  Tolerance: rel-L2 <= 2e-2."""
    from realtime_video_b200.vae import VAEEncoderWrapper
    g = load_npz("vae_encoder_stream.npz")
    m = VAEEncoderWrapper()
    m.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
    m = m.to(device="cuda", dtype=torch.float16).eval()
    cache = [None] * 55
    with torch.no_grad():
        for tag, stream in (("cold9_64x96", False), ("stream8_64x96", True), ("stream4_64x96", True)):
            mu, cache = m(g[f"{tag}/x"].cuda().half(), cache, stream=stream)
            assert mu.shape == g[f"{tag}/mu"].shape
            r = rel_l2(mu, g[f"{tag}/mu"])
            assert r < 2e-2, f"{tag}: rel_l2={r:.3e}"
