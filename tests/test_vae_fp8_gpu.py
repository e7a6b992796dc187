"""The FP8 (e4m3) tier of the VAE decoder on the GPU.

* bytes: the e4m3 out_norm of a conv epilogue and the e4m3 RMS_norm + SiLU are bit-exact against torch's cast of the
  16-bit kernels' outputs times s (the 16-bit chain is unchanged, the cast is round-to-nearest);
* per conv: every FP8 instantiation against an fp32 conv of the same e4m3 operands (rel-L2 <= 2e-3, the FP8 GEMM
  bound: the e4m3 wgmma adder alone drifts past it over K = 27 C, the promotion every <= 128 k keeps it), T = 1 and 3
  with non-zero cached frames, borders at 832x480 and 1280x720 widths;
* the whole decoder at 832x480 (first block + two steady blocks) against the fp16 engine, and at 64x96 against the
  fake-quantised oracle (oracle/vae_fp8_oracle.py) and the fp32 oracle; determinism; the server loop with the tier on.
"""
import pytest
import torch
import torch.nn.functional as F

from tests.golden_io import load_npz, rel_l2

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def exact_fp32():
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _tile(H, W):
    from realtime_video_b200.vae import _tile_for
    return _tile_for(H, W)


def _ref_conv(x, w5):
    """fp32 causal conv of channels-last x [t_in, H, W, C] with w5 [n, C, kt, kh, kw] -> [T, H, W, n]."""
    kh, kw = w5.shape[3], w5.shape[4]
    xin = F.pad(x.float().permute(3, 0, 1, 2)[None], (kw // 2, kw // 2, kh // 2, kh // 2, 0, 0))
    return F.conv3d(xin, w5)[0].permute(1, 2, 3, 0)


# (cin, n, latent-stage H at 832x480, halo?)  H x W of the stage the conv runs at
CONVS = [(384, 384, 60, 104), (192, 384, 120, 208), (192, 192, 240, 416), (96, 96, 480, 832), (96, 16, 480, 832)]


@pytest.mark.parametrize("T", [1, 3])
@pytest.mark.parametrize("cin,n,H,W", CONVS + [(384, 384, 90, 160), (96, 96, 720, 1280)])
def test_fp8_conv_vs_fp32_conv_of_the_same_e4m3_operands(cin, n, H, W, T):
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_quantize_weight
    torch.manual_seed(cin + n + H + T)
    dev = "cuda"
    cout = 3 if n == 16 else n
    w = torch.randn(n, 27 * cin, device=dev) * (torch.rand(n, 1, device=dev) + 0.2) / (27 * cin) ** 0.5
    if n == 16:
        w[cout:] = 0
        w *= 0.3
    w_q, w_scale = fp8_quantize_weight(w.half())
    s = 37.5
    x = (torch.randn(T + 2, H, W, cin, device=dev) * 3).to(E4M3)          # cached frames 0, 1 are non-zero too
    bias = (torch.randn(max(n, 32), device=dev) * 0.1).half()
    if n == 16:
        bias[cout:] = 0
    w5 = (w_q.float() * w_scale[:, None]).reshape(n, 3, 3, 3, cin).permute(0, 4, 1, 2, 3)
    ref = _ref_conv(x.float() / s, w5)[:T] + bias.float()[:n]
    if n == 16:
        pix = torch.empty(T, cout, H, W, device=dev)
        ops.vae_conv_fp8(x, w_q, bias, n=n, cout=cout, T=T, taps=(3, 3, 3), tile=_tile(H, W), w_scale=w_scale,
                         in_scale=s, out_pix=pix)
        ref = ref[..., :cout].clamp(-1, 1).permute(0, 3, 1, 2)
        got = pix
    else:
        got = torch.empty(T, H, W, n, device=dev, dtype=torch.float16)
        ops.vae_conv_fp8(x, w_q, bias, n=n, cout=n, T=T, taps=(3, 3, 3), tile=_tile(H, W), w_scale=w_scale,
                         in_scale=s, out_raw=got)
    r = rel_l2(got.float(), ref)
    print(f"cin={cin} n={n} {H}x{W} T={T}: rel_l2 {r:.3e}")
    assert r <= 2e-3, r
    # borders: the outermost rows / columns of the last frame alone
    edge = torch.cat([got[-1, 0].flatten(), got[-1, -1].flatten()] if n != 16 else [got[-1, :, 0].flatten()])
    edge_ref = torch.cat([ref[-1, 0].flatten(), ref[-1, -1].flatten()] if n != 16 else [ref[-1, :, 0].flatten()])
    assert rel_l2(edge.float(), edge_ref) <= 2e-3


@pytest.mark.parametrize("cin,n,H,W", [(384, 384, 60, 104), (192, 384, 60, 104), (192, 192, 120, 208),
                                       (96, 96, 240, 416)])
def test_fp8_conv_fused_epilogue_residual_and_e4m3_norm(cin, n, H, W):
    """Residual add, raw store and the e4m3 out_norm of the FP8 convs (N = 384: the norm's sum of squares completed
    across the two consumer warpgroups).  The norm bytes are checked against the 16-bit chain recomputed from the raw
    output the kernel stored: dequantised rel-L2 <= 3e-2 (e4m3 rounding) and >= 97 % identical bytes."""
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_input_scale, fp8_quantize_weight
    from tests.kernel_refs import vae_rmsnorm_silu
    torch.manual_seed(n + H)
    dev, T = "cuda", 3
    w = torch.randn(n, 27 * cin, device=dev) / (27 * cin) ** 0.5
    w_q, w_scale = fp8_quantize_weight(w.half())
    x = (torch.randn(T + 2, H, W, cin, device=dev) * 40).to(E4M3)
    s = 21.0
    res = torch.randn(T, H, W, n, device=dev).half()
    gamma = (torch.rand(n, device=dev) + 0.5).half()
    sq = fp8_input_scale(gamma)
    raw = torch.empty(T, H, W, n, device=dev, dtype=torch.float16)
    nrm = torch.empty(T, H, W, n, device=dev, dtype=E4M3)
    ops.vae_conv_fp8(x, w_q, None, n=n, cout=n, T=T, taps=(3, 3, 3), tile=_tile(H, W), w_scale=w_scale, in_scale=s,
                     out_raw=raw, out_norm=nrm, norm_scale=sq, gamma=gamma, residual=res)
    w5 = (w_q.float() * w_scale[:, None]).reshape(n, 3, 3, 3, cin).permute(0, 4, 1, 2, 3)
    ref = _ref_conv(x.float() / s, w5)[:T] + res.float()
    assert rel_l2(raw.float(), ref) <= 2e-3
    want16 = vae_rmsnorm_silu(raw.reshape(-1, n), gamma, torch.float16)[0].reshape(raw.shape)
    want = (want16.float() * sq).to(E4M3)
    same = (want.view(torch.uint8) == nrm.view(torch.uint8)).float().mean().item()
    r = rel_l2(nrm.float(), want16.float() * sq)
    print(f"cin={cin} n={n}: norm bytes identical {same:.4f}, dequantised rel_l2 {r:.3e}")
    assert same >= 0.97 and r <= 3e-2


@pytest.mark.parametrize("cin,n,H,W,halo", [(64, 384, 60, 104, False), (384, 192, 120, 208, True),
                                             (192, 96, 480, 832, True)])
def test_e4m3_out_norm_bytes_are_the_cast_of_the_fp16_kernel(cin, n, H, W, halo):
    """The 16-bit producers of FP8 inputs (conv1, the Resample convs): same conv, out_norm as e4m3 — bit-exact against
    torch's cast of the fp16 kernel's out_norm times s."""
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_input_scale
    torch.manual_seed(cin)
    dev, T = "cuda", 2
    kt = 3 if not halo else 1
    x = torch.randn(T + kt - 1, H, W, cin, device=dev).half()
    w = (torch.randn(n, kt * 9 * cin, device=dev) / (kt * 9 * cin) ** 0.5).half()
    b = (torch.randn(n, device=dev) * 0.1).half()
    gamma = (torch.randn(n, device=dev)).half()
    s = fp8_input_scale(gamma)
    kw = dict(n=n, cout=n, T=T, taps=(kt, 3, 3), tile=_tile(H, W), gamma=gamma)
    n16, raw16 = torch.empty(T, H, W, n, device=dev, dtype=torch.float16), torch.empty(T, H, W, n, device=dev,
                                                                                          dtype=torch.float16)
    ops.vae_conv(x, w, b, out_raw=raw16, out_norm=n16, **kw)
    n8, raw8 = torch.empty(T, H, W, n, device=dev, dtype=E4M3), torch.empty(T, H, W, n, device=dev,
                                                                              dtype=torch.float16)
    ops.vae_conv_fp8(x, w, b, out_raw=raw8, out_norm=n8, norm_scale=s, **kw)
    assert torch.equal(raw8, raw16)
    assert torch.equal(n8.view(torch.uint8), (n16.float() * s).to(E4M3).view(torch.uint8))
    assert float((n16.float() * s).abs().max()) <= 448.0


@pytest.mark.parametrize("C", [384, 192])
def test_e4m3_rmsnorm_silu_bytes_are_the_cast_of_the_fp16_kernel(C):
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_input_scale
    x = torch.randn(3, 60, 104, C, device="cuda").half() * 5
    x[0, 0, 0] = 0
    gamma = torch.randn(C, device="cuda").half()
    s = fp8_input_scale(gamma)
    y16 = ops.vae_rmsnorm_silu(x, gamma, torch.empty_like(x))
    y8 = ops.vae_rmsnorm_silu_fp8(x, gamma, torch.empty(x.shape, dtype=E4M3, device="cuda"), s)
    assert torch.equal(y8.view(torch.uint8), (y16.float() * s).to(E4M3).view(torch.uint8))


def _decoders():
    from realtime_video_b200 import factory
    a = factory.synthetic_vae_decoder(device="cuda")
    b = factory.synthetic_vae_decoder(device="cuda")
    b.quant = "fp8"
    return a, b


def test_whole_decoder_832x480_vs_fp16_engine_and_determinism():
    torch.manual_seed(0)
    zs = [torch.randn(1, 3, 16, 60, 104, device="cuda").half() for _ in range(3)]
    ref_dec, dec = _decoders()
    with torch.no_grad():
        cr, c8, c8b = [None] * 55, [None] * 55, [None] * 55
        _, dec2 = _decoders()
        for i, z in enumerate(zs):                       # first block + two steady blocks
            pr, cr = ref_dec(z, *cr)
            p8, c8 = dec(z, *c8)
            p8b, c8b = dec2(z, *c8b)
            r = rel_l2(p8, pr)
            print(f"832x480 block {i}: FP8 vs fp16 engine rel_l2 {r:.3e}, mean|d| {(p8 - pr).abs().mean():.3e}")
            assert r <= 8e-2
            assert torch.equal(p8, p8b)                  # deterministic: no atomics, static scales
    assert sum(c is not None and c.dtype == E4M3 for c in c8) == 29


def test_whole_decoder_vs_fake_quant_and_fp32_oracles():
    from oracle import vae_fp8_oracle as O8
    from oracle.vae_oracle import VAEDecoderOracle, synthetic_vae_params
    g = load_npz("vae_small.npz")
    _, dec = _decoders()
    p = {k: v.float() for k, v in synthetic_vae_params(seed=0).items()}
    o8, o32 = O8.VAEDecoderFp8Oracle(p), VAEDecoderOracle(p)
    c, co8, co32 = [None] * 55, {}, {}
    with torch.no_grad():
        for call in range(3):
            z = g[f"s8x12/z{call}"]
            px, c = dec(z.cuda().half(), *c)
            r8 = rel_l2(px.cpu(), o8.forward(z.float(), co8)[0])
            r32 = rel_l2(px.cpu(), o32.forward(z.float(), co32)[0])
            print(f"64x96 call {call}: vs fake-quant oracle {r8:.3e}, vs fp32 oracle {r32:.3e}")
            assert r8 <= 6e-2 and r32 <= 8e-2


def test_server_loop_with_the_tier_on():
    """The server loop of test_server_loop_gpu.py with the decoder on the FP8 tier: pixels mean|d| against the
    reference-executed golden <= 4e-2 on [-1, 1] (the fp16 decoder is held to 1.5e-2)."""
    import harness
    from realtime_video_b200.factory import synthetic_vae_params
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEEncoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    from tests.golden_io import ReplayRandn, weights
    gold, gd = load_npz("server_loop_small.npz"), load_npz("dit_small.npz")
    draws = [gold[f"keep/draw{i}"] for i in range(int(gold["keep/ndraws"]))]
    tr = WanDiffusionWrapper(model_name="synthetic", timestep_shift=5.0, is_causal=True,
                             model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    tr.model.load_state_dict(weights(gd, torch.bfloat16), strict=False)
    tr = tr.to(device="cuda", dtype=torch.bfloat16).eval().requires_grad_(False)
    for blk in tr.model.blocks:
        blk.self_attn.fuse_projections()
    dec = VAEDecoderWrapper()
    dec.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    dec = dec.to(device="cuda", dtype=torch.float16).eval()
    dec.quant = "fp8"
    enc = VAEEncoderWrapper()
    enc.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
    enc = enc.to(device="cuda", dtype=torch.float16).eval()
    models = harness.build_models(tr, vae_decoder=dec, vae_encoder=enc, device="cuda")
    params = harness.GenerateParams(width=96, height=64, seed=11, kv_cache_num_frames=3, num_blocks=4,
                                    num_denoising_steps=4, keep_first_frame=True)
    with ReplayRandn(draws):
        sess = harness.GenerationSession(params, models, prompt_embeds=gold["prompt_embeds"], device="cuda")
        px = [sess.generate_block().float().cpu() for _ in range(4)]
    for b in range(4):
        ref = gold[f"keep/px{b}_sub"].float()
        mad = (px[b][..., ::2, ::2] - ref).abs().mean().item()
        print(f"server loop block {b}: mean|d| {mad:.3e}")
        assert mad < 4e-2, f"block {b}: mean|d|={mad:.3e}"
