"""The FP8 (e4m3) tier of the VAE encoder on the GPU.

* bytes: every fp16 producer of an e4m3 conv input (conv_in, the stride-2 convs, the (3,1,1) time_convs) writes out_norm
  bytes bit-exact against torch's cast of the fp16 kernel's out_norm times s, and the same raw output;
* per conv: the encoder's new e4m3 convs, (96,192) halo and the (384,32) head, against an fp32 conv of the same e4m3
  operands (rel-L2 <= 2e-3), T = 1 and 4 with non-zero cached frames, at the 832x480 and 1280x720 stage sizes;
* the whole encoder: a fresh 1 + 4k clip and a warm stream=True sequence against the fake-quantised oracle
  (oracle/vae_enc_fp8_oracle.py) at 64x96 and against the fp16 engine at 832x480; determinism and CUDA-graph replay.
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


# (cin, n, taps, sub2, H, W of the conv's input at 832x480 / 1280x720)
PRODUCERS = [(64, 96, (3, 3, 3), False, 480, 832), (96, 96, (1, 3, 3), True, 480, 832),
             (192, 192, (1, 3, 3), True, 240, 416), (384, 384, (1, 3, 3), True, 120, 208),
             (192, 192, (3, 1, 1), False, 120, 208), (384, 384, (3, 1, 1), False, 60, 104),
             (96, 96, (1, 3, 3), True, 720, 1280), (384, 384, (3, 1, 1), False, 90, 160)]


@pytest.mark.parametrize("cin,n,taps,sub2,H,W", PRODUCERS)
def test_e4m3_out_norm_bytes_are_the_cast_of_the_fp16_kernel(cin, n, taps, sub2, H, W):
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_input_scale
    torch.manual_seed(cin + n + H)
    dev = "cuda"
    kt = taps[0]
    T = 1 if kt == 3 and taps[1] == 1 else 2            # the time_convs run one output frame per launch
    x = torch.randn(T + kt - 1, H, W, cin, device=dev).half()
    K = kt * taps[1] * taps[2] * cin
    w = (torch.randn(n, K, device=dev) / K ** 0.5).half()
    b = (torch.randn(n, device=dev) * 0.1).half()
    gamma = torch.randn(n, device=dev).half()
    s = fp8_input_scale(gamma)
    Ho, Wo = (H // 2, W // 2) if sub2 else (H, W)
    kw = dict(n=n, cout=n, T=T, taps=taps, tile=_tile(H, W), gamma=gamma, sub2=sub2)
    n16, raw16 = (torch.empty(T, Ho, Wo, n, device=dev, dtype=torch.float16) for _ in range(2))
    ops.vae_conv(x, w, b, out_raw=raw16, out_norm=n16, **kw)
    n8 = torch.empty(T, Ho, Wo, n, device=dev, dtype=E4M3)
    raw8 = torch.empty(T, Ho, Wo, n, device=dev, dtype=torch.float16)
    ops.vae_conv_fp8(x, w, b, out_raw=raw8, out_norm=n8, norm_scale=s, **kw)
    assert float((n16.float() * s).abs().max()) <= 448.0
    assert torch.equal(raw8, raw16)
    assert torch.equal(n8.view(torch.uint8), (n16.float() * s).to(E4M3).view(torch.uint8))


# (cin, n, H, W of the stage the conv runs at)
CONVS = [(96, 192, 240, 416), (96, 192, 360, 640), (384, 32, 60, 104), (384, 32, 90, 160)]


@pytest.mark.parametrize("T", [1, 4])
@pytest.mark.parametrize("cin,n,H,W", CONVS)
def test_fp8_conv_vs_fp32_conv_of_the_same_e4m3_operands(cin, n, H, W, T):
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_quantize_weight
    torch.manual_seed(cin + n + H + T)
    dev = "cuda"
    w = torch.randn(n, 27 * cin, device=dev) * (torch.rand(n, 1, device=dev) + 0.2) / (27 * cin) ** 0.5
    w_q, w_scale = fp8_quantize_weight(w.half())
    s = 37.5
    x = (torch.randn(T + 2, H, W, cin, device=dev) * 3).to(E4M3)          # cached frames 0, 1 are non-zero too
    bias = (torch.randn(max(n, 32), device=dev) * 0.1).half()
    res = torch.randn(T, H, W, n, device=dev).half()
    w5 = (w_q.float() * w_scale[:, None]).reshape(n, 3, 3, 3, cin).permute(0, 4, 1, 2, 3)
    ref = _ref_conv(x.float() / s, w5)[:T] + bias.float()[:n] + res.float()
    got = torch.empty(T, H, W, n, device=dev, dtype=torch.float16)
    ops.vae_conv_fp8(x, w_q, bias, n=n, cout=n, T=T, taps=(3, 3, 3), tile=_tile(H, W), w_scale=w_scale, in_scale=s,
                     out_raw=got, residual=res)
    r = rel_l2(got.float(), ref)
    print(f"cin={cin} n={n} {H}x{W} T={T}: rel_l2 {r:.3e}")
    assert r <= 2e-3, r
    edge = torch.cat([got[-1, 0].flatten(), got[-1, -1].flatten(), got[-1, :, 0].flatten(), got[-1, :, -1].flatten()])
    edge_ref = torch.cat([ref[-1, 0].flatten(), ref[-1, -1].flatten(), ref[-1, :, 0].flatten(),
                          ref[-1, :, -1].flatten()])
    assert rel_l2(edge.float(), edge_ref) <= 2e-3


def test_fp8_halo_conv_writes_the_e4m3_norm_of_its_raw_output():
    """(96,192) with an e4m3 out_norm: the bytes against the fp16 chain recomputed from the raw output the kernel
    stored (>= 97 % identical bytes, dequantised rel-L2 <= 3e-2, as the decoder's FP8 convs)."""
    from realtime_video_b200 import ops
    from realtime_video_b200.vae import fp8_input_scale, fp8_quantize_weight
    from tests.kernel_refs import vae_rmsnorm_silu
    torch.manual_seed(5)
    dev, T, cin, n, H, W = "cuda", 4, 96, 192, 240, 416
    w_q, w_scale = fp8_quantize_weight((torch.randn(n, 27 * cin, device=dev) / (27 * cin) ** 0.5).half())
    x = (torch.randn(T + 2, H, W, cin, device=dev) * 40).to(E4M3)
    gamma = (torch.rand(n, device=dev) + 0.5).half()
    sq = fp8_input_scale(gamma)
    raw = torch.empty(T, H, W, n, device=dev, dtype=torch.float16)
    nrm = torch.empty(T, H, W, n, device=dev, dtype=E4M3)
    ops.vae_conv_fp8(x, w_q, None, n=n, cout=n, T=T, taps=(3, 3, 3), tile=_tile(H, W), w_scale=w_scale, in_scale=21.0,
                     out_raw=raw, out_norm=nrm, norm_scale=sq, gamma=gamma)
    want16 = vae_rmsnorm_silu(raw.reshape(-1, n), gamma, torch.float16)[0].reshape(raw.shape)
    want = (want16.float() * sq).to(E4M3)
    same = (want.view(torch.uint8) == nrm.view(torch.uint8)).float().mean().item()
    r = rel_l2(nrm.float(), want16.float() * sq)
    print(f"norm bytes identical {same:.4f}, dequantised rel_l2 {r:.3e}")
    assert same >= 0.97 and r <= 3e-2


# ---------------------------------------------------------------------------------------------
# the whole encoder
# ---------------------------------------------------------------------------------------------
def _encoder(quant):
    from realtime_video_b200 import factory
    m = factory.synthetic_vae_encoder(device="cuda")
    m.quant = quant
    return m


def test_encoder_against_the_fake_quant_oracle_at_64x96():
    """Fresh 1 + 4 + 4 frames, then warm 4 + 4 and 4 frames with stream=True.  CPU probe: the fake-quant oracle is at
    6.5e-2 of the fp32 oracle on the cold clip; the fp32 stand-ins of the FP8 engine at 4.5e-2 of the fake-quant
    oracle and those of the fp16 engine at 6.5e-2, so the 5.5e-2 bound also tells an engaged tier from an idle one."""
    from oracle.vae_enc_fp8_oracle import VAEEncoderFp8Oracle
    from oracle.vae_oracle import synthetic_vae_params
    gs = load_npz("vae_encoder_stream.npz")
    o8 = VAEEncoderFp8Oracle({k: v.float() for k, v in synthetic_vae_params(seed=0, encoder=True).items()})
    m = _encoder("fp8")
    cache, co = [None] * 55, {}
    with torch.no_grad():
        for tag, stream in (("cold9_64x96", False), ("stream8_64x96", True), ("stream4_64x96", True)):
            x = gs[f"{tag}/x"]
            mu, cache = m(x.cuda().half(), cache, stream=stream)
            ref, co = o8.forward(x.float(), co, stream=stream)
            r = rel_l2(mu.float().cpu(), ref)
            print(f"{tag}: FP8 encoder vs fake-quant oracle rel_l2 {r:.3e}")
            assert r < 5.5e-2, (tag, r)


def _clip(T, H=480, W=832, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.rand(1, 3, 1, H, W, device="cuda", generator=g) * 2 - 1
    drift = torch.randn(1, 3, T, H, W, device="cuda", generator=g) * 0.05
    return (base + drift.cumsum(2)).clamp(-1, 1).half()


def test_encoder_against_the_fp16_engine_at_832x480():
    a, b = _encoder(None), _encoder("fp8")
    clip, warm = _clip(9), _clip(8, seed=1)
    with torch.no_grad():
        r16, c16 = a(clip, [None] * 55)
        r8, c8 = b(clip, [None] * 55)
        s16, _ = a(warm, c16, stream=True)
        s8, _ = b(warm, c8, stream=True)
    for name, u, v in (("cold 1+4+4", r8, r16), ("warm 4+4", s8, s16)):
        r = rel_l2(u.float(), v.float())
        print(f"832x480 {name}: FP8 vs fp16 encoder rel_l2 {r:.3e}")
        assert 1e-2 < r < 1e-1, (name, r)              # the lower bound: the tier is engaged


def test_encoder_is_deterministic_and_replays_in_a_cuda_graph():
    m = _encoder("fp8")
    clip, warm = _clip(5, 256, 448), _clip(4, 256, 448, seed=1)          # latent 32 x 56: attention rows % 32
    with torch.no_grad():
        a0, c = m(clip, [None] * 55)
        a1, c = m(warm, c, stream=True)
        b0, c = m(clip, [None] * 55)
        b1, c = m(warm, c, stream=True)
        assert torch.equal(a0, b0) and torch.equal(a1, b1)
        # a warm 4-frame chunk as one CUDA graph, replayed from the same cache state as the eager call
        m(clip, [None] * 55)
        snap = [t.clone() if t is not None else None for t in m._engine.export_cache()]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            m(warm, c, stream=True)                             # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        cache = m._engine.export_cache()
        with torch.cuda.graph(g):
            out, _ = m(warm, cache, stream=True)
        for t, v in zip(m._engine.export_cache(), snap):
            if t is not None:
                t.copy_(v)
        g.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, a1)
