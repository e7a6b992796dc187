"""Frame-tiled high-resolution VAE stages without a GPU: the buffer accounting on the meta device (1280x720 fits the
budgets, 832x480 keeps its whole-chunk buffers) and, on the fp32 stand-ins of tests/cpu_ops_emulation*.py, tiled and
untiled decode / encode give identical results for every way the engines are called."""
import pytest
import torch

from oracle.vae_oracle import synthetic_vae_params
from tests import cpu_ops_emulation as emu
from tests import cpu_ops_emulation_vae_fp8 as emu8
from tests.golden_io import load_npz

GiB = 1 << 30


def _decoder_buffers(eng):
    bufs = [eng.conv1.buf]
    for b in eng.blocks:
        if b["kind"] == "res":
            bufs += [b["c1"].buf, b["c2"].buf]
        elif "tcache" in b:
            bufs.append(b["tcache"])
    return bufs + [eng.head.buf]


def _encoder_buffers(eng):
    bufs = [eng.conv_in.buf]
    for b in eng.blocks:
        if b["kind"] == "res":
            bufs += [b["c1"].buf, b["c2"].buf]
        elif "tcache" in b:
            bufs.append(b["tcache"])
    return bufs + [eng.head.buf]


def _nbytes(bufs):
    return sum(t.numel() * t.element_size() for t in bufs)


def _meta_decoder(h, w):
    from realtime_video_b200.vae import VAEDecoderWrapper
    eng = VAEDecoderWrapper().half().engine
    eng._prepare(torch.float16, "meta", h, w)
    return eng


def _meta_encoder(H, W):
    from realtime_video_b200.vae import EncoderEngine, VAEEncoderWrapper
    m = VAEEncoderWrapper().half()
    eng = EncoderEngine(m.encoder, m.conv1, m.mean, m.std)
    eng._prepare(torch.float16, "meta", H, W)
    return eng


# ---------------------------------------------------------------------------------------------
# accounting
# ---------------------------------------------------------------------------------------------
def test_720p_buffers_fit_the_budgets():
    dec = _meta_decoder(90, 160)
    assert dec.frame_tile == 1 and dec.head.buf.shape == (3, 720, 1280, 96)
    assert _nbytes(_decoder_buffers(dec)) <= 8 * GiB
    enc = _meta_encoder(720, 1280)
    assert enc.frame_tile == 1 and enc.conv_in.buf.shape == (3, 720, 1280, 64)
    assert _nbytes(_encoder_buffers(enc)) <= 4.5 * GiB
    # the stages below the tiled segment keep their whole-chunk buffers
    assert dec.conv1.buf.shape[0] == 2 + 3 and enc.head.buf.shape[0] == 2 + 1


def test_480p_keeps_the_whole_chunk_buffers():
    """832x480: one buffer per causal conv for a whole chunk, as before frame tiling existed (decoder: 3 latent
    frames, doubled at every up3d; encoder: 4 pixel frames, halved at every downsample3d)."""
    h, w = 60, 104
    dec = _meta_decoder(h, w)
    want = [(5, h, w, 64)] + [(5, h, w, 384)] * 10 + [(2, h, w, 384)] \
        + [(8, 2 * h, 2 * w, 192)] + [(8, 2 * h, 2 * w, 384)] * 5 + [(2, 2 * h, 2 * w, 384)] \
        + [(14, 4 * h, 4 * w, 192)] * 6 + [(14, 8 * h, 8 * w, 96)] * 7
    assert dec.frame_tile == 12
    assert [tuple(t.shape) for t in _decoder_buffers(dec)] == want
    enc = _meta_encoder(8 * h, 8 * w)
    H, W = 8 * h, 8 * w
    want = [(6, H, W, 64)] + [(6, H, W, 96)] * 4 \
        + [(6, H // 2, W // 2, 96)] + [(6, H // 2, W // 2, 192)] * 3 + [(1, H // 4, W // 4, 192)] \
        + [(4, H // 4, W // 4, 192)] + [(4, H // 4, W // 4, 384)] * 3 + [(1, H // 8, W // 8, 384)] \
        + [(3, H // 8, W // 8, 384)] * 8 + [(3, H // 8, W // 8, 384)]
    assert enc.frame_tile == 4
    assert [tuple(t.shape) for t in _encoder_buffers(enc)] == want


def test_exported_cache_keeps_its_shapes_and_positions_when_tiled():
    dec = _meta_decoder(90, 160)
    views = dec._views()
    assert len(views) == 55 and sum(v is not None for v in views) == 32
    assert all(v.shape[0] == 2 for v in views if v is not None)
    assert views[31].shape == (2, 720, 1280, 96) and all(v is None for v in views[32:])


# ---------------------------------------------------------------------------------------------
# tiled == untiled on the stand-ins
# ---------------------------------------------------------------------------------------------
class _PerFrame:
    """The stand-ins with every conv computed one output frame at a time.  CPU conv3d sums in an order that depends on
    the number of frames; the kernels' does not (tests/test_vae_tiling_gpu.py), so exact equality of tiled and untiled
    runs needs per-frame convs here.  The up3d time_conv (strided output frames) runs unchanged: it is outside the
    tiled segment."""
    FRAMED = ("out_raw", "out_norm", "residual", "out_pix")

    def __init__(self, base):
        self.base = base

    def __getattr__(self, name):
        fn = getattr(self.base, name)
        if not name.startswith("vae_conv"):
            return fn

        def conv(x, weight, bias, *, T, taps, **kw):
            if kw.get("raw_frame_stride") is not None:
                return fn(x, weight, bias, T=T, taps=taps, **kw)
            for t in range(T):
                kwt = {k: v[t:t + 1] if k in self.FRAMED and v is not None else v for k, v in kw.items()}
                fn(x[t:t + taps[0]], weight, bias, T=1, taps=taps, **kwt)
        return conv


@pytest.fixture(scope="module")
def g():
    return load_npz("vae_small.npz")


def _decode(g, monkeypatch, quant, tile):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", _PerFrame(emu8 if quant else emu))
    m = vae.VAEDecoderWrapper()
    m.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    m = m.half().eval()
    m.quant = quant
    m.engine._tile_override = tile
    cache, outs = [None] * 55, []
    with torch.no_grad():
        for call in range(3):                            # first block (1 + 2 latent frames), then later blocks
            px, cache = m(g[f"s8x12/z{call}"].half(), *cache)
            outs.append(px)
    assert m.engine.frame_tile == (tile or 12) and m.engine.head.buf.shape[0] == 2 + (tile or 12)
    return outs, [c.clone() for c in cache if c is not None]


@pytest.mark.parametrize("quant", [None, "fp8"], ids=["fp16", "fp8"])
@pytest.mark.parametrize("tile", [1, 5])
def test_tiled_decode_equals_untiled(g, monkeypatch, quant, tile):
    want, want_cache = _decode(g, monkeypatch, quant, None)
    got, got_cache = _decode(g, monkeypatch, quant, tile)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    for a, b in zip(got_cache, want_cache):
        assert a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize("quant", [None, "fp8"], ids=["fp16", "fp8"])
def test_tiled_single_frame_wrapper_equals_untiled(g, monkeypatch, quant):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", _PerFrame(emu8 if quant else emu))
    h, w = 8, 12
    shapes = [(16, h, w)] + [(384, h, w)] * 11 + [(192, 2 * h, 2 * w)] + [(384, 2 * h, 2 * w)] * 6 \
        + [(192, 4 * h, 4 * w)] * 6 + [(96, 8 * h, 8 * w)] * 7

    def run(tile):
        m = vae.VAEDecoderWrapperSingle()
        m.load_state_dict(synthetic_vae_params(seed=0), strict=False)
        m = m.half().eval()
        m.quant = quant
        m._engine = vae.DecoderEngine(m.decoder, m.conv2, m.mean, m.std, single_mode=True)
        m._engine._tile_override = tile
        cache = [torch.zeros(1, c, 2, hh, ww, dtype=torch.float16) for (c, hh, ww) in shapes]
        outs = []
        with torch.no_grad():
            for i in range(3):
                px, cache = m(g[f"single8x12/z{i}"].half(), torch.tensor(i == 0), *cache)
                outs.append(px)
        return outs

    for a, b in zip(run(3), run(None)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("tile", [1, 3])
def test_tiled_encode_equals_untiled(monkeypatch, tile):
    """1 + 4 + 4 frames on a fresh cache, 4 + 4 with stream=True, then the one-frame re-encode on a fresh cache."""
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", _PerFrame(emu))
    gs = load_npz("vae_encoder_stream.npz")

    def run(t):
        m = vae.VAEEncoderWrapper()
        m.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
        m = m.half().eval()
        m._engine = vae.EncoderEngine(m.encoder, m.conv1, m.mean, m.std)
        m._engine._tile_override = t
        outs = []
        with torch.no_grad():
            mu, cache = m(gs["cold9_64x96/x"].half(), [None] * 55)
            outs.append(mu)
            mu, cache = m(gs["stream8_64x96/x"].half(), cache, stream=True)
            outs += [mu] + [c.clone() for c in cache if c is not None]
            mu, _ = m(gs["stream8_64x96/x"][:, :, :1].half(), [None] * 55)
            outs.append(mu)
        assert m._engine.frame_tile == (t or 4) and m._engine.conv_in.buf.shape[0] == 2 + (t or 4)
        return outs

    got, want = run(tile), run(None)
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
