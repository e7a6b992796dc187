"""The FP8 (e4m3) tier of the VAE encoder without a GPU: the fake-quant oracle (oracle/vae_enc_fp8_oracle.py) pinned to
the fp32 encoder oracle and probed against it, the host schedule on the fp32 stand-ins of
tests/cpu_ops_emulation_vae_enc_fp8.py (which convs read e4m3, which write it, the fp16 tier unchanged), the buffer plan
and frame tile, feature-cache round trips, tier switches, the switch, argument validation, and the SASS / resource usage
of the encoder's kernels."""
import ctypes
import re
import shutil
import subprocess

import pytest
import torch

from oracle.vae_enc_fp8_oracle import VAEEncoderFp8Oracle
from oracle.vae_oracle import VAEEncoderOracle, synthetic_vae_params
from tests import cpu_ops_emulation_vae_enc_fp8 as emu
from tests.golden_io import load_npz, rel_l2

E4M3 = torch.float8_e4m3fn
GiB = 1 << 30


@pytest.fixture(scope="module")
def gs():
    return load_npz("vae_encoder_stream.npz")


def encoder(quant="fp8"):
    from realtime_video_b200.vae import VAEEncoderWrapper
    m = VAEEncoderWrapper()
    m.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
    m = m.half().eval()
    m.quant = quant
    return m


def _params():
    return {k: v.float() for k, v in synthetic_vae_params(seed=0, encoder=True).items()}


# ---------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------
def test_fake_quant_oracle_without_quantisation_is_the_fp32_oracle(gs):
    p = _params()
    x = gs["cold9_64x96/x"].float()
    ref, _ = VAEEncoderOracle(p).forward(x, {})
    got, _ = VAEEncoderFp8Oracle(p, quant=False).forward(x, {})
    assert torch.equal(got, ref)


def test_fake_quant_oracle_is_close_to_the_fp32_oracle(gs):
    """The CPU probe the GPU bounds are set from: cold 1 + 4 + 4 frames, then two warm 4-frame chunks."""
    p = _params()
    o32, o8 = VAEEncoderOracle(p), VAEEncoderFp8Oracle(p)
    assert len(o8.scales) == 2 * 10 + 1           # residual.2 / .6 of the 10 ResidualBlocks and head.2
    c32, c8 = {}, {}
    for tag, stream in (("cold9_64x96", False), ("stream8_64x96", True)):
        x = gs[f"{tag}/x"].float()
        ref, c32 = o32.forward(x, c32, stream=stream)
        got, c8 = o8.forward(x, c8, stream=stream)
        r = rel_l2(got, ref)
        print(f"{tag}: fake-quant vs fp32 oracle rel_l2 {r:.3e}")
        assert 0 < r < 1e-1, (tag, r)


# ---------------------------------------------------------------------------------------------
# host schedule on the stand-ins
# ---------------------------------------------------------------------------------------------
class _Recorder:
    def __init__(self, monkeypatch):
        import realtime_video_b200.vae as vae
        self.log = []
        rec = self

        class Ops:
            def __getattr__(self, name):
                fn = getattr(emu, name)
                if not name.startswith("vae_") and name != "kv_roll":
                    return fn

                def wrapped(*a, **kw):
                    x = a[0]
                    on = kw.get("out_norm") if name.startswith("vae_conv") else (a[2] if "rmsnorm" in name else None)
                    rec.log.append(dict(op=name, shape=tuple(x.shape), x=x.dtype, n=kw.get("n"), T=kw.get("T"),
                                        taps=kw.get("taps"), raw=kw.get("out_raw") is not None,
                                        res=kw.get("residual") is not None, sub2=kw.get("sub2", False),
                                        norm=None if on is None else on.dtype, kw=sorted(kw)))
                    return fn(*a, **kw)
                return wrapped

        monkeypatch.setattr(vae, "ops", Ops())


def _canon(e):
    """The launch as the fp16 schedule issues it."""
    op = {"vae_conv_fp8": "vae_conv", "vae_rmsnorm_silu_fp8": "vae_rmsnorm_silu"}.get(e["op"], e["op"])
    return (op, e["shape"], e["n"], e["T"], e["taps"], e["raw"], e["res"], e["sub2"], e["norm"] is not None)


FP16_KW = {"n", "cout", "T", "taps", "tile"}


def test_schedule_reads_and_writes_e4m3_exactly_where_listed(gs, monkeypatch):
    rec = _Recorder(monkeypatch)
    x9, x8 = gs["cold9_64x96/x"].half(), gs["stream8_64x96/x"].half()
    with torch.no_grad():
        m16 = encoder(None)
        _, c = m16(x9, [None] * 55)
        m16(x8, c, stream=True)
        base, rec.log = rec.log, []
        m = encoder("fp8")
        _, c = m(x9, [None] * 55)
        m(x8, c, stream=True)
        q = rec.log
    # the fp16 tier: only vae_conv / vae_rmsnorm_silu, with the keyword sets the engine always passed
    assert not [e for e in base if e["op"].endswith("_fp8")]
    for e in base:
        if e["op"] == "vae_conv":
            assert FP16_KW <= set(e["kw"]) and not {"norm_scale", "w_scale", "in_scale"} & set(e["kw"]), e
    eng = m._engine
    fp8_convs = [c for b in eng.blocks if b["kind"] == "res" for c in (b["c1"], b["c2"])] + [eng.head]
    assert len(fp8_convs) == 21 and all(c.weight.dtype == E4M3 and c.buf.dtype == E4M3 for c in fp8_convs)
    others = [eng.conv_in] + [b["sc"] for b in eng.blocks if b["kind"] == "res" and b["sc"] is not None] \
        + [b[k] for b in eng.blocks if b["kind"] == "down" for k in ("conv", "tconv") if k in b]
    assert all(c.weight.dtype == torch.float16 and c.w_scale is None for c in others)
    assert all(c.buf is None or c.buf.dtype == torch.float16 for c in others)
    # e4m3-input launches: one per FP8 conv per chunk (chunks: 1, 4, 4 frames, then 4, 4 streamed)
    f8_in = [e for e in q if e["op"] == "vae_conv_fp8" and e["x"] == E4M3]
    assert len(f8_in) == 5 * 21
    assert sorted({(e["shape"][-1], e["n"]) for e in f8_in}) == [(96, 96), (96, 192), (192, 192), (192, 384),
                                                                 (384, 32), (384, 384)]
    # 16-bit convs writing an FP8 conv's input: conv_in every chunk, the 96-channel stride-2 conv every chunk, the 192 /
    # 384 stride-2 convs on the first chunk (no time_conv then), their time_convs once per output frame later
    f8_out = [e for e in q if e["op"] == "vae_conv_fp8" and e["x"] == torch.float16]
    assert all(e["norm"] == E4M3 for e in f8_out)
    got = sorted((e["shape"][-1], e["n"], e["taps"], e["sub2"]) for e in f8_out)
    later = 4                                              # chunks after the first
    want = sorted(5 * [(64, 96, (3, 3, 3), False), (96, 96, (1, 3, 3), True)]
                  + [(192, 192, (1, 3, 3), True), (384, 384, (1, 3, 3), True)]
                  + later * 2 * [(192, 192, (3, 1, 1), False)] + later * [(384, 384, (3, 1, 1), False)])
    assert got == want
    assert [e for e in q if e["op"] == "vae_rmsnorm_silu_fp8"] and not [e for e in q if e["op"] == "vae_rmsnorm_silu"
                                                                         and e["norm"] == E4M3]
    # every launch in the same order with the same geometry; the e4m3 buffers roll as 16-bit pairs of half the width
    assert len(base) == len(q)
    for b, e in zip(base, q):
        cb, ce = _canon(b), _canon(e)
        if e["op"] == "kv_roll" and cb != ce:
            assert cb[0] == "kv_roll" and ce[1][1] * 2 == cb[1][1] and ce[1][0] == cb[1][0]
        else:
            assert cb == ce, (b, e)


def test_stand_in_encoder_matches_the_fake_quant_oracle(gs, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu)
    o8 = VAEEncoderFp8Oracle(_params())
    m = encoder("fp8")
    cache, co = [None] * 55, {}
    with torch.no_grad():
        for tag, stream in (("cold9_64x96", False), ("stream8_64x96", True), ("stream4_64x96", True)):
            x = gs[f"{tag}/x"]
            mu, cache = m(x.half(), cache, stream=stream)
            ref, co = o8.forward(x.float(), co, stream=stream)
            r = rel_l2(mu, ref)
            print(f"{tag}: stand-in FP8 encoder vs fake-quant oracle rel_l2 {r:.3e}")
            assert r < 5.5e-2, (tag, r)        # the fp16 stand-ins are at 6.5e-2 of this oracle


# ---------------------------------------------------------------------------------------------
# buffer plan and frame tile
# ---------------------------------------------------------------------------------------------
def _meta_encoder(H, W, quant, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "fp8_input_scale", lambda gamma: 1.0)      # .item() has no value on the meta device
    m = vae.VAEEncoderWrapper().half()
    eng = vae.EncoderEngine(m.encoder, m.conv1, m.mean, m.std, quant=quant)
    eng._prepare(torch.float16, "meta", H, W)
    return eng


def _plan_gib(eng, tile):
    from realtime_video_b200.vae import _buf_bytes
    return _buf_bytes(eng._buf_plan(eng.H, eng.W, tile)) / GiB


@pytest.mark.parametrize("H,W,tile16,tile8", [(480, 832, 4, 4), (720, 1280, 1, 4)])
def test_buffer_plan_and_frame_tile(H, W, tile16, tile8, monkeypatch):
    """e4m3 conv-input buffers halve the FP8 convs' bytes: 832x480 keeps whole 4-frame buffers (3.12 -> 1.70 GiB);
    at 1280x720 the whole chunk fits the 4.5 GiB budget (7.20 -> 3.93 GiB), so the FP8 tier drops the one-frame tiles
    (4.03 GiB) of the fp16 tier."""
    e16, e8 = _meta_encoder(H, W, None, monkeypatch), _meta_encoder(H, W, "fp8", monkeypatch)
    assert (e16.frame_tile, e8.frame_tile) == (tile16, tile8)
    plan = e8._buf_plan(H, W, e8.frame_tile)
    assert sum(dt == E4M3 for _, _, dt in plan) == 21 and len(plan) == 22
    assert all((dt == E4M3) == (c.in_scale is not None) for c, _, dt in plan)
    for eng in (e16, e8):
        assert _plan_gib(eng, eng.frame_tile) <= 4.5
    print(f"{W}x{H}: fp16 tile {e16.frame_tile} ({_plan_gib(e16, e16.frame_tile):.2f} GiB, untiled "
          f"{_plan_gib(e16, 4):.2f}), fp8 tile {e8.frame_tile} ({_plan_gib(e8, e8.frame_tile):.2f} GiB, untiled "
          f"{_plan_gib(e8, 4):.2f})")
    assert _plan_gib(e8, 4) < 0.66 * _plan_gib(e16, 4)


# ---------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------
def test_cache_list_round_trips_with_e4m3_entries(gs, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu)
    x9, x4 = gs["cold9_64x96/x"].half(), gs["stream4_64x96/x"].half()
    m = encoder("fp8")
    with torch.no_grad():
        a, cache = m(x9, [None] * 55)
        used = [c for c in cache if c is not None]
        assert len(cache) == 55 and len(used) == int(gs["n_cache_slots"][0])
        assert sum(c.dtype == E4M3 for c in used) == 21
        snap = [c.clone() if c is not None else None for c in cache]
        b, _ = m(x4, cache, stream=True)
        # a second stream detaches the handed-out list first: it keeps the values it had
        a2, _ = m(x9, [None] * 55)
        assert torch.equal(a, a2)
        assert all(torch.equal(c.view(torch.uint8), s.view(torch.uint8)) for c, s in zip(cache, snap)
                   if c is not None and c.dtype == E4M3)
        # a foreign copy of the state (.to() copies) restores it
        b2, _ = m(x4, [c.to("cpu", copy=True) if c is not None else None for c in snap], stream=True)
        assert torch.equal(b, b2)


def test_interleaved_streams_have_value_semantics(gs, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu)
    fa, fb = gs["cold9_64x96/x"].half(), gs["cold9_64x96/x"].flip(-1).half()

    def alone(f):
        m = encoder("fp8")
        mu0, c = m(f[:, :, :5], [None] * 55)
        mu1, _ = m(f[:, :, 5:], c, stream=True)
        return mu0, mu1

    with torch.no_grad():
        wa, wb = alone(fa), alone(fb)
        m = encoder("fp8")
        a0, ca = m(fa[:, :, :5], [None] * 55)
        b0, cb = m(fb[:, :, :5], [None] * 55)
        a1, _ = m(fa[:, :, 5:], ca, stream=True)
        b1, _ = m(fb[:, :, 5:], cb, stream=True)
    assert all(torch.equal(u, v) for u, v in zip((a0, a1, b0, b1), (*wa, *wb)))


def test_switching_the_tier_rebuilds_and_starts_a_new_stream(gs, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu)
    x5, x4 = gs["cold9_64x96/x"][:, :, :5].half(), gs["stream4_64x96/x"].half()
    with torch.no_grad():
        m = encoder(None)
        _, cache16 = m(x5, [None] * 55)
        bufs16 = m._engine.head.buf
        m.quant = "fp8"
        got = m(x4[:, :, :1], cache16)[0]               # a cache of the fp16 tier is ignored: new stream
        assert m._engine.head.buf is not bufs16 and m._engine.head.buf.dtype == E4M3
        assert torch.equal(got, encoder("fp8")(x4[:, :, :1], [None] * 55)[0])
        _, cache8 = m(x5, [None] * 55)
        m.quant = None
        back = m(x4[:, :, :1], cache8)[0]
        assert m._engine.head.buf.dtype == torch.float16
        assert torch.equal(back, encoder(None)(x4[:, :, :1], [None] * 55)[0])


def test_env_switch_and_validation(gs, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu)
    monkeypatch.setenv("KR_VAE_ENC_FP8", "1")
    monkeypatch.delenv("KR_VAE_FP8", raising=False)
    assert vae.VAEEncoderWrapper().quant == "fp8" and vae.VAEDecoderWrapper().quant is None
    monkeypatch.setenv("KR_VAE_ENC_FP8", "0")
    monkeypatch.setenv("KR_VAE_FP8", "1")                 # the decoder's switch leaves the encoder alone
    assert vae.VAEEncoderWrapper().quant is None and vae.VAEDecoderWrapper().quant == "fp8"
    x = gs["cold9_64x96/x"][:, :, :1]
    with pytest.raises(ValueError, match="quant must be"):
        encoder("int8")(x.half(), [None] * 55)
    m = encoder("fp8").to(torch.bfloat16)
    m.quant = "fp8"
    with pytest.raises(ValueError, match="float16"):
        m(x.to(torch.bfloat16), [None] * 55)


def test_sub2_entry_point_rejects_bad_arguments():
    from realtime_video_b200 import _lib, ops
    lib = _lib.load()
    with pytest.raises(_lib.KreaB200Error):           # CPU tensors: no fallback
        ops.vae_conv_fp8(torch.zeros(1, 8, 8, 96, dtype=torch.float16), torch.zeros(96, 9 * 96, dtype=torch.float16),
                         None, n=96, cout=96, T=1, taps=(1, 3, 3), tile=(16, 8), sub2=True, norm_scale=1.0,
                         gamma=torch.ones(96, dtype=torch.float16),
                         out_norm=torch.zeros(1, 4, 4, 96, dtype=E4M3))
    f = lib.kr_vae_conv_fp8_sub2

    def call(in_fp8=0, taps=(1, 3, 3), out_pix=None, t_in=1):
        return f(in_fp8, 96, 96, 1, t_in, 1, 8, ctypes.c_float(1.0), 96, None, 96, 1, 8, 8, 16, 8, taps[0], taps[1],
                 taps[2], 1, 96, 96 * 16, 1, 96, 96 * 16, ctypes.c_float(1.0), 1, None, 0, 0, out_pix, None)

    for kw in (dict(in_fp8=1), dict(taps=(3, 3, 3), t_in=3), dict(taps=(1, 1, 1)), dict(out_pix=1)):
        assert call(**kw) == -1, kw
        assert b"sub2" in lib.kr_last_error()


# ---------------------------------------------------------------------------------------------
# SASS and resources
# ---------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_and_resources_of_the_encoder_kernels():
    from tests.test_sass_cpu import _ops
    from realtime_video_b200 import _lib
    _lib.load()
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            funcs[name] = []
        elif name and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            funcs[name].append(line.split("*/", 1)[1].strip())
    res = subprocess.run(["cuobjdump", "--dump-resource-usage", str(_lib.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    usage, fn = {}, None
    for line in res.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and "REG:" in line:
            usage[fn] = tuple(int(re.search(k + r":(\d+)", line).group(1)) for k in ("REG", "STACK", "LOCAL"))
            fn = None
    f8 = sorted(k for k in funcs if "enc_f8_" in k)
    f8n = sorted(k for k in funcs if "enc_igemm_conv_f8n_kernel" in k or "enc_halo_conv_f8n_kernel" in k)
    assert len(f8) == 2 and len(f8n) == 5, (f8, f8n)
    for k in f8 + f8n:
        ops = _ops(funcs[k])
        mma = "QGMMA" if k in f8 else "HGMMA"
        assert any(o.startswith(mma) for o in ops) and any(o.startswith("UTMALDG") for o in ops), k
        assert not any(o.startswith(("HMMA", "IMMA", "LDL", "STL")) for o in ops), k
        assert usage[k][1:] == (0, 0), (k, usage[k])
        print(f"{k}: {usage[k][0]} registers at launch (consumers raise theirs to 232 with setmaxnreg)")
