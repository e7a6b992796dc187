"""The FP8 (e4m3) tier of the VAE decoder without a GPU: the static scale rule and the weight quantiser (product vs
oracle/vae_fp8_oracle.py), the host schedule on the fp32 stand-ins of tests/cpu_ops_emulation_vae_fp8.py (which convs
go to FP8, every other launch unchanged), feature-cache and tier-switch semantics, torch.compile, argument validation,
and the SASS / resource usage of the new kernels."""
import ctypes
import math
import re
import shutil
import subprocess

import pytest
import torch
import torch.nn.functional as F

from oracle import vae_fp8_oracle as O8
from oracle.vae_oracle import VAEDecoderOracle, synthetic_vae_params
from tests import cpu_ops_emulation_vae_fp8 as emu8
from tests.golden_io import load_npz, rel_l2

E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module")
def g():
    return load_npz("vae_small.npz")


def decoder(quant="fp8", single=False):
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEDecoderWrapperSingle
    m = VAEDecoderWrapperSingle() if single else VAEDecoderWrapper()
    m.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    m = m.half().eval()
    m.quant = quant
    return m


# ---------------------------------------------------------------------------------------------
# numerics: scale rule and weight quantiser
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [96, 192, 384])
def test_static_scale_never_saturates_and_a_one_hot_pixel_reaches_the_bound(C):
    from realtime_video_b200.vae import fp8_input_scale
    gen = torch.Generator().manual_seed(C)
    for trial in range(20):
        gamma = torch.randn(C, generator=gen) * (0.05 + 3 * torch.rand(1, generator=gen))
        s = fp8_input_scale(gamma)
        assert s == O8.input_scale(gamma)
        y = torch.randn(512, C, generator=gen) * torch.rand(512, 1, generator=gen) * 100
        y[0] = 0.0
        x = F.silu(F.normalize(y, dim=-1) * math.sqrt(C) * gamma)
        assert float((x * s).abs().max()) <= 448.0
        # a one-hot pixel on the channel of max|gamma| puts sqrt(C) max|gamma| in front of the SiLU
        c = int(gamma.abs().argmax())
        onehot = torch.zeros(1, C)
        onehot[0, c] = math.copysign(1.0, float(gamma[c]))
        pre = F.normalize(onehot, dim=-1) * math.sqrt(C) * gamma
        assert abs(float(pre.abs().max()) * s - 448.0) < 448.0 * 1e-6


def test_scale_of_a_tiny_gamma_covers_the_negative_silu_range():
    from realtime_video_b200.vae import fp8_input_scale
    gamma = torch.full((96,), 1e-4)
    s = fp8_input_scale(gamma)
    assert float(F.silu(torch.tensor(-1.2785)).abs()) * s <= 448.0


def test_weight_quantiser_round_trips():
    from realtime_video_b200.vae import fp8_quantize_weight
    gen = torch.Generator().manual_seed(1)
    w = torch.randn(48, 3 * 9 * 96, generator=gen) * torch.rand(48, 1, generator=gen)
    w[5] = 0.0                                               # a padding row
    w_q, scale = fp8_quantize_weight(w.half())
    o_q, o_scale = O8.quantize_weight(w.half())
    assert w_q.dtype == E4M3 and torch.equal(w_q.view(torch.uint8), o_q.view(torch.uint8))
    assert torch.equal(scale, o_scale) and scale[5] == 1.0 and not w_q[5].float().any()
    deq = w_q.float() * scale[:, None]
    amax = w.half().float().abs().amax(dim=1, keepdim=True)
    assert float(((deq - w.half().float()).abs() / amax.clamp_min(1e-30)).max()) <= 2.0 ** -4
    assert float(w_q.float().abs().amax(dim=1)[torch.arange(48) != 5].min()) == 448.0
    w_q2, scale2 = fp8_quantize_weight(deq)                  # quantising the dequantised weights is exact
    assert torch.equal(w_q2.view(torch.uint8), w_q.view(torch.uint8)) and torch.allclose(scale2, scale)


def test_fake_quant_oracle_is_close_to_the_fp32_oracle(g):
    p = {k: v.float() for k, v in synthetic_vae_params(seed=0).items()}
    z = g["s8x12/z0"].float()
    ref, _ = VAEDecoderOracle(p).forward(z, {})
    o8 = O8.VAEDecoderFp8Oracle(p)
    got, _ = o8.forward(z, {})
    assert len(o8.scales) == 2 * 14 + 1
    r = rel_l2(got, ref)
    assert 0 < r < 8e-2, r


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
                fn = getattr(emu8, name)
                if not name.startswith("vae_") and name != "kv_roll":
                    return fn

                def wrapped(*a, **kw):
                    x = a[0]
                    on = kw.get("out_norm") if name.startswith("vae_conv") else (a[2] if "rmsnorm" in name else None)
                    rec.log.append(dict(op=name, shape=tuple(x.shape), x=x.dtype, n=kw.get("n"), T=kw.get("T"),
                                        taps=kw.get("taps"), raw=kw.get("out_raw") is not None,
                                        res=kw.get("residual") is not None,
                                        norm=None if on is None else on.dtype, pix=kw.get("out_pix") is not None))
                    return fn(*a, **kw)
                return wrapped

        monkeypatch.setattr(vae, "ops", Ops())


def _canon(e):
    """The launch as the fp16 schedule issues it."""
    op = {"vae_conv_fp8": "vae_conv", "vae_rmsnorm_silu_fp8": "vae_rmsnorm_silu"}.get(e["op"], e["op"])
    return (op, e["shape"], e["n"], e["T"], e["taps"], e["raw"], e["res"], e["norm"] is not None, e["pix"])


def test_schedule_sends_exactly_the_normalised_input_convs_to_fp8(g, monkeypatch):
    rec = _Recorder(monkeypatch)
    z = g["s8x12/z0"].half()
    with torch.no_grad():
        decoder(None)(z, *([None] * 55))
        base, rec.log = rec.log, []
        m = decoder("fp8")
        m(z, *([None] * 55))
        q = rec.log
    eng = m.engine
    fp8_convs = [c for b in eng.blocks if b["kind"] == "res" for c in (b["c1"], b["c2"])] + [eng.head]
    assert len(fp8_convs) == 29 and all(c.weight.dtype == E4M3 and c.buf.dtype == E4M3 for c in fp8_convs)
    others = [eng.conv1] + [b["sc"] for b in eng.blocks if b["kind"] == "res" and b["sc"] is not None] \
        + [b[k] for b in eng.blocks if b["kind"] == "up" for k in ("conv", "tconv") if k in b]
    assert all(c.weight.dtype == torch.float16 and c.w_scale is None for c in others)
    assert all(c.buf is None or c.buf.dtype == torch.float16 for c in others)
    # e4m3-input launches: one per FP8 conv per latent chunk (3 latent frames on a new stream: chunks of 1 and 2)
    f8_in = [e for e in q if e["op"] == "vae_conv_fp8" and e["x"] == E4M3]
    assert len(f8_in) == 2 * 29
    assert sorted({(e["shape"][-1], e["n"]) for e in f8_in}) == [(96, 16), (96, 96), (192, 192), (192, 384),
                                                                 (384, 384)]
    # 16-bit convs that write an FP8 conv's input: conv1 and the three Resample convs
    f8_out = [e for e in q if e["op"] == "vae_conv_fp8" and e["x"] == torch.float16]
    assert sorted((e["shape"][-1], e["n"]) for e in f8_out) == sorted(2 * [(64, 384), (192, 96), (384, 192),
                                                                            (384, 192)])
    assert all(e["norm"] == E4M3 for e in f8_out)
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


def test_stand_in_decoder_matches_the_fake_quant_oracle(g, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu8)
    p = {k: v.float() for k, v in synthetic_vae_params(seed=0).items()}
    o8 = O8.VAEDecoderFp8Oracle(p)
    m = decoder("fp8")
    cache_o, cache = {}, [None] * 55
    with torch.no_grad():
        for call in range(3):
            z = g[f"s8x12/z{call}"].half()
            px, cache = m(z, *cache)
            ref, cache_o = o8.forward(z.float(), cache_o)
            r = rel_l2(px, ref)
            print(f"call {call}: rel_l2 vs fake-quant oracle {r:.3e}")
            assert r < 6e-2, f"call {call}: {r:.3e}"


# ---------------------------------------------------------------------------------------------
# streams
# ---------------------------------------------------------------------------------------------
def test_cache_list_slots_are_e4m3_views_with_value_semantics(g, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu8)
    m = decoder("fp8")
    z0, z1 = g["s8x12/z0"].half(), g["s8x12/z1"].half()
    with torch.no_grad():
        a, cache = m(z0, *([None] * 55))
        used = [c for c in cache if c is not None]
        assert len(used) == 32 and sum(c.dtype == E4M3 for c in used) == 29
        assert all(c.dtype in (E4M3, torch.float16) for c in used)
        snap = [c.clone() if c is not None else None for c in cache]
        b, _ = m(z1, *cache)
        # the handed-out list was a view of the buffers: a second stream detaches it first
        a2, cache2 = m(z0, *([None] * 55))
        assert torch.equal(a, a2)
        assert all(c is None or torch.equal(c.view(torch.uint8), s.view(torch.uint8)) for c, s in zip(cache, snap)
                   if c is not None and c.dtype == E4M3)
        b2, _ = m(z1, *[c.to("cpu", copy=True) if c is not None else None for c in snap])   # .to() copies restore
        assert torch.equal(b, b2)


def test_switching_the_tier_starts_a_new_stream(g, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu8)
    z0, z1 = g["s8x12/z0"].half(), g["s8x12/z1"].half()
    with torch.no_grad():
        m = decoder(None)
        _, cache16 = m(z0, *([None] * 55))
        m.quant = "fp8"
        fresh_from_16 = m(z1, *cache16)[0]          # a cache of the fp16 tier: ignored, new stream
        ref = decoder("fp8")(z1, *([None] * 55))[0]
        assert torch.equal(fresh_from_16, ref)
        _, cache8 = m(z0, *([None] * 55))
        m.quant = None
        back = m(z1, *cache8)[0]
        assert torch.equal(back, decoder(None)(z1, *([None] * 55))[0])


def test_single_frame_wrapper_runs_the_tier(g, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu8)
    m = decoder("fp8", single=True)
    h, w = 8, 12
    shapes = [(16, h, w)] + [(384, h, w)] * 11 + [(192, 2 * h, 2 * w)] + [(384, 2 * h, 2 * w)] * 6 \
        + [(192, 4 * h, 4 * w)] * 6 + [(96, 8 * h, 8 * w)] * 7
    cache = [torch.zeros(1, c, 2, hh, ww, dtype=torch.float16) for (c, hh, ww) in shapes]
    ref = decoder(None, single=True)
    cache_r = list(cache)
    with torch.no_grad():
        for i in range(2):
            px, cache = m(g[f"single8x12/z{i}"].half(), torch.tensor(i == 0), *cache)
            pr, cache_r = ref(g[f"single8x12/z{i}"].half(), torch.tensor(i == 0), *cache_r)
            assert px.shape == (1, 4, 3, 64, 96) and sum(c.dtype == E4M3 for c in cache) == 29
            assert rel_l2(px.float(), pr.float()) < 8e-2


def test_env_switch_and_validation(monkeypatch, g):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu8)
    monkeypatch.setenv("KR_VAE_FP8", "1")
    assert vae.VAEDecoderWrapper().quant == "fp8" and vae.VAEDecoderWrapperSingle().quant == "fp8"
    monkeypatch.setenv("KR_VAE_FP8", "0")
    assert vae.VAEDecoderWrapper().quant is None
    m = decoder("int8")
    with pytest.raises(ValueError, match="quant must be"):
        m(g["s8x12/z0"].half(), *([None] * 55))
    m = decoder("fp8").to(torch.bfloat16)
    m.quant = "fp8"
    with pytest.raises(ValueError, match="float16"):
        m(g["s8x12/z0"].to(torch.bfloat16), *([None] * 55))


def test_compiled_fullgraph_decoder_runs_the_tier(g, monkeypatch):
    import realtime_video_b200.vae as vae
    monkeypatch.setattr(vae, "ops", emu8)
    z0, z1 = g["s8x12/z0"].half(), g["s8x12/z1"].half()
    with torch.no_grad():
        dec = decoder("fp8")
        px0, _ = dec(z0, *([None] * 55))
        px0b, _ = dec(z1, *dec.engine.export_cache())
        dec2 = decoder("fp8")
        compiled = torch.compile(dec2, fullgraph=True)
        px1, cache = compiled(z0, *([None] * 55))
        px1b, cache = compiled(z1, *cache)
    assert torch.equal(px0, px1) and torch.equal(px0b, px1b)
    assert dec2.engine.head.buf.dtype == E4M3


def test_ops_and_c_abi_reject_bad_arguments():
    from realtime_video_b200 import _lib, ops
    lib = _lib.load()
    x = torch.zeros(3, 8, 8, 96, dtype=E4M3)
    w = torch.zeros(96, 27 * 96, dtype=E4M3)
    with pytest.raises(_lib.KreaB200Error):           # CPU tensors: no fallback
        ops.vae_conv_fp8(x, w, None, n=96, cout=96, T=1, taps=(3, 3, 3), tile=(16, 8), w_scale=torch.ones(96),
                         in_scale=1.0, out_raw=torch.zeros(1, 8, 8, 96, dtype=torch.float16))
    f = lib.kr_vae_conv_fp8

    def call(in_fp8=1, inp=1, wgt=1, w_scale=8, in_scale=1.0, out_raw=1, out_norm=None, nq=0.0, gamma=None,
             tile=(16, 8), taps=(3, 3, 3), t_in=3, T=1):
        return f(in_fp8, 96, 96, inp, t_in, wgt, w_scale, ctypes.c_float(in_scale), 96, None, 96, T, 8, 8, tile[0],
                 tile[1], taps[0], taps[1], taps[2], out_raw, 96, 96 * 64, out_norm, 96, 96 * 64, ctypes.c_float(nq),
                 gamma, None, 0, 0, None, None)

    cases = [dict(inp=None), dict(in_fp8=2), dict(out_raw=None), dict(w_scale=None), dict(w_scale=4),
             dict(in_scale=0.0), dict(in_scale=float("inf")), dict(out_norm=1, gamma=1, nq=0.0),
             dict(out_norm=1, gamma=None, nq=1.0), dict(in_fp8=0, w_scale=None), dict(tile=(16, 16)),
             dict(taps=(2, 3, 3)), dict(t_in=2)]
    for kw in cases:
        assert call(**kw) == -1, kw
        assert lib.kr_last_error()
    assert lib.kr_vae_rmsnorm_silu_fp8(None, 1, 1, 4, 96, ctypes.c_float(1.0), None) == -1
    assert lib.kr_vae_rmsnorm_silu_fp8(1, 1, 1, 4, 96, ctypes.c_float(-1.0), None) == -1


# ---------------------------------------------------------------------------------------------
# SASS and resources
# ---------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_and_resources_of_the_fp8_conv_kernels():
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
    f8 = sorted(k for k in funcs if "conv_f8_igemm_kernel" in k or "conv_f8_halo_kernel" in k)
    assert len(f8) == 5, f8
    for k in f8:
        ops = _ops(funcs[k])
        assert any(o.startswith("QGMMA") for o in ops) and any(o.startswith("UTMALDG") for o in ops), k
        assert not any(o.startswith(("HMMA", "IMMA", "LDL", "STL")) for o in ops), k
        assert usage[k][1:] == (0, 0), (k, usage[k])
        print(f"{k}: {usage[k][0]} registers at launch (consumers raise theirs to 232 with setmaxnreg)")
    # the 16-bit producers with an e4m3 out_norm and the e4m3 RMS_norm
    prod = [k for k in funcs if re.search(r"conv_(igemm|halo)_kernel.*Lb0ELb1E", k)]
    assert len(prod) == 3 and all(usage[k][1:] == (0, 0) for k in prod), prod
    assert any("rmsnorm_silu_kernelILb0ELb1E" in k for k in funcs)
