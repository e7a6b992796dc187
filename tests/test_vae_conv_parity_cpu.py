"""The float64 conv checker of ``tests/kernel_refs.py`` (``conv_interval`` / ``check_conv`` / ``guarded_frames``) and the
case table of ``tests/test_vae_conv_parity_gpu.py`` proven without a GPU:

- the GPU test's own per-case checks, run on an emulation of a correct kernel (fp32 accumulation per (tap, 64-channel
  chunk), then conv_epilogue_frag's rounding points), accept every epilogue form in both 16-bit types and reject each
  of nine plausible kernel bugs through the check named for it;
- the table covers every (cin, n) case of ``dispatch_conv`` and every conv launch the fp16 and bf16 decoder and encoder
  schedules issue, and the per-tap tiles ``_tile_for`` picks at the production stage sizes;
- ``kr_vae_conv3d`` / ``kr_vae_conv_fp8`` refuse the requests their epilogue would silently mishandle."""
import ctypes
import math
import re
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from oracle.vae_oracle import synthetic_vae_params
from tests import cpu_ops_emulation as C
from tests import kernel_refs as R
from tests import test_vae_conv_parity_gpu as G

ROOT = Path(__file__).resolve().parent.parent
DTYPES = [torch.bfloat16, torch.float16]


# ---------------------------------------------------------------------------------------------
# emulated kernel
# ---------------------------------------------------------------------------------------------
class EmuOps:
    """``ops.vae_conv`` as the kernels compute it, on the CPU; ``mutate`` names a deliberate bug."""

    def __init__(self, mutate=None):
        self.mutate = mutate

    def vae_conv(self, x, weight, bias, *, n, cout, T, taps, tile, out_raw=None, out_norm=None, gamma=None,
                 residual=None, out_pix=None, raw_frame_stride=None, sub2=False):
        mut = self.mutate
        kt, kh, kw = taps
        _, H, W, cin = x.shape
        w5 = weight.float().view(weight.shape[0], kt, kh, kw, cin)[:n]
        xp = F.pad(x.float().permute(0, 3, 1, 2), (kw // 2, kw // 2, kh // 2, kh // 2),
                   mode="circular" if mut == "border_wraps" else "constant").permute(0, 2, 3, 1)
        acc = torch.zeros(T, H, W, n)
        for a in range(kt):
            f = torch.arange(T) + a - (1 if mut == "kt_offset" else 0)
            for b in range(kh):
                for c in range(kw):
                    xs = xp[f.clamp_min(0), b:b + H, c:c + W]
                    for c0 in range(0, cin, 64):
                        if mut == "drop_remainder32" and c0 + 64 > cin:
                            continue
                        acc += xs[..., c0:c0 + 64] @ w5[:, a, b, c, c0:c0 + 64].t()
        v = acc + bias.float()[:n]
        rnd = lambda t: t.to(x.dtype).float()   # noqa: E731
        if sub2:
            s = slice(0 if mut == "sub2_even" else 1, None, 2)
            v = v[:, s, s][:, :H // 2, :W // 2]
        if out_pix is not None:
            out_pix.copy_(rnd(v)[..., :cout].clamp(-1, 1).permute(0, 3, 1, 2))
            if mut == "head_channel_ge_cout":       # channel cout of frame t lands on channel 0 of frame t + 1
                Ho, Wo = v.shape[1:3]
                torch.as_strided(out_pix, (T, Ho, Wo), (cout * Ho * Wo, Wo, 1),
                                 out_pix.storage_offset() + cout * Ho * Wo).copy_(rnd(v)[..., cout].clamp(-1, 1))
            return
        if residual is not None:
            y = rnd(residual[:T].float() + (v if mut == "residual_before_rounding" else rnd(v)))
        else:
            y = rnd(v)
        if out_raw is not None:
            fr = raw_frame_stride if raw_frame_stride is not None else out_raw.stride(0)
            shape = (T,) + tuple(y.shape[1:])
            st = (fr, out_raw.stride(1), out_raw.stride(2), 1)
            torch.as_strided(out_raw, shape, st, out_raw.storage_offset()).copy_(y)
            if mut == "pixel_past_w":               # the partial tile's pixel (h, W) of every row
                torch.as_strided(out_raw, (T, shape[1], 1, n), st,
                                 out_raw.storage_offset() + shape[2] * st[2]).copy_(y[:, :, -1:])
        if out_norm is not None:
            nrm = rnd(torch.sqrt((y * y).sum(-1, keepdim=True)))
            a = rnd(y * (1.0 / nrm.clamp_min(1e-30)))
            scale = math.sqrt(n if mut == "norm_sqrt_n" else cout)
            a = rnd(rnd(a * torch.tensor(scale, dtype=torch.float32)) * gamma.float()[:n])
            out_norm[:T].copy_(a / (1 + torch.exp(-a)))


def run_emulated(case, dtype, mutate=None):
    arm = G.Arm("halo", ops=EmuOps(mutate), device="cpu")
    arm.case(case, dtype, seed=7)
    return arm


# small shapes of every form: partial tiles, odd H / W for sub2, history frames, a longer input, CIN = 96 (64 + 32)
FORMS = {
    "raw, res, norm": G.Case(96, 32, G.T3, ["raw+res", "norm", "raw+res+norm", "res+norm"], T=2, H=5, W=9, extra=1),
    "1x1 raw, res": G.Case(192, 32, G.T111, ["raw+res"], T=2, H=7, W=5),
    "norm, n > cout": G.Case(96, 32, G.T3, ["raw+norm"], T=1, H=6, W=7, cout=24),
    "head": G.Case(96, 16, G.T3, ["pix"], T=2, H=5, W=9),
    "sub2": G.Case(96, 32, G.T133, ["raw+norm"], T=2, H=7, W=9, sub2=True),
    "interleave": G.Case(64, 32, G.T311, ["raw+norm"], T=2, H=4, W=6, interleave=True, extra=1),
}


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("name", list(FORMS))
def test_checker_accepts_a_correct_kernel(name, dtype):
    arm = run_emulated(FORMS[name], dtype)
    assert not arm.viol, arm.viol
    assert arm.excess == 0
    c = FORMS[name]
    assert arm.served == {(G.kernel_for("halo", c.cin, c.n, c.taps, c.n), c.cin, c.n, G.DTN[dtype], f)
                          for f in c.form_names()}


# (bug, case, the check that must reject it)
BUGS = [
    ("kt_offset", "raw, res, norm", "outside the accumulation interval"),
    ("border_wraps", "raw, res, norm", "outside the accumulation interval"),
    ("drop_remainder32", "raw, res, norm", "outside the accumulation interval"),
    ("residual_before_rounding", "raw, res, norm", "res chain"),
    ("norm_sqrt_n", "norm, n > cout", "norm: "),
    ("sub2_even", "sub2", "outside the accumulation interval"),
    ("head_channel_ge_cout", "head", "out_pix guard overwritten"),
    ("pixel_past_w", "raw, res, norm", "raw guard overwritten"),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mutate,name,check", BUGS)
def test_checker_rejects_each_kernel_bug(mutate, name, check, dtype):
    arm = run_emulated(FORMS[name], dtype, mutate)
    assert any(check in v for v in arm.viol), (mutate, arm.viol[:5])


@pytest.mark.parametrize("dtype", DTYPES)
def test_checker_rejects_one_element_one_ulp_outside(dtype):
    c = FORMS["raw, res, norm"]
    g = torch.Generator().manual_seed(3)
    kt, kh, kw = c.taps
    x = torch.randn(c.T + kt - 1, c.H, c.W, c.cin, generator=g).to(dtype)
    w = (torch.randn(c.n, kt * kh * kw * c.cin, generator=g) / 40).to(dtype)
    b = (torch.randn(32, generator=g) * 0.5).to(dtype)
    z, m, E = R.conv_interval(x, w.view(c.n, kt, kh, kw, c.cin), b, c.taps)
    _, y = R.guarded_frames(c.T, c.H, c.W, c.n, dtype, "cpu")
    EmuOps().vae_conv(x, w, b, n=c.n, cout=c.n, T=c.T, taps=c.taps, tile=(16, 8), out_raw=y)
    assert not R.check_conv("raw", y, z, m, E, dtype)[0]
    hi = R.r16(z[1, 2, 3, 4] + E[1, 2, 3, 4], dtype)
    y[1, 2, 3, 4] = R._bits_neighbour(hi.view(1), torch.tensor([True]), dtype)[0].to(dtype)
    viol, _ = R.check_conv("raw", y, z, m, E, dtype)
    assert any("outside the accumulation interval" in v for v in viol), viol


def test_conv_interval_against_torch_and_the_stand_in():
    """z is F.conv3d of the padded input (history frames in front), chunked over frames; sub2 is the stride-2 conv of
    ZeroPad2d((0,1,0,1)), which equals the odd positions of the stride-1 conv (the kernel's restatement) for 3x3
    taps; the fp32 stand-in of tests/cpu_ops_emulation.py lies inside the interval."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(6, 7, 9, 32, generator=g, dtype=torch.float64)
    w = torch.randn(16, 3, 3, 3, 32, generator=g, dtype=torch.float64) / 30
    b = torch.randn(32, generator=g, dtype=torch.float64)
    z, m, E = R.conv_interval(x, w, b, (3, 3, 3), T=3, frames_per_chunk=2)
    ref = F.conv3d(F.pad(x[:5].permute(3, 0, 1, 2)[None], (1, 1, 1, 1)), w.permute(0, 4, 1, 2, 3))[0]
    assert torch.allclose(z, ref.permute(1, 2, 3, 0) + b[:16], atol=1e-12)
    assert torch.equal(E, R.C_ACC_16 * m + R.F32_EPI * (z.abs() + b[:16].abs()))
    assert bool((m >= z.abs() - 1e-12).all())
    w2 = w[:, :1]
    zs, _, _ = R.conv_interval(x, w2, None, (1, 3, 3), sub2=True)
    full, _, _ = R.conv_interval(x, w2, None, (1, 3, 3))
    assert zs.shape == (6, 3, 4, 16) and torch.allclose(zs, full[:, 1::2, 1::2][:, :3, :4], atol=1e-12)
    w1 = w[:, :1, 1:2, 1:2]
    z1, _, _ = R.conv_interval(x, w1, None, (1, 1, 1))
    assert not torch.allclose(z1[:, 1::2, 1::2], z1[:, 0::2, 0::2][:, :3, :4])   # why 1x1 sub2 is refused
    xh = x.half()
    wk = w.half().reshape(16, -1)
    zh, mh, Eh = R.conv_interval(xh, wk.view(16, 3, 3, 3, 32), b.half(), (3, 3, 3))
    y = torch.empty(4, 7, 9, 16, dtype=torch.float16)
    C.vae_conv(xh, wk, b.half(), n=16, cout=16, T=4, taps=(3, 3, 3), tile=(16, 8), out_raw=y)
    assert not R.check_conv("raw", y, zh, mh, Eh, torch.float16)[0]


def test_guarded_frames():
    buf, v = R.guarded_frames(2, 3, 5, 32, torch.bfloat16, "cpu", fill=torch.ones(2, 3, 5, 32))
    assert v.stride() == (3 * 5 * 40, 5 * 40, 40, 1) and R.frames_intact(buf, 2, 32)
    buf[1, 0, 0, 32] = 0                                 # pitch guard of the first pixel
    assert not R.frames_intact(buf, 2, 32)
    buf, v = R.guarded_frames(4, 3, 5, 8, torch.float16, "cpu")
    v[0::2] = 1
    assert R.frames_intact(buf, 4, 8, untouched=[1, 3]) and not R.frames_intact(buf, 4, 8, untouched=[0])
    buf, v = R.guarded_frames(2, 3, 5, 3, torch.float32, "cpu")
    assert v.shape == (2, 3, 3, 5) and v.is_contiguous() and torch.isnan(buf).all()
    buf[3, 0, 0, 0] = 1.0                                # the extra NCHW frame
    assert not R.frames_intact(buf, 2, 3)


# ---------------------------------------------------------------------------------------------
# the table against dispatch_conv and the production schedules
# ---------------------------------------------------------------------------------------------
def test_table_covers_dispatch_conv():
    src = (ROOT / "realtime_video_b200" / "csrc" / "kr_vae.cu").read_text()
    body = src[src.index("static int dispatch_conv("):src.index("int vae_conv(int dtype")]
    halo = {(int(a), int(b)) for a, b in re.findall(r"^\s*KR_HALO_CASE\((\d+), (\d+)\)\s*$", body, re.M)}
    conv = {(int(a), int(b)) for a, b in re.findall(r"^\s*KR_CONV_CASE\((\d+), (\d+)\)\s*$", body, re.M)}
    assert halo == G.HALO_PAIRS
    assert conv == {(c.cin, c.n) for c in G.CASES}
    # every halo pair reaches the halo kernel in the default arm, and every pair the per-tap kernel in one of the arms
    assert {(k, cin, n) for k, cin, n, _, _ in G.want_set("halo") if k == "halo"} == {("halo",) + p for p in halo}
    assert {(cin, n) for k, cin, n, _, _ in G.want_set("pertap")} == conv
    assert all(k == "pertap" for k, *_ in G.want_set("pertap"))


def _form(kw):
    if kw.get("out_pix") is not None:
        f = "pix"
    else:
        f = "+".join(p for p, k in (("raw", "out_raw"), ("res", "residual"), ("norm", "out_norm"))
                     if kw.get(k) is not None)
        if kw.get("raw_frame_stride") is not None:
            f = "raw/interleave"
    return f + "/sub2" if kw.get("sub2") else f


def _record(monkeypatch, dtype):
    """Every vae_conv launch of a decoder call (3 latent frames on a new stream, then 2 more) and an encoder call (1 + 4
    frames, then 4 streamed) of the synthetic VAE on the fp32 stand-ins: {(cin, n, taps, kernel, form, tile)}."""
    import realtime_video_b200.vae as vae
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEEncoderWrapper
    log = set()

    class Ops:
        def __getattr__(self, name):
            fn = getattr(C, name)
            if name != "vae_conv":
                return fn

            def wrapped(x, weight, bias, **kw):
                k = G.kernel_for("halo", x.shape[-1], kw["n"], kw["taps"], weight.shape[0])
                log.add((x.shape[-1], kw["n"], kw["taps"], k, _form(kw), kw["tile"] if k == "pertap" else None))
                return fn(x, weight, bias, **kw)
            return wrapped

    monkeypatch.setattr(vae, "ops", Ops())
    g = torch.Generator().manual_seed(0)
    with torch.no_grad():
        dec = VAEDecoderWrapper()
        dec.load_state_dict(synthetic_vae_params(seed=0), strict=False)
        dec = dec.to(dtype).eval()
        _, cache = dec(torch.randn(1, 3, 16, 8, 12, generator=g).to(dtype), *([None] * 55))
        dec(torch.randn(1, 2, 16, 8, 12, generator=g).to(dtype), *cache)
        enc = VAEEncoderWrapper()
        enc.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
        enc = enc.to(dtype).eval()
        _, cache = enc(torch.randn(1, 3, 5, 64, 96, generator=g).to(dtype), [None] * 55)
        enc(torch.randn(1, 3, 4, 64, 96, generator=g).to(dtype), cache, stream=True)
    return log


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_production_launch_is_in_the_table(dtype, monkeypatch):
    launches = _record(monkeypatch, dtype)
    table = {(c.cin, c.n, c.taps, G.kernel_for("halo", c.cin, c.n, c.taps, c.n), f) for c in G.CASES
             for f in c.form_names()}
    prod = {key[:5] for key in launches}
    assert prod <= table, sorted(prod - table)
    # the decoder's head, its time_conv interleave and the encoder's stride-2 forms are among them
    assert {f for *_, f in prod} >= {"pix", "raw/interleave", "raw+norm/sub2", "raw/sub2", "norm", "raw+res+norm",
                                     "res+norm", "raw+res", "raw", "raw+norm"}


def test_production_tiles_are_in_the_table():
    """The per-tap tile of every production stage size: the 832x480 and 1280x720 latents (60x104, 90x160) times 1, 2,
    4, 8 (decoder), the same sizes as the encoder's inputs; at least one 384-channel and one CIN = 96 case runs it."""
    from realtime_video_b200.vae import _tile_for
    picked = {_tile_for(h * s, w * s) for h, w in ((60, 104), (90, 160)) for s in (1, 2, 4, 8)}
    for cin in (96, 384):
        run = {c.tile or _tile_for(c.H, c.W) for c in G.CASES
               if c.cin == cin and G.kernel_for("halo", c.cin, c.n, c.taps, c.n) == "pertap"}
        assert picked <= run and set(G.TILES) <= run, (cin, picked, run)


# ---------------------------------------------------------------------------------------------
# the entry points refuse what the epilogue would mishandle
# ---------------------------------------------------------------------------------------------
def _conv3d(lib, n=96, taps=(3, 3, 3), raw=True, norm=False, res=False, pix=False, sub2=0):
    kt, kh, kw = taps
    return lib.kr_vae_conv3d(1, 96, n, 1, kt, 1, n, None, 3 if n == 16 else n, 1, 8, 8, 16, 8, kt, kh, kw,
                             1 if raw else None, n, n * 64, 1 if norm else None, n, n * 64, 1 if norm else None,
                             1 if res else None, n, n * 64, 1 if pix else None, sub2, None)


CONV3D_BAD = {
    "out_pix with n != 16": dict(raw=False, pix=True),
    "out_raw with n = 16": dict(n=16, pix=True),
    "out_norm with n = 16": dict(n=16, raw=False, norm=True, pix=True),
    "residual with n = 16": dict(n=16, raw=False, res=True, pix=True),
    "n = 16 raw only": dict(n=16),
    "sub2 with 1x1 taps": dict(taps=(1, 1, 1), sub2=1),
    "sub2 with (3,3,3) taps": dict(taps=(3, 3, 3), sub2=1),
    "sub2 with (3,1,1) taps": dict(taps=(3, 1, 1), sub2=1),
    "sub2 with out_pix": dict(n=16, raw=False, taps=(1, 3, 3), pix=True, sub2=1),
}


@pytest.mark.parametrize("name", list(CONV3D_BAD))
def test_conv3d_rejects_mishandled_requests(name):
    from realtime_video_b200 import _lib
    lib = _lib.load()
    assert _conv3d(lib, **CONV3D_BAD[name]) == -1, name
    msg = lib.kr_last_error()
    assert b"kr_vae_conv3d" in msg and (b"n = 16" in msg or b"sub2" in msg), msg


def test_conv_fp8_applies_the_head_rules():
    from realtime_video_b200 import _lib
    lib = _lib.load()

    def call(n, raw=False, norm=True, res=False, pix=False):
        return lib.kr_vae_conv_fp8(0, 96, n, 1, 3, 1, 8, ctypes.c_float(1.0), n, None, 3 if n == 16 else n, 1, 8, 8,
                                   16, 8, 3, 3, 3, 1 if raw else None, n, n * 64, 1 if norm else None, n, n * 64,
                                   ctypes.c_float(1.0), 1, 1 if res else None, n, n * 64, 1 if pix else None, None)

    for kw in (dict(n=96, pix=True), dict(n=16, pix=True), dict(n=16, norm=True, pix=False, raw=False),
               dict(n=16, norm=True, res=True)):
        assert call(**kw) == -1, kw
        assert b"n = 16" in lib.kr_last_error(), (kw, lib.kr_last_error())
