"""Element-wise float64 parity of the 16-bit VAE convolutions (kr_vae.cu): the per-tap implicit-GEMM kernel
(conv_igemm_kernel) and the halo kernel (conv_halo_kernel), every (cin, n, taps) the decoder and the encoder launch,
both 16-bit types, every fused epilogue form the engines use, the stride-2 epilogue (sub2) and the up3d time_conv's
frame interleave.

Each output is held by ``tests/kernel_refs.check_conv``: r16(acc + b) of every element lies in [r16(z - E), r16(z + E)],
z the float64 causal conv (history frames in front on T, zero padding on H / W; for sub2 ZeroPad2d((0,1,0,1)) and the
stride-2 conv), E = C_ACC_16 * (|x| * |w|) + 2^-22 (|z| + |b|); the residual form equals r16(res + raw) of the raw-only
output of the same kernel exactly; the fused RMS_norm -> SiLU is within 1 ulp of the restatement on the kernel's own raw
values; the head's fp32 pixels are clamp(r16(acc + b), -1, 1).  Every output and residual sits inside a sentinel-filled
buffer (pixel pitch n + 8, a frame before and after, the other half of an interleave, an extra NCHW frame) that must be
unchanged, and a repeated launch is bit-identical.  Shapes include partial tiles in H and W, W below the tile width,
T = 1 and 3 with non-zero history, inputs longer than T + kt - 1, all five per-tap tile shapes, and one shape per kernel
with at least two tiles (work items) per SM.

Largest accumulation ratio |acc + b - z| / (|x| * |w|) observed on an H100 SXM (80 GB HBM3, 132 SMs, 700 W limit), the
same in both arms (K <= 27 * 384): bf16 5.6e-7 (2^-20.8), fp16 6.6e-7 (2^-20.5) -> c_acc = C_ACC_16 = 2^-16 (23x).

The library reads KR_CONV_HALO once per process, so each arm runs ``python -m tests.test_vae_conv_parity_gpu ARM`` in
a subprocess and prints one summary line: ``halo`` (the default dispatch) and ``pertap`` (KR_CONV_HALO=0, every conv on
the per-tap kernel).  The kernel that served each configuration is read from the profiler's kernel names."""
import json
import math
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from tests import kernel_refs as R

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
BF, FP = torch.bfloat16, torch.float16
DTN = {BF: "bf16", FP: "fp16"}

# dispatch_conv's rule, restated: the halo kernel serves 3x3-spatial taps with kt in {1, 3}, w_rows >= n and one of
# these (cin, n) pairs when KR_CONV_HALO is not 0; every other launch goes to the per-tap kernel
HALO_PAIRS = {(384, 192), (192, 192), (192, 96), (96, 96), (96, 192)}
TILES = [(4, 32), (8, 16), (16, 8), (32, 4), (64, 2)]     # (TW, TH) of the per-tap kernel
ARMS = {"halo": {}, "pertap": {"KR_CONV_HALO": "0"}}


def kernel_for(arm, cin, n, taps, w_rows):
    kt, kh, kw = taps
    halo = arm == "halo" and kh == 3 and kw == 3 and kt in (1, 3) and w_rows >= n and (cin, n) in HALO_PAIRS
    return "halo" if halo else "pertap"


class Case:
    """One (cin, n, taps) configuration at one shape.  Every case but the head runs the raw-only launch (the y16 of the
    chain checks) and then each form in ``forms``: '+'-joined outputs of one launch (raw, res, norm; pix for the head).
    ``interleave``: two row-halves of one [2n, K] weight into alternating frames (the up3d time_conv)."""

    def __init__(self, cin, n, taps, forms=(), T=1, H=13, W=19, extra=0, tile=None, sub2=False, interleave=False,
                 cout=None):
        self.cin, self.n, self.taps, self.forms, self.T, self.H, self.W = cin, n, taps, tuple(forms), T, H, W
        self.cout = cout or (3 if n == 16 else n)       # weight rows >= cout are zero, as _prep_conv pads them
        self.extra, self.tile, self.sub2, self.interleave = extra, tile, sub2, interleave

    def form_names(self):
        """The epilogue forms this case serves, as the schedule coverage of test_vae_conv_parity_cpu.py names them."""
        if self.n == 16:
            return ["pix"]
        names = ["raw"] + list(self.forms)
        if self.interleave:
            names.append("raw/interleave")
        return [f + "/sub2" if self.sub2 else f for f in names]

    def __repr__(self):
        return (f"({self.cin}->{self.n} taps {self.taps} T={self.T} {self.H}x{self.W} extra={self.extra} "
                f"tile={self.tile}{' sub2' if self.sub2 else ''}{' interleave' if self.interleave else ''})")


T3, T311, T111, T133 = (3, 3, 3), (3, 1, 1), (1, 1, 1), (1, 3, 3)
CASES = [
    # decoder: conv1, middle / stage ResidualBlocks (c1 norm only; c2 with residual, raw and / or the next norm)
    Case(64, 384, T3, ["raw+norm"], T=3, H=90, W=160),                       # >= 2 x SMs per-tap tiles
    Case(384, 384, T3, ["norm", "raw+res+norm", "raw+res", "res+norm"], T=3, H=10, W=14, extra=1),
    Case(192, 384, T3, ["norm"], T=1, H=9, W=17),
    Case(192, 384, T111, ["raw+res", "raw+res+norm"], T=3, H=20, W=28),
    Case(384, 384, T311, [], T=1, H=8, W=12, interleave=True),
    Case(384, 384, T311, ["raw+norm", "raw+res+norm"], T=3, H=12, W=20, interleave=True, extra=2),
    Case(384, 192, T133, ["raw+norm", "raw+res+norm"], T=2, H=16, W=16),
    Case(192, 192, T3, ["norm", "raw+res+norm", "raw+res"], T=2, H=12, W=20),
    Case(192, 96, T133, ["raw+norm", "raw+res+norm"], T=1, H=24, W=40),
    Case(96, 96, T3, ["norm", "raw+res+norm", "res+norm"], T=3, H=120, W=200),   # >= 2 x SMs halo items
    Case(96, 96, T3, ["raw+res+norm", "raw+res"], T=1, H=37, W=6, extra=1),            # W below every tile width
    Case(96, 16, T3, ["pix"], T=3, H=20, W=28, extra=1),
    Case(96, 16, T3, ["pix"], T=1, H=9, W=70),
    # encoder: conv_in, shortcuts, the stride-2 convs (odd and even H / W), the time_convs, the head
    Case(64, 96, T3, ["raw+norm"], T=3, H=24, W=40),
    Case(96, 192, T111, ["raw+res"], T=2, H=20, W=28),
    Case(96, 192, T3, ["norm", "raw+res+norm"], T=1, H=21, W=29),
    Case(96, 96, T133, ["raw+norm"], T=2, H=33, W=45, sub2=True),
    Case(96, 96, T133, ["raw+norm"], T=1, H=16, W=24, sub2=True),
    Case(192, 192, T133, ["raw+norm"], T=2, H=23, W=17, sub2=True),
    Case(384, 384, T133, ["raw+norm"], T=1, H=15, W=21, sub2=True),
    Case(384, 384, T133, [], T=2, H=16, W=12, sub2=True),
    Case(192, 192, T311, ["raw+norm"], T=1, H=11, W=19, extra=1),
    Case(384, 384, T311, ["raw+norm"], T=1, H=7, W=13),
    Case(384, 32, T3, [], T=3, H=7, W=13, extra=2),
    Case(384, 384, T3, ["raw+res+norm"], T=1, H=7, W=13),
    Case(192, 384, T3, ["norm"], T=2, H=15, W=26),
] + [
    # every per-tap tile shape on a CIN = 96 (kHas32) and a 384-channel configuration
    Case(96, 192, T111, ["raw+res"], T=2, H=11, W=70, tile=t) for t in TILES
] + [
    Case(384, 384, T3, ["raw+res+norm"], T=1, H=13, W=19, tile=t) for t in TILES
]


def want_set(arm):
    out = set()
    for c in CASES:
        k = kernel_for(arm, c.cin, c.n, c.taps, c.n)
        for d in ("bf16", "fp16"):
            out |= {(k, c.cin, c.n, d, f) for f in c.form_names()}
    return out


def work_items(kernel, H, W, T, tile):
    """Tiles (per-tap) or 16 x 16 work items (halo) of one launch: the persistent grid is min(SMs, this)."""
    if kernel == "halo":
        return T * ((H + 15) // 16) * ((W + 15) // 16)
    tw, th = tile
    return T * ((H + th - 1) // th) * ((W + tw - 1) // tw)


_KNAME = re.compile(r"(conv_halo_kernel|conv_igemm_kernel)<(\d+), (\d+), ([^,>]+), ([^,>]+)>")


class Arm:
    """Runs every case of one arm, collecting violations, the served set and statistics.  ``ops`` / ``device`` let
    tests/test_vae_conv_parity_cpu.py run the same checks on an emulated kernel (the kernel is then the restated one)."""

    def __init__(self, name, ops=None, device="cuda"):
        from realtime_video_b200.vae import _tile_for
        if ops is None:
            from realtime_video_b200 import ops
        self.name, self.ops, self.tile_for, self.dev = name, ops, _tile_for, device
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count if device == "cuda" else 132
        self.viol, self.served, self.ratio, self.norm_frac, self.excess = [], set(), {}, 0.0, 0.0
        self.big, self.norm_ulps = set(), 0.0

    def fail(self, tag, msg):
        self.viol.append(f"{tag}: {msg}")

    def launch(self, x, w, b, c, tile, T, **outs):
        self.ops.vae_conv(x, w, b, n=c.n, cout=c.cout, T=T, taps=c.taps, tile=tile, sub2=c.sub2, **outs)

    def observed_kernel(self, fn, c, dt, tag):
        """Run ``fn`` (one launch) under the profiler -> 'halo' / 'pertap' from the kernel's name, whose template
        arguments must be this configuration's (cin, n, dtype)."""
        if self.dev != "cuda":
            fn()
            return kernel_for(self.name, c.cin, c.n, c.taps, c.n)
        from torch.profiler import ProfilerActivity, profile
        fn()                      # load the kernel first: a launch that lazily loads it can miss the profiler's buffer
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [m for m in (_KNAME.search(e.name) for e in prof.events()) if m]
        if len(names) != 1:
            self.fail(tag, f"expected one conv kernel, profiler saw {[e.name for e in prof.events()][:6]}")
            return None
        kind, cin, n, bf, f8 = names[0].groups()
        if (int(cin), int(n), bf in ("true", "1", "(bool)1"), f8 in ("true", "1", "(bool)1")) != (c.cin, c.n, dt == BF,
                                                                                                 False):
            self.fail(tag, f"served by {names[0].group(0)}")
        return "halo" if kind == "conv_halo_kernel" else "pertap"

    def record(self, tag, viol, stats, dt):
        self.viol += [f"{tag}: {v}" for v in viol]
        self.excess = max(self.excess, stats.get("excess", 0.0))
        if "ratio" in stats:
            self.ratio[DTN[dt]] = max(self.ratio.get(DTN[dt], 0.0), stats["ratio"])

    def case(self, c, dt, seed):
        kt, kh, kw = c.taps
        T, H, W, n, cin = c.T, c.H, c.W, c.n, c.cin
        cout, dev = c.cout, self.dev
        Ho, Wo = (H // 2, W // 2) if c.sub2 else (H, W)
        tile = c.tile or self.tile_for(H, W)
        tag = f"{c} {DTN[dt]}"
        g = torch.Generator(device=dev).manual_seed(seed)
        K = kt * kh * kw * cin
        x = torch.randn(T + kt - 1 + c.extra, H, W, cin, device=dev, generator=g).to(dt)
        rows = 2 * n if c.interleave else n
        w = torch.randn(rows, K, device=dev, generator=g) / math.sqrt(K)
        b = torch.zeros(max(rows, 32), device=dev)
        b[:rows] = torch.randn(rows, device=dev, generator=g) * 0.5
        w[cout:n], b[cout:n] = 0, 0                   # _prep_conv's zero padding rows (the head's n = 16 > 3)
        w, b = w.to(dt), b.to(dt)
        res = torch.randn(T, Ho, Wo, n, device=dev, generator=g).to(dt)
        gamma = (1 + 0.3 * torch.randn(n, device=dev, generator=g)).to(dt)
        w5 = lambda half: w[half * n:(half + 1) * n].view(n, kt, kh, kw, cin)      # noqa: E731
        z, m, E = R.conv_interval(x, w5(0), b, c.taps, sub2=c.sub2, T=T)
        kernel = None

        if n == 16:
            pbuf, pix = R.guarded_frames(T, H, W, cout, torch.float32, dev)
            kernel = self.observed_kernel(lambda: self.launch(x, w, b, c, tile, T, out_pix=pix), c, dt, tag)
            got = pix.permute(0, 2, 3, 1)
            viol, st = R.check_conv("head", got, z, m, E, dt)
            self.record(tag + " pix", viol, st, dt)
            if not R.frames_intact(pbuf, T, cout):
                self.fail(tag, "out_pix guard overwritten")
            pbuf2, pix2 = R.guarded_frames(T, H, W, cout, torch.float32, dev)
            self.launch(x, w, b, c, tile, T, out_pix=pix2)
            if not torch.equal(pbuf.view(torch.int32), pbuf2.view(torch.int32)):
                self.fail(tag, "a repeated launch is not bit-identical")
        else:
            ybuf, y16 = R.guarded_frames(T, Ho, Wo, n, dt, dev)
            kernel = self.observed_kernel(lambda: self.launch(x, w, b, c, tile, T, out_raw=y16), c, dt, tag)
            viol, st = R.check_conv("raw", y16, z, m, E, dt)
            self.record(tag + " raw", viol, st, dt)
            if not R.frames_intact(ybuf, T, n):
                self.fail(tag, "raw guard overwritten")
            ybuf2, y2 = R.guarded_frames(T, Ho, Wo, n, dt, dev)
            self.launch(x, w, b, c, tile, T, out_raw=y2)
            if not torch.equal(ybuf.view(torch.int16), ybuf2.view(torch.int16)):
                self.fail(tag, "a repeated launch is not bit-identical")
            for form in c.forms:
                parts = form.split("+")
                outs, bufs = {}, []
                if "res" in parts:
                    rbuf, rv = R.guarded_frames(T, Ho, Wo, n, dt, dev, fill=res)
                    outs["residual"] = rv
                    bufs.append((rbuf, "residual"))
                if "raw" in parts:
                    obuf, outs["out_raw"] = R.guarded_frames(T, Ho, Wo, n, dt, dev)
                    bufs.append((obuf, "out_raw"))
                if "norm" in parts:
                    nbuf, outs["out_norm"] = R.guarded_frames(T, Ho, Wo, n, dt, dev)
                    bufs.append((nbuf, "out_norm"))
                    outs["gamma"] = gamma
                self.launch(x, w, b, c, tile, T, **outs)
                raw = y16
                if "res" in parts:
                    raw = R.r16(res.double() + y16.double(), dt)
                    if not torch.equal(outs["residual"], res):
                        self.fail(tag, f"{form}: the residual was written")
                if "raw" in parts:
                    f = "res" if "res" in parts else "raw"
                    viol, st = R.check_conv(f, outs["out_raw"], z, m, E, dt, y16=y16, residual=res)
                    self.record(f"{tag} {form}", viol, st, dt)
                    if f == "raw" and not torch.equal(outs["out_raw"], y16):
                        self.fail(tag, f"{form}: raw output differs from the raw-only launch")
                if "norm" in parts:
                    viol, st = R.check_conv("norm", outs["out_norm"], z, m, E, dt, y16=raw, gamma=gamma, cout=cout)
                    self.record(f"{tag} {form}", viol, st, dt)
                    self.norm_frac = max(self.norm_frac, st["frac"])
                    self.norm_ulps = max(self.norm_ulps, st["worst_ulps"])
                for buf, what in bufs:
                    if not R.frames_intact(buf, T, n):
                        self.fail(tag, f"{form}: {what} guard overwritten")
            if c.interleave:
                # the up3d time_conv: half h of the weight rows (bias offset by h * n) into frames h, h + 2, ...
                ibuf, iv = R.guarded_frames(2 * T, Ho, Wo, n, dt, dev)
                fr = 2 * iv.stride(0)
                self.ops.vae_conv(x, w[:n], b, n=n, cout=n, T=T, taps=c.taps, tile=tile, out_raw=iv,
                                  raw_frame_stride=fr)
                if not R.frames_intact(ibuf, 2 * T, n, untouched=range(1, 2 * T, 2)):
                    self.fail(tag, "interleave: half 0 wrote outside its frames")
                self.ops.vae_conv(x, w[n:], b[n:], n=n, cout=n, T=T, taps=c.taps, tile=tile, out_raw=iv[1:],
                                  raw_frame_stride=fr)
                if not R.frames_intact(ibuf, 2 * T, n):
                    self.fail(tag, "interleave: guard overwritten")
                if not torch.equal(iv[0::2], y16):
                    self.fail(tag, "interleave: half 0 differs from the raw-only launch")
                z1, m1, E1 = R.conv_interval(x, w5(1), b[n:], c.taps, T=T)
                viol, st = R.check_conv("raw", iv[1::2], z1, m1, E1, dt)
                self.record(tag + " interleave half 1", viol, st, dt)
        if kernel is not None:
            self.served |= {(kernel, cin, n, DTN[dt], f) for f in c.form_names()}
            items = work_items(kernel, H, W, T, tile)
            if items >= 2 * self.sms:
                self.big.add(kernel)

    def run(self):
        for i, c in enumerate(CASES):
            for dt in (BF, FP):
                self.case(c, dt, seed=1000 * i + (dt == FP))
            torch.cuda.empty_cache()
        torch.cuda.synchronize()
        want = want_set(self.name)
        if self.served != want:
            self.fail("coverage", f"missing {sorted(want - self.served)}, unexpected {sorted(self.served - want)}")
        kernels = {k for k, *_ in want}
        if self.big != kernels:
            self.fail("coverage", f"no shape with >= 2 x {self.sms} SMs work items on {sorted(kernels - self.big)}")
        try:
            card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                  capture_output=True, text=True, timeout=60).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            card = torch.cuda.get_device_name(0)
        served = {}
        for k, cin, n, _, _ in self.served:
            served.setdefault(k, set()).add((cin, n))
        line = {"arm": self.name, "card": card, "sms": self.sms,
                "served": {k: sorted(v) for k, v in served.items()}, "served_entries": len(self.served),
                "acc_ratio": self.ratio,
                "acc_ratio_log2": {k: (math.log2(v) if v > 0 else None) for k, v in self.ratio.items()},
                "margin_over_c_acc": {k: (R.C_ACC_16 / v if v > 0 else None) for k, v in self.ratio.items()},
                "max_norm_nonidentical_frac": self.norm_frac, "max_norm_ulps": self.norm_ulps,
                "worst_excess": self.excess,
                "violations": len(self.viol)}
        print("ARM " + json.dumps(line))
        for v in self.viol[:30]:
            print("VIOLATION " + v)
        return not self.viol


def _run_arm(name):
    env = dict(os.environ, **ARMS[name])
    if name == "halo":
        env.pop("KR_CONV_HALO", None)
    r = subprocess.run([sys.executable, "-m", "tests.test_vae_conv_parity_gpu", name], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1500)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith(("ARM ", "VIOLATION "))]
    print("\n".join(lines))
    assert r.returncode == 0, "\n".join(lines) + r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("arm", list(ARMS))
def test_vae_conv_parity_arm(arm):
    _run_arm(arm)


if __name__ == "__main__":
    torch.cuda.set_device(0)
    sys.exit(0 if Arm(sys.argv[1]).run() else 1)
