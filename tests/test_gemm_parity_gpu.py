"""Element-wise float64 parity of every 16-bit GEMM kernel (fixed widths 32..256 and runtime widths 96..224 of
kr_gemm.cu, the 2-CTA cluster kernel of kr_gemm2.cu, stream-K of kr_gemm_sk.cu), every epilogue, both 16-bit types,
M / N / K tails, strided operands, in-place and separate residuals, a gate boundary inside a 64-row half and the split
output; the VAE attention GEMMs at their production shapes; the promoted FP8 GEMMs; and the argument contract.

Each output is held by ``tests/kernel_refs.check_gemm``: the first rounding r16(acc + b) of every element lies in
[r16(z - E), r16(z + E)], z the float64 product, E = c_acc * (|a| |w|^T); when EPI_BIAS ran on the same kernel the
rest of the chain is restated exactly on its output (GELU: within the fp32 tanhf error).  Every output, ``out2`` and
residual sits inside a sentinel-filled buffer (pitch > N, rows past M) that must be unchanged after the launch.

Largest accumulation ratio |acc + b - z| / (|a| |w|^T) observed on an H100 SXM (80 GB HBM3, 132 SMs, 700 W limit):
the distance from z to the nearest rounding boundary of the 16-bit output, or |out / alpha - z| for EPI_F32.
  16-bit operands, four arms (K <= 5120): bf16 4.8e-7 (2^-21.0), fp16 5.9e-7 (2^-20.7), EPI_F32 8.6e-7 (2^-20.2)
  16-bit operands, VAE attention P V (fp16, K = 14400): 3.7e-6 (2^-18.0)            -> c_acc = 2^-16 (4.1x)
  e4m3 operands (gemm_fp8 / gemm_fp8_rowwise, promoted accumulation): 6.4e-5 (2^-13.9) -> c_acc = 2^-11 (7.7x)

The library reads its kernel switches once per process, so each arm runs ``python -m tests.test_gemm_parity_gpu ARM``
in a subprocess and prints one summary line."""
import json
import math
import os
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
E16 = [R.EPI_BIAS, R.EPI_BIAS_GELU, R.EPI_BIAS_GATE_RES, R.EPI_BIAS_RES, R.EPI_MUL]
RPG, ROW_OFF, ALPHA = 50, 37, 1.0 / math.sqrt(384)     # gate boundaries at rows 13, 63, 113, ...: inside the halves
FIXED, FLEX, CLUSTER, STREAMK = 1, 4, 2, 3              # kr_gemm_kernel_id


# ---- the planner's tile-width rules (kr_gemm.cu gemm_single / gemm_flex_bn), restated ------------------------------
def fixed_width(M, N, sms):
    bn = 256 if N % 256 == 0 else 128 if N % 128 == 0 else 64 if N % 64 == 0 else 32
    num_m = (M + 127) // 128
    if bn == 256 and num_m * (N // 256) < sms and N % 128 == 0:
        bn = 128
    if bn == 128 and num_m * (N // 128) < sms and N % 64 == 0:
        bn = 64
    return bn


def flex_width(M, N, K, sms):
    cost = lambda bn: max(4.0 * bn, 2.0 * (128 + bn))   # noqa: E731
    num_m = (M + 127) // 128
    bn0 = 256 if N % 256 == 0 else 128
    if bn0 == 256 and num_m * (N // 256) < sms:
        bn0 = 128
    best, best_cost = 0, (num_m * (N // bn0) + sms - 1) // sms * cost(bn0) * 0.94
    for bn in range(256, 95, -32):
        c = (num_m * ((N + bn - 1) // bn) + sms - 1) // sms * cost(bn)
        if c < best_cost:
            best, best_cost = bn, c
    return best


def tile_width(kid, M, N, K, sms):
    return {FIXED: lambda: fixed_width(M, N, sms), FLEX: lambda: flex_width(M, N, K, sms)}.get(kid, lambda: 256)()


def sk_contributors(M, N, K, sms):
    """Number of CTAs that share each output tile under kr_gemm_sk.cu's equal split of the (tile, k-block) range."""
    nt, nk = (M + 127) // 128 * (N // 256), (K + 63) // 64
    total = nt * nk
    grid = min(sms, total)
    q, r = total // grid, total % grid
    cta = lambda it: it // (q + 1) if it < r * (q + 1) else r + (it - r * (q + 1)) // q   # noqa: E731
    return {cta(t * nk + nk - 1) - cta(t * nk) + 1 for t in range(nt)}


# ---- arms: environment, shapes (M, N, K, kernel id of EPI_BIAS), epilogues, target kernels ---------------------------
FIXED_SHAPES = [(4680, 1280, 96, FIXED), (4680, 640, 200, FIXED), (4680, 320, 32, FIXED), (4680, 352, 5120, FIXED),
                (1, 1280, 200, FIXED), (7, 352, 96, FIXED), (127, 640, 32, FIXED), (128, 320, 200, FIXED),
                (129, 352, 5120, FIXED), (300, 1280, 96, FIXED), (4680, 256, 200, FIXED)]
FLEX_SHAPES = [(4680, 1024, 512, FLEX), (4680, 512, 520, FLEX), (4680, 1536, 5120, FLEX), (4680, 4096, 512, FLEX),
               (1170, 512, 512, FLEX), (1170, 2560, 512, FLEX), (1, 512, 512, FLEX)]
E_ALL = E16 + [R.EPI_F32]
ARMS = {   # want: every (kernel, width, epilogue) the arm must serve, in bf16 and fp16
    "default": dict(env={"KR_GEMM_EPI_WARPS": "1", "KR_GEMM2": "0", "KR_GEMM_SK": "0"}, sk=False,
                    shapes=FIXED_SHAPES + FLEX_SHAPES, epis=E_ALL,
                    want={(FIXED, w, e) for w in (32, 64, 128, 256) for e in E_ALL} |
                    {(FLEX, w, e) for w in (96, 128, 160, 192, 224) for e in E16}),
    "registers": dict(env={"KR_GEMM_EPI_WARPS": "0", "KR_GEMM_FLEX": "0", "KR_GEMM2": "0", "KR_GEMM_SK": "0"},
                      sk=False, shapes=FIXED_SHAPES + [(M, N, K, FIXED) for M, N, K, _ in FLEX_SHAPES[:3]],
                      epis=E_ALL, want={(FIXED, w, e) for w in (32, 64, 128, 256) for e in E_ALL}),
    "cluster": dict(env={"KR_GEMM_EPI_WARPS": "1", "KR_GEMM2": "2", "KR_GEMM_SK": "0"}, sk=False,
                    shapes=[(1, 512, 264, CLUSTER), (129, 256, 5120, CLUSTER), (300, 768, 256, CLUSTER),
                            (4680, 512, 264, CLUSTER)],
                    epis=E16, want={(CLUSTER, 256, e) for e in E16 if e != R.EPI_MUL}),   # EPI_MUL: another kernel
    "streamk": dict(env={"KR_GEMM_EPI_WARPS": "1", "KR_GEMM2": "1", "KR_GEMM_SK": "1"}, sk=True,
                    shapes=[(1, 256, 5120, STREAMK), (129, 512, 520, STREAMK), (300, 768, 5120, STREAMK),
                            (585, 5120, 5120, STREAMK), (4480, 1024, 512, STREAMK)],
                    epis=E16, want={(STREAMK, 256, e) for e in E16}),
}


def _operands(M, N, K, dt, seed, strided):
    """a [M, K], w [N, K] (views with row pitch K + 40 / K + 24 when ``strided``), bias, residual, gate."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K + 40 if strided else K, device="cuda", generator=g).to(dt)[:, :K]
    w = (torch.randn(N, K + 24 if strided else K, device="cuda", generator=g) / math.sqrt(K)).to(dt)[:, :K]
    b = (torch.randn(N, device="cuda", generator=g) * 0.5).to(dt)
    res = torch.randn(M, N, device="cuda", generator=g).to(dt)
    gate = (torch.randn((M + ROW_OFF) // RPG + 1, N, device="cuda", generator=g) * 0.5).to(dt)
    return a, w, b, res, gate


def _with_bias(z0, m, b, c_acc):
    z = z0 + b.double()
    return z, c_acc * m + R.F32_EPI * (z.abs() + b.double().abs())


class Arm:
    """Runs every case of one arm, collecting violations, coverage and statistics."""

    def __init__(self, name):
        from realtime_video_b200 import _lib, ops
        self.name, self.cfg, self.ops, self.lib = name, ARMS[name], ops, _lib.load()
        ops.stream_k = self.cfg["sk"]
        self.sms = torch.cuda.get_device_properties(0).multi_processor_count
        self.viol, self.covered, self.excess = [], set(), 0.0
        self.frac, self.ratio, self.contrib = {}, {}, set()
        self.n = 0

    def kid(self, epi, M, N, K):
        return self.lib.kr_gemm_kernel_id_ws(epi, M, N, K, 1 if self.cfg["sk"] else 0)

    def launch(self, epi, a, w, b, dt, *, residual=None, gate=None, in_place=False, split=0):
        """One ops.gemm into guarded buffers -> (output, list of guard buffers with their view shapes)."""
        M, N = a.shape[0], w.shape[0]
        odt = torch.float32 if epi == R.EPI_F32 else dt
        guards, kw = [], {}
        if residual is not None:
            rbuf, r = R.guarded(M, N, dt, "cuda", fill=residual)
            guards.append((rbuf, M, N))
            kw["residual"] = r
        if gate is not None:
            gbuf, gv = R.guarded(gate.shape[0], N, dt, "cuda", fill=gate)
            guards.append((gbuf, gate.shape[0], N))
            kw.update(gate=gv, rows_per_gate=RPG, row_offset=ROW_OFF)
        if in_place and residual is not None:
            out = kw["residual"]
        else:
            obuf, out = R.guarded(M, N - split, odt, "cuda")
            guards.append((obuf, M, N - split))
        if split:
            o2buf, out2 = R.guarded(M, split, dt, "cuda")
            guards.append((o2buf, M, split))
            kw.update(out2=out2, n_split=N - split)
        self.ops.gemm(a, w, b, epilogue=epi, out=out, alpha=ALPHA if epi == R.EPI_F32 else 1.0, **kw)
        got = torch.cat([out, out2], dim=1) if split else out.clone()
        return got, guards

    def record(self, tag, viol, stats, guards):
        self.viol += [f"{tag}: {v}" for v in viol]
        for buf, rows, cols in guards:
            if not R.guard_intact(buf, rows, cols):
                self.viol.append(f"{tag}: guard overwritten")
        self.excess = max(self.excess, stats["excess"])

    def shape(self, M, N, K, kid_want):
        sms = self.sms
        kid = self.kid(R.EPI_BIAS, M, N, K)
        if kid != kid_want:
            self.viol.append(f"{(M, N, K)}: EPI_BIAS served by kernel {kid}, expected {kid_want}")
            return
        if kid == STREAMK:
            self.contrib |= sk_contributors(M, N, K, sms)
        for dt in (BF, FP):
            self.n += 1
            strided = self.n % 2 == 1
            a, w, b, res, gate = _operands(M, N, K, dt, M * 7 + N * 3 + K + (dt == FP), strided)
            z0, m, _ = R.gemm_interval(a, w)
            for bias in (True, False):
                z, E = _with_bias(z0, m, b, R.C_ACC_16) if bias else (z0, R.C_ACC_16 * m + R.F32_EPI * z0.abs())
                bb = b if bias else None
                y16, guards = self.launch(R.EPI_BIAS, a, w, bb, dt)
                outs = {}
                gate_r = R.gate_rows(M, gate, RPG, ROW_OFF, "cuda")
                # without bias: EPI_BIAS, EPI_F32 and one of the chains, in turn
                no_bias = (R.EPI_BIAS, R.EPI_F32, E16[1 + self.n % 4])
                for epi in self.cfg["epis"]:
                    if not bias and epi not in no_bias:
                        continue
                    kid_e = self.kid(epi, M, N, K)
                    if epi == R.EPI_F32 and kid_e != FIXED:
                        self.viol.append(f"{(M, N, K)}: EPI_F32 served by kernel {kid_e}")
                        continue
                    in_place = (self.n + epi) % 2 == 0
                    got, guards = (y16, guards) if epi == R.EPI_BIAS else self.launch(
                        epi, a, w, bb, dt, residual=res if epi in (R.EPI_BIAS_GATE_RES, R.EPI_BIAS_RES, R.EPI_MUL)
                        else None, gate=gate if epi == R.EPI_BIAS_GATE_RES else None, in_place=in_place)
                    outs[epi] = got
                    tag = f"{(M, N, K)} {DTN[dt]} {R.EPI_NAMES[epi]} bias={bias} kernel {kid_e}"
                    viol, st = R.check_gemm(epi, got, z, m, E, dt, residual=res, gate_r=gate_r, alpha=ALPHA,
                                            y16=y16 if kid_e == kid and epi != R.EPI_F32 else None)
                    self.record(tag, viol, st, guards)
                    self.frac.setdefault(R.EPI_NAMES[epi], []).append(st["frac"])
                    if "ratio" in st:
                        key = DTN[dt] if epi != R.EPI_F32 else DTN[dt] + "/f32"
                        self.ratio[key] = max(self.ratio.get(key, 0.0), st["ratio"])
                    if kid_e in {k for k, _, _ in self.cfg["want"]}:
                        self.covered.add((kid_e, tile_width(kid_e, M, N, K, sms), DTN[dt], R.EPI_NAMES[epi]))
                # split output: columns >= n_split into a strided second destination, bit-identical to the
                # unsplit output of the same epilogue
                if bias and N > 256:
                    epi = (R.EPI_BIAS, R.EPI_BIAS_GELU, R.EPI_BIAS_RES)[self.n % 3]
                    ns = (N - 32) // 256 * 256
                    if epi == R.EPI_BIAS_RES:
                        got, guards = self.launch(epi, a, w, bb, dt, residual=res, split=N - ns)
                    else:
                        got, guards = self.launch(epi, a, w, bb, dt, split=N - ns)
                    self.record(f"{(M, N, K)} {DTN[dt]} split {R.EPI_NAMES[epi]}", [] if torch.equal(
                        got, outs[epi]) else ["split output differs from the unsplit one"], {"excess": 0.0}, guards)
            del z0, m

    def run(self):
        for M, N, K, kid in self.cfg["shapes"]:
            self.shape(M, N, K, kid)
        torch.cuda.synchronize()
        want = {(k, w, d, R.EPI_NAMES[e]) for k, w, e in self.cfg["want"] for d in ("bf16", "fp16")}
        if self.covered != want:
            self.viol.append(f"coverage: missing {sorted(want - self.covered)}, unexpected "
                             f"{sorted(self.covered - want)}")
        if self.cfg["sk"]:
            if not ({1, 2} <= self.contrib and max(self.contrib) >= 3):
                self.viol.append(f"stream-K contributors per tile {sorted(self.contrib)}: need 1, 2 and 3+")
            ws = next(iter(self.ops._sk_ws.values()))
            if int(ws[:65536].view(torch.int32).abs().sum()) != 0:
                self.viol.append("stream-K tile counters not reset")
        served = {}
        for k, w, _, _ in self.covered:
            served.setdefault(k, set()).add(w)
        frac = {e: max(v) for e, v in self.frac.items()}
        line = {"arm": self.name, "served": {k: sorted(v) for k, v in served.items()}, "worst_excess": self.excess,
                "max_nonidentical_frac": frac, "acc_ratio": self.ratio,
                "acc_ratio_log2": {k: (math.log2(v) if v > 0 else None) for k, v in self.ratio.items()},
                "contributors": sorted(self.contrib), "violations": len(self.viol)}
        print("ARM " + json.dumps(line))
        for v in self.viol[:20]:
            print("VIOLATION " + v)
        return not self.viol


def _run_arm(name):
    env = dict(os.environ, **ARMS[name]["env"])
    r = subprocess.run([sys.executable, "-m", "tests.test_gemm_parity_gpu", name], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith(("ARM ", "VIOLATION "))]
    print("\n".join(lines))
    assert r.returncode == 0, "\n".join(lines) + r.stdout[-2000:] + r.stderr[-4000:]


@pytest.mark.parametrize("arm", list(ARMS))
def test_gemm_parity_arm(arm):
    _run_arm(arm)


# ---- the VAE attention GEMMs at their production shapes (vae._vae_attention) ----------------------------------------
@pytest.mark.parametrize("L,s_width", [(96, 32), (6240, 32), (14400, 64)])
def test_vae_attention_gemms(L, s_width):
    """fp16, C = 384, L = H*W tokens of one frame (8x12, the 832x480 latent 60x104, the 1280x720 latent 90x160)."""
    from realtime_video_b200 import _lib, ops
    lib, C, sms = _lib.load(), 384, torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(L)
    xn = torch.randn(L, C, device="cuda", generator=g).half()
    wqkv = (torch.randn(3 * C, C, device="cuda", generator=g) / math.sqrt(C)).half()
    bqkv = (torch.randn(3 * C, device="cuda", generator=g) * 0.1).half()
    wproj = (torch.randn(C, C, device="cuda", generator=g) / math.sqrt(C)).half()
    bproj = (torch.randn(C, device="cuda", generator=g) * 0.1).half()
    xt = torch.randn(L, C, device="cuda", generator=g).half()
    bad = []

    def check(tag, epi, got, a, w, bias, guards, y16=None, residual=None):
        z, m, E = R.gemm_interval(a, w, bias)
        viol, st = R.check_gemm(epi, got, z, m, E, FP, residual=residual, alpha=ALPHA, y16=y16)
        bad.extend(f"L={L} {tag}: {v}" for v in viol)
        bad.extend(f"L={L} {tag}: guard overwritten" for buf, r, c in guards if not R.guard_intact(buf, r, c))
        print(f"L={L} {tag}: {st}")

    qbuf, qkv = R.guarded(L, 3 * C, FP, "cuda")
    ops.gemm(xn, wqkv, bqkv, out=qkv)
    check("qkv", R.EPI_BIAS, qkv, xn, wqkv, bqkv, [(qbuf, L, 3 * C)])
    q, k = qkv[:, :C], qkv[:, C:2 * C]                        # strided views: lda = ldw = 3C + 24
    assert q.stride(0) == k.stride(0) > 3 * C
    assert lib.kr_gemm_kernel_id(R.EPI_F32, L, L, C) == FIXED and fixed_width(L, L, sms) == s_width
    sbuf, s = R.guarded(L, L, torch.float32, "cuda")
    ops.gemm(q, k, None, epilogue=ops.EPI_F32, alpha=ALPHA, out=s)
    check("S = q k^T / sqrt(C)", R.EPI_F32, s, q, k, None, [(sbuf, L, L)])
    p = ops.softmax_rows(s, torch.empty(L, L, dtype=FP, device="cuda"))
    del sbuf, s
    assert lib.kr_gemm_kernel_id(R.EPI_BIAS, C, L, C) == FIXED and fixed_width(C, L, sms) == s_width
    vbuf, vt = R.guarded(C, L, FP, "cuda")
    ops.gemm(wqkv[2 * C:], xn, None, out=vt)
    check("V^T", R.EPI_BIAS, vt, wqkv[2 * C:], xn, None, [(vbuf, C, L)])
    obuf, o = R.guarded(L, C, FP, "cuda")
    ops.gemm(p, vt, bqkv[2 * C:], out=o)                     # K = L: 32 of the last 64-wide k-block zero-filled
    check("P V", R.EPI_BIAS, o, p, vt, bqkv[2 * C:], [(obuf, L, C)])
    ybuf, y16 = R.guarded(L, C, FP, "cuda")
    ops.gemm(o, wproj, bproj, out=y16)
    pbuf, out = R.guarded(L, C, FP, "cuda")
    rbuf, xr = R.guarded(L, C, FP, "cuda", fill=xt)
    ops.gemm(o, wproj, bproj, epilogue=ops.EPI_BIAS_RES, residual=xr, out=out)
    check("proj + x", R.EPI_BIAS_RES, out, o, wproj, bproj, [(pbuf, L, C), (rbuf, L, C)], y16=y16, residual=xt)
    assert not bad, bad[:10]


def test_vae_attention_end_to_end_per_row():
    """vae._vae_attention on one 60x104 fp16 frame against a float64 restatement of vae.py's attention block on the
    same input: relative error of every token row of the block's contribution (out - x)."""
    from realtime_video_b200 import vae
    C, H, W = 384, 60, 104
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(1, H, W, C, device="cuda", generator=g).half()
    blk = dict(g=(1 + 0.1 * torch.randn(C, device="cuda", generator=g)).half(),
               wqkv=(torch.randn(3 * C, C, device="cuda", generator=g) / math.sqrt(C)).half(),
               bqkv=(torch.randn(3 * C, device="cuda", generator=g) * 0.1).half(),
               wproj=(torch.randn(C, C, device="cuda", generator=g) / math.sqrt(C)).half(),
               bproj=(torch.randn(C, device="cuda", generator=g) * 0.1).half())
    got = vae._vae_attention(blk, x)[0].view(H * W, C).double()
    xd = x[0].view(H * W, C).double()
    xn = xd / xd.norm(dim=-1, keepdim=True) * math.sqrt(C) * blk["g"].double()
    qkv = xn @ blk["wqkv"].double().t() + blk["bqkv"].double()
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    o = torch.softmax(q @ k.t() / math.sqrt(C), dim=-1) @ v
    ref = xd + o @ blk["wproj"].double().t() + blk["bproj"].double()
    rel = (got - ref).norm(dim=-1) / (ref - xd).norm(dim=-1)
    print(f"VAE attention 60x104: per-row relative error max {float(rel.max()):.3e} median {float(rel.median()):.3e}")
    assert float(rel.max()) < 5e-3      # measured 1.8e-3 on an H100: fp16 roundings of qkv, P and o


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


# ---- the promoted FP8 GEMMs -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rowwise", [False, True])
def test_fp8_gemm_parity(rowwise):
    """gemm_fp8 / gemm_fp8_rowwise (fast_accum=False): e4m3 operands decode exactly, so z is exact; c_acc = C_ACC_E4M3.
    M tails, N at the 128-wide tile, K = 208 (a k tail), 5120."""
    from realtime_video_b200 import ops
    ratio, bad = 0.0, []
    for M, N, K in [(1, 128, 208), (7, 384, 5120), (129, 1280, 208), (300, 256, 5120), (4680, 1280, 5120)]:
        g = torch.Generator(device="cuda").manual_seed(M + N + K)
        aq = (torch.randn(M, K, device="cuda", generator=g) * 32).to(torch.float8_e4m3fn)
        wq = (torch.randn(N, K, device="cuda", generator=g) * 32).to(torch.float8_e4m3fn)
        b = (torch.randn(N, device="cuda", generator=g) * 0.5).bfloat16()
        res = torch.randn(M, N, device="cuda", generator=g).bfloat16()
        gate = (torch.randn((M + ROW_OFF) // RPG + 1, N, device="cuda", generator=g) * 0.5).bfloat16()
        if rowwise:
            sa = torch.rand(M, device="cuda", generator=g) * 2e-3 + 1e-4
            sw = (torch.rand(N, device="cuda", generator=g) * 2e-3 + 1e-4).contiguous()
            z, m, E = R.gemm_interval(aq.float(), wq.float(), b, row_scale=sa, col_scale=sw, c_acc=R.C_ACC_E4M3)
            run = lambda epi, **kw: ops.gemm_fp8_rowwise(ops.Fp8Rows(aq.view(torch.uint8), sa, BF),   # noqa: E731
                                                         wq.view(torch.uint8), sw, b, epilogue=epi, **kw)
        else:
            state = torch.tensor([0.0, 3e-3], device="cuda")
            sw = 7e-4
            z, m, E = R.gemm_interval(aq.float(), wq.float(), b,
                                      col_scale=_f32(3e-3) * _f32(sw), c_acc=R.C_ACC_E4M3)
            run = lambda epi, **kw: ops.gemm_fp8(aq.view(torch.uint8), wq.view(torch.uint8), state, sw, b,  # noqa: E731
                                                 epilogue=epi, **kw)
        obuf, y16 = R.guarded(M, N, BF, "cuda")
        run(R.EPI_BIAS, out=y16)
        gate_r = R.gate_rows(M, gate, RPG, ROW_OFF, "cuda")
        for epi in (R.EPI_BIAS, R.EPI_BIAS_GELU, R.EPI_BIAS_GATE_RES, R.EPI_BIAS_RES):
            if epi == R.EPI_BIAS:
                got, guards = y16, [(obuf, M, N)]
            else:
                ebuf, got = R.guarded(M, N, BF, "cuda")
                rbuf, r = R.guarded(M, N, BF, "cuda", fill=res)
                gbuf, gv = R.guarded(gate.shape[0], N, BF, "cuda", fill=gate)
                run(epi, out=got, residual=r, gate=gv, rows_per_gate=RPG, row_offset=ROW_OFF)
                guards = [(ebuf, M, N), (rbuf, M, N), (gbuf, gate.shape[0], N)]
            viol, st = R.check_gemm(epi, got, z, m, E, BF, residual=res, gate_r=gate_r,
                                    y16=None if epi == R.EPI_BIAS else y16)
            bad += [f"{(M, N, K)} {R.EPI_NAMES[epi]}: {v}" for v in viol]
            bad += [f"{(M, N, K)} {R.EPI_NAMES[epi]}: guard" for bf, rr, cc in guards if not R.guard_intact(bf, rr, cc)]
            ratio = max(ratio, st.get("ratio", 0.0))
    print(f"FP8 {'rowwise' if rowwise else 'per-tensor'}: largest accumulation ratio {ratio:.3e} "
          f"(2^{math.log2(ratio) if ratio else float('-inf'):.2f}), c_acc 2^{math.log2(R.C_ACC_E4M3):.0f}")
    assert not bad, bad[:10]


# ---- the argument contract ---------------------------------------------------------------------------------------------
def test_gemm_argument_contract_raises_without_launching():
    from realtime_video_b200 import _lib, ops
    E = _lib.KreaB200Error
    a = torch.randn(64, 64, device="cuda").bfloat16()
    w = torch.randn(64, 64, device="cuda").bfloat16()
    r = torch.randn(64, 64, device="cuda").bfloat16()
    wide = torch.randn(64, 68, device="cuda").bfloat16()
    gate = torch.randn(2, 64, device="cuda").bfloat16()
    cases = {
        "N % 32": dict(a=a, w=w[:48]),
        "K % 8": dict(a=torch.randn(64, 40, device="cuda").bfloat16()[:, :36],
                      w=torch.randn(64, 40, device="cuda").bfloat16()[:, :36]),
        "lda % 8": dict(a=wide[:, :32], w=w[:, :32].contiguous()),
        "ldw % 8": dict(a=a[:, :32].contiguous(), w=wide[:, :32]),
        "ldr % 8": dict(a=a, w=w, epilogue=ops.EPI_BIAS_RES, residual=wide[:, :64]),
        "missing residual": dict(a=a, w=w, epilogue=ops.EPI_BIAS_RES),
        "missing residual (mul)": dict(a=a, w=w, epilogue=ops.EPI_MUL),
        "missing gate": dict(a=a, w=w, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, rows_per_gate=32),
        "gate without rows_per_gate": dict(a=a, w=w, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, gate=gate),
        "out2 with EPI_F32": dict(a=a, w=w, epilogue=ops.EPI_F32, out2=torch.empty(64, 32, device="cuda").bfloat16(),
                                  n_split=256),
        "n_split % 256": dict(a=torch.randn(64, 64, device="cuda").bfloat16(),
                              w=torch.randn(512, 64, device="cuda").bfloat16(),
                              out2=torch.empty(64, 256, device="cuda").bfloat16(), n_split=256 + 32),
    }
    for name, kw in cases.items():
        a_, w_ = kw.pop("a"), kw.pop("w")
        odt = torch.float32 if kw.get("epilogue") == ops.EPI_F32 else torch.bfloat16
        buf, out = R.guarded(a_.shape[0], w_.shape[0] if "out2" not in kw else kw.get("n_split", 0), odt, "cuda")
        torch.cuda.synchronize()
        with pytest.raises(E):
            ops.gemm(a_, w_, None, out=out, **kw)
        torch.cuda.synchronize()
        assert R.guard_intact(buf, out.shape[0], out.shape[1]) and bool(
            (out.view(torch.int32 if odt == torch.float32 else torch.int16) ==
             (R.SENTINEL32 if odt == torch.float32 else R.SENTINEL16)).all()), f"{name}: the kernel ran"


if __name__ == "__main__":
    torch.cuda.set_device(0)
    sys.exit(0 if Arm(sys.argv[1]).run() else 1)
