"""GPU bring-up checks for the raw kernels (run on a GPU box).

    python tools/bringup.py gemm|attn|elem|perf

Each group compares a kernel with a plain torch fp32 computation on the same inputs and prints
one line per case.  Not a test-suite replacement (tests/ holds the parity tests); this is the
fast first contact with hardware, written so a hang in one group cannot block the others
(run every group under its own `timeout`).
"""
import math
import sys
import time

import torch

sys.path.insert(0, ".")
from realtime_video_b200 import ops  # noqa: E402

dev = "cuda"


def rel(a, b):
    a = a.float(); b = b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item(), (a - b).abs().max().item(), b.abs().max().item()


def report(name, got, ref, tol):
    r, mx, mref = rel(got, ref)
    ok = r < tol and math.isfinite(r)
    print(f"{'OK ' if ok else 'BAD'} {name}: rel_l2={r:.3e} max_abs={mx:.3e} max_ref={mref:.3e}", flush=True)
    return ok


def t_gemm():
    torch.manual_seed(0)
    ok = True
    shapes = [(128, 256, 64), (128, 256, 128), (200, 512, 256), (4680, 5120, 5120), (77, 64, 128),
              (3, 5120, 256), (333, 1536, 1536), (512, 5120, 4096), (130, 96, 192), (4680, 64, 5120)]
    for dt in (torch.bfloat16, torch.float16):
        for (M, N, K) in shapes:
            a = torch.randn(M, K, device=dev, dtype=dt)
            w = torch.randn(N, K, device=dev, dtype=dt) / math.sqrt(K)
            b = torch.randn(N, device=dev, dtype=dt)
            ref = a.float() @ w.float().t() + b.float()
            got = ops.gemm(a, w, b)
            torch.cuda.synchronize()
            ok &= report(f"gemm bias {dt} {M}x{N}x{K}", got, ref, 6e-3)
    M, N, K, F = 720, 1536, 1536, 3
    a = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
    w = torch.randn(N, K, device=dev, dtype=torch.bfloat16) / math.sqrt(K)
    b = torch.randn(N, device=dev, dtype=torch.bfloat16)
    res = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
    gate = torch.randn(F, 6, N, device=dev, dtype=torch.bfloat16)
    y = a.float() @ w.float().t() + b.float()
    got = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GELU)
    ok &= report("gemm gelu", got, torch.nn.functional.gelu(y, approximate="tanh"), 8e-3)
    got = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_RES, residual=res)
    ok &= report("gemm res", got, res.float() + y, 8e-3)
    g = gate[:, 2]
    got = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=res, gate=g, rows_per_gate=M // F)
    gfull = g.float().repeat_interleave(M // F, dim=0)
    ok &= report("gemm gate res", got, res.float() + y * gfull, 8e-3)
    got = ops.gemm(a, w, None, epilogue=ops.EPI_F32, alpha=0.5)
    ok &= report("gemm f32", got, (a.float() @ w.float().t()) * 0.5, 1e-4)
    # in-place residual stream update (out aliases residual)
    x = res.clone()
    ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_RES, residual=x, out=x)
    ok &= report("gemm res inplace", x, res.float() + y, 8e-3)
    print("GEMM", "PASS" if ok else "FAIL", flush=True)


def attn_ref(q, k, v, heads, block_len=0, window=0):
    Lq, Lkv = q.shape[0], k.shape[0]
    qf = q.float().view(Lq, heads, 128).transpose(0, 1)
    kf = k.float().view(Lkv, heads, 128).transpose(0, 1)
    vf = v.float().view(Lkv, heads, 128).transpose(0, 1)
    s = qf @ kf.transpose(1, 2) / math.sqrt(128)
    if block_len > 0:
        qi = torch.arange(Lq, device=q.device)[:, None]
        ki = torch.arange(Lkv, device=q.device)[None, :]
        ends = (qi // block_len + 1) * block_len
        m = ki < ends
        if window > 0:
            m &= ki >= ends - window
        s = s.masked_fill(~m, float("-inf"))
    p = torch.softmax(s, dim=-1)
    return (p @ vf).transpose(0, 1).reshape(Lq, heads * 128)


def t_attn():
    torch.manual_seed(1)
    ok = True
    cases = [(256, 256, 1, 0, 0), (128, 128, 2, 0, 0), (300, 500, 2, 0, 0), (720, 1440, 3, 0, 0),
             (1000, 2000, 4, 0, 0), (720, 720, 2, 240, 0), (1200, 1200, 2, 480, 0),
             (1200, 1200, 2, 240, 480), (512, 512, 1, 0, 0), (333, 77, 2, 0, 0)]
    for (Lq, Lkv, H, bl, win) in cases:
        q = torch.randn(Lq, H * 128, device=dev, dtype=torch.bfloat16)
        k = torch.randn(Lkv, H * 128, device=dev, dtype=torch.bfloat16)
        v = torch.randn(Lkv, H * 128, device=dev, dtype=torch.bfloat16)
        got = ops.attention(q, k, v, heads=H, block_len=bl, window=win)
        torch.cuda.synchronize()
        ok &= report(f"attn Lq={Lq} Lkv={Lkv} H={H} bl={bl} win={win}", got, attn_ref(q, k, v, H, bl, win), 1e-2)
    # peaked distribution (exercises the lazy rescale path)
    q = torch.randn(512, 128, device=dev, dtype=torch.bfloat16) * 6
    k = torch.randn(1024, 128, device=dev, dtype=torch.bfloat16) * 6
    v = torch.randn(1024, 128, device=dev, dtype=torch.bfloat16)
    got = ops.attention(q, k, v, heads=1)
    ok &= report("attn peaked", got, attn_ref(q, k, v, 1), 2e-2)
    # strided K/V view (cache prefix)
    cache_k = torch.randn(2000, 2 * 128, device=dev, dtype=torch.bfloat16)
    cache_v = torch.randn(2000, 2 * 128, device=dev, dtype=torch.bfloat16)
    q = torch.randn(400, 2 * 128, device=dev, dtype=torch.bfloat16)
    got = ops.attention(q, cache_k[:900], cache_v[:900], heads=2)
    ok &= report("attn cache prefix", got, attn_ref(q, cache_k[:900], cache_v[:900], 2), 1e-2)
    print("ATTN", "PASS" if ok else "FAIL", flush=True)


def t_elem():
    torch.manual_seed(2)
    ok = True
    L, D, F = 720, 1536, 3
    x = torch.randn(L, D, device=dev, dtype=torch.bfloat16) * 2 + 0.3
    mod = torch.randn(F, 6, D, device=dev, dtype=torch.bfloat16) * 0.5
    ln = torch.nn.functional.layer_norm(x.float(), (D,), eps=1e-6)
    sc = mod[:, 1].float().repeat_interleave(L // F, 0)
    sh = mod[:, 0].float().repeat_interleave(L // F, 0)
    got = ops.ln_modulate(x, eps=1e-6, mod=mod, shift_idx=0, scale_idx=1, rows_per_frame=L // F)
    ok &= report("ln_modulate", got, ln * (1 + sc) + sh, 6e-3)
    w = torch.randn(D, device=dev, dtype=torch.bfloat16); b = torch.randn(D, device=dev, dtype=torch.bfloat16)
    got = ops.ln_modulate(x, eps=1e-6, weight=w, bias=b)
    ok &= report("ln_affine", got, ln * w.float() + b.float(), 6e-3)
    got = ops.rmsnorm(x, w, 1e-6)
    xf = x.float()
    ok &= report("rmsnorm", got, xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * w.float(), 6e-3)
    modulation = torch.randn(1, 6, D, device=dev, dtype=torch.bfloat16)
    got = ops.add_modulation(modulation, mod)
    ok &= report("add_modulation", got, modulation.float() + mod.float(), 4e-3)
    got = ops.activation(x, "silu")
    ok &= report("silu", got, torch.nn.functional.silu(xf), 4e-3)
    # qkv norm + rope
    heads, hd = D // 128, 128
    gh, gw = 12, 20
    qkv = torch.randn(L, 3 * D, device=dev, dtype=torch.bfloat16)
    wq = torch.randn(D, device=dev, dtype=torch.bfloat16); wk = torch.randn(D, device=dev, dtype=torch.bfloat16)
    c = hd // 2
    def rp(n, dim):
        fr = torch.outer(torch.arange(n, dtype=torch.float64),
                         1.0 / torch.pow(10000, torch.arange(0, dim, 2, dtype=torch.float64) / dim))
        return fr
    ang = torch.cat([rp(1024, hd - 4 * (hd // 6)), rp(1024, 2 * (hd // 6)), rp(1024, 2 * (hd // 6))], 1)
    table = torch.stack([ang.cos(), ang.sin()], -1).float().to(dev).contiguous()   # [1024, 64, 2]
    qo = torch.empty(L, D, device=dev, dtype=torch.bfloat16)
    kc = torch.zeros(2 * L, D, device=dev, dtype=torch.bfloat16)
    vc = torch.zeros(2 * L, D, device=dev, dtype=torch.bfloat16)
    start = 2
    ops.qkv_norm_rope(qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], wq, wk, qo, kc[L:], vc[L:], table,
                      head_dim=hd, grid_h=gh, grid_w=gw, start_frame=start, eps=1e-6)
    def ref_one(t, wt):
        tf = t.float()
        n = (tf * torch.rsqrt(tf.pow(2).mean(-1, keepdim=True) + 1e-6)) * wt.float()
        n = n.view(L, heads, c, 2).double()
        idx = torch.arange(L, device=dev)
        f = idx // (gh * gw) + start; h = (idx % (gh * gw)) // gw; wv = idx % gw
        ct = c - 2 * (c // 3); ch = c // 3
        a = torch.cat([ang[:, :ct].to(dev)[f], ang[:, ct:ct + ch].to(dev)[h], ang[:, ct + ch:].to(dev)[wv]], 1)
        cs, sn = a.cos()[:, None, :], a.sin()[:, None, :]
        x0, x1 = n[..., 0], n[..., 1]
        return torch.stack([x0 * cs - x1 * sn, x0 * sn + x1 * cs], -1).reshape(L, D).float()
    ok &= report("qkv rope q", qo, ref_one(qkv[:, :D], wq), 8e-3)
    ok &= report("qkv rope k", kc[L:], ref_one(qkv[:, D:2 * D], wk), 8e-3)
    ok &= report("qkv v copy", vc[L:], qkv[:, 2 * D:], 1e-9)
    ok &= bool((kc[:L] == 0).all())
    # patchify / unpatchify
    C, Fr, H, W = 16, 3, 24, 40
    lat = torch.randn(1, Fr, C, H, W, device=dev, dtype=torch.bfloat16)
    xp = lat[0].permute(1, 0, 2, 3)     # [C,F,H,W] view
    got = ops.patchify(xp)
    refp = xp.reshape(C, Fr, H // 2, 2, W // 2, 2).permute(1, 2, 4, 0, 3, 5).reshape(Fr * (H // 2) * (W // 2), C * 4)
    ok &= report("patchify", got, refp, 1e-9)
    ho = torch.randn(Fr * (H // 2) * (W // 2), 64, device=dev, dtype=torch.bfloat16)
    sig = torch.tensor([0.9, 0.5, 0.1], device=dev, dtype=torch.float64)
    flow, x0 = ops.unpatchify_x0(ho, lat[0].contiguous(), sig, C, Fr, H, W)
    u = ho.view(Fr, H // 2, W // 2, 1, 2, 2, C)
    u = torch.einsum("fhwpqrc->cfphqwr", u).reshape(C, Fr, H, W).permute(1, 0, 2, 3)
    ok &= report("unpatchify flow", flow, u, 1e-9)
    ok &= report("unpatchify x0", x0, (lat[0].double() - sig.view(-1, 1, 1, 1) * u.double()).to(torch.bfloat16), 1e-9)
    print("ELEM", "PASS" if ok else "FAIL", flush=True)


def timeit(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s = torch.cuda.Event(enable_timing=True); e = torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def t_perf():
    torch.manual_seed(3)
    L, D, FF, H = 4680, 5120, 13824, 40
    x = torch.randn(L, D, device=dev, dtype=torch.bfloat16)
    for (N, K, name) in [(15360, D, "qkv"), (D, D, "proj"), (FF, D, "ffn1"), (D, FF, "ffn2")]:
        a = torch.randn(L, K, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, K, device=dev, dtype=torch.bfloat16) * 0.02
        b = torch.zeros(N, device=dev, dtype=torch.bfloat16)
        o = torch.empty(L, N, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.gemm(a, w, b, out=o))
        ms_t = timeit(lambda: torch.nn.functional.linear(a, w, b))
        fl = 2.0 * L * N * K
        print(f"PERF gemm {name} {L}x{N}x{K}: {ms:.3f} ms {fl / ms / 1e9:.1f} TF/s | cuBLAS {ms_t:.3f} ms {fl / ms_t / 1e9:.1f} TF/s", flush=True)
    q = torch.randn(L, D, device=dev, dtype=torch.bfloat16)
    for Lkv in (9360, 4680, 512):
        k = torch.randn(Lkv, D, device=dev, dtype=torch.bfloat16)
        v = torch.randn(Lkv, D, device=dev, dtype=torch.bfloat16)
        o = torch.empty(L, D, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.attention(q, k, v, heads=H, out=o))
        fl = 4.0 * L * Lkv * D
        line = f"PERF attn Lq={L} Lkv={Lkv}: {ms:.3f} ms {fl / ms / 1e9:.1f} TF/s"
        try:
            from flash_attn import flash_attn_func
            q4 = q.view(1, L, H, 128); k4 = k.view(1, Lkv, H, 128); v4 = v.view(1, Lkv, H, 128)
            ms_f = timeit(lambda: flash_attn_func(q4, k4, v4))
            line += f" | FA2 {ms_f:.3f} ms {fl / ms_f / 1e9:.1f} TF/s"
        except Exception as ex:  # noqa: BLE001
            line += f" | FA2 unavailable ({type(ex).__name__})"
        print(line, flush=True)
    mod = torch.randn(3, 6, D, device=dev, dtype=torch.bfloat16)
    o = torch.empty_like(x)
    ms = timeit(lambda: ops.ln_modulate(x, eps=1e-6, mod=mod, rows_per_frame=1560, out=o))
    print(f"PERF ln_modulate: {ms:.3f} ms {2 * x.numel() * 2 / ms / 1e6:.0f} GB/s", flush=True)


def t_attnperf():
    torch.manual_seed(3)
    L, D, H = 4680, 5120, 40
    q = torch.randn(L, D, device=dev, dtype=torch.bfloat16)
    tag = "attn_fwd_kernel"
    for Lkv in (9360, 4680, 512):
        k = torch.randn(Lkv, D, device=dev, dtype=torch.bfloat16)
        v = torch.randn(Lkv, D, device=dev, dtype=torch.bfloat16)
        o = torch.empty(L, D, device=dev, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.attention(q, k, v, heads=H, out=o), n=30, warm=5)
        print(f"PERF attn [{tag}] Lq={L} Lkv={Lkv}: {ms:.3f} ms {4.0 * L * Lkv * D / ms / 1e9:.1f} TF/s", flush=True)


if __name__ == "__main__":
    which = sys.argv[1]
    t0 = time.time()
    {"gemm": t_gemm, "attn": t_attn, "elem": t_elem, "perf": t_perf, "attnperf": t_attnperf}[which]()
    print(f"[{which}] done in {time.time() - t0:.1f}s", flush=True)
