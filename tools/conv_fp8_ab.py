"""Two library A/Bs on one GPU (short): (1) the VAE's two heavy 3x3x3 causal convs (S3: 96->96 at 480x832, S2: 192->192 at
240x416, 12 output frames, fp16) — ours (conv_halo_kernel incl. the fused RMS-norm/SiLU + residual epilogue) vs cuDNN
through torch.nn.functional.conv3d (channels_last_3d, conv only, no epilogue); (2) FP8 GEMM — ours vs cuBLASLt
(torch._scaled_mm) on the ffn.0 / ffn.2 shapes.    python tools/conv_fp8_ab.py"""
import sys

import torch

sys.path.insert(0, ".")
from realtime_video_b200 import fp8, ops  # noqa: E402
from realtime_video_b200.vae import _prep_conv, _tile_for  # noqa: E402

dev = "cuda"


def timeit(fn, n=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


torch.manual_seed(0)
for (C, H, W, T) in [(96, 480, 832, 12), (192, 240, 416, 12)]:
    w = (torch.randn(C, C, 3, 3, 3) / (27 * C) ** 0.5).half()
    c = _prep_conv(w, torch.zeros(C).half(), torch.float16, dev)
    x = torch.randn(T + 2, H, W, C, device=dev, dtype=torch.float16)
    out = torch.empty(T, H, W, C, device=dev, dtype=torch.float16)
    nrm = torch.empty(T, H, W, C, device=dev, dtype=torch.float16)
    gamma = torch.ones(C, device=dev, dtype=torch.float16)
    ms = timeit(lambda: ops.vae_conv(x, c.weight, c.bias, n=c.n, cout=c.cout, T=T, taps=(3, 3, 3), tile=_tile_for(H, W),
                                     out_raw=out, out_norm=nrm, gamma=gamma, residual=out))
    fl = 2.0 * T * H * W * C * C * 27
    # cuDNN: NCDHW logical shape in channels_last_3d memory, spatial padding 1, the 2 cached frames in front (causal)
    xc = x.permute(3, 0, 1, 2)[None].contiguous(memory_format=torch.channels_last_3d)
    wc = w.to(dev).contiguous(memory_format=torch.channels_last_3d)
    bc = torch.zeros(C, device=dev, dtype=torch.float16)
    torch.backends.cudnn.benchmark = True
    ms_c = timeit(lambda: torch.nn.functional.conv3d(xc, wc, bc, padding=(0, 1, 1)))
    print(f"conv3d 3x3x3 {C}->{C} @ {H}x{W} x {T} frames: ours (conv + norm/SiLU + residual epilogue) {ms:.3f} ms "
          f"{fl / ms / 1e9:.0f} TF/s | cuDNN conv only {ms_c:.3f} ms {fl / ms_c / 1e9:.0f} TF/s | ours/cuDNN time {ms / ms_c:.2f}",
          flush=True)

M = 4680
for (N, K, name) in [(13824, 5120, "ffn1"), (5120, 13824, "ffn2"), (15360, 5120, "qkv")]:
    a = torch.randn(M, K, device=dev).bfloat16()
    w = (torch.randn(N, K, device=dev) * 0.02).bfloat16()
    b = torch.zeros(N, device=dev, dtype=torch.bfloat16)
    wq, sw = fp8.quantize_weight(w)
    aq, st = ops.fp8_quantize(a)
    o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    ms = timeit(lambda: ops.gemm_fp8(aq, wq, st, sw, b, out=o), n=20)
    ms_q = timeit(lambda: ops.fp8_quantize(a, aq, st), n=20)
    a8, w8 = aq.view(torch.float8_e4m3fn), wq.view(torch.float8_e4m3fn)
    sa, sb = st[1:2].clone(), torch.tensor([sw], device=dev)
    try:
        ms_c = timeit(lambda: torch._scaled_mm(a8, w8.t(), scale_a=sa, scale_b=sb, bias=b, out_dtype=torch.bfloat16,
                                               use_fast_accum=True), n=20)
        lib = f"cuBLASLt fp8 {ms_c:.3f} ms {2.0 * M * N * K / ms_c / 1e9:.0f} TF/s | ours/cuBLASLt {ms_c / ms:.3f}"
    except Exception as ex:  # noqa: BLE001
        lib = f"torch._scaled_mm unavailable ({type(ex).__name__}: {str(ex)[:80]})"
    print(f"fp8 gemm {name} {M}x{N}x{K}: ours {ms:.3f} ms {2.0 * M * N * K / ms / 1e9:.0f} TF/s (+ activation cast {ms_q:.3f} ms) | {lib}",
          flush=True)
