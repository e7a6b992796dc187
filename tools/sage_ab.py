"""A/B of the bf16 attention kernel (kr_attn_fwd) against the quantised tier (kr_sage_quantize + kr_sage_attn) at
(a) the cache-branch shape Lq 4680, Lkv 9360, 40 heads, K/V row pitch 5120 and (b) the cross-attention shape, Lkv 512.
CUDA events, warmed, the variants alternated rep by rep; quantisation is timed on its own and as part of the total.
TFLOP/s = 4 Lq Lkv heads 128 / time.  Prints the GPU name, power limit and max SM clock with the numbers.

    python tools/sage_ab.py [--reps 100] [--out sage_ab.json]
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from realtime_video_b200 import ops  # noqa: E402


def gpu_info() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_clock_max_sm"] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        info["power_limit_clock_max_sm"] = f"unavailable: {ex}"
    return info


def bench(Lq: int, Lkv: int, heads: int, ld: int, reps: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(0)
    W = heads * 128
    q = torch.randn(Lq, W, device="cuda", generator=g).bfloat16()
    k = torch.randn(Lkv, ld, device="cuda", generator=g).bfloat16()[:, :W]
    v = torch.randn(Lkv, ld, device="cuda", generator=g).bfloat16()[:, :W]
    out = torch.empty(Lq, W, device="cuda", dtype=torch.bfloat16)
    buf = ops.sage_buffers(Lq, Lkv, heads, q.device)
    lib = ops._lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    scale = 1.0 / 128 ** 0.5

    def bf16():
        ops.attention(q, k, v, heads=heads, out=out)

    def quant():
        ops.sage_quantize(q, k, v, heads=heads, buffers=buf)

    def attn():
        rc = lib.kr_sage_attn(buf["q_i8"].data_ptr(), buf["q_scale"].data_ptr(), buf["k_i8"].data_ptr(),
                              buf["k_scale"].data_ptr(), buf["v_t8"].data_ptr(), buf["v_scale"].data_ptr(),
                              out.data_ptr(), W, Lq, Lkv, heads, scale, stream)
        ops._lib.check(rc, "kr_sage_attn")

    variants = {"bf16": [bf16], "sage_quantize": [quant], "sage_attn": [attn], "sage_total": [quant, attn]}
    for _ in range(10):
        for fns in variants.values():
            for f in fns:
                f()
    torch.cuda.synchronize()
    times = {n: [] for n in variants}
    for _ in range(reps):
        for n, fns in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for f in fns:
                f()
            b.record()
            times[n].append((a, b))
    torch.cuda.synchronize()
    flops = 4.0 * Lq * Lkv * heads * 128
    res = {"shape": dict(Lq=Lq, Lkv=Lkv, heads=heads, ld=ld), "reps": reps}
    for n, ev in times.items():
        ms = sorted(x.elapsed_time(y) for x, y in ev)
        med = ms[len(ms) // 2]
        res[n] = {"ms_median": med, "ms_min": ms[0], "ms_max": ms[-1]}
        if n != "sage_quantize":
            res[n]["tflops"] = flops / (med * 1e-3) / 1e12
    res["speedup_total_vs_bf16"] = res["bf16"]["ms_median"] / res["sage_total"]["ms_median"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.reps < 50:
        ap.error("--reps must be at least 50")
    if not torch.cuda.is_available():
        sys.exit("sage_ab.py needs a CUDA device")
    res = {"gpu": gpu_info(),
           "cache_branch": bench(4680, 9360, 40, 5120, a.reps),
           "cross_attention": bench(4680, 512, 40, 5120, a.reps)}
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
