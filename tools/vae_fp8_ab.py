"""A/B of the VAE decoder's FP8 (e4m3) conv tier against fp16, alternated in one process (16, 8, 16, 8 by default).

1. The bench's VAE-decode-only workload (BASELINE configs[4]): a warm stream of 3-latent-frame blocks at 832x480
   through the synthetic decoder; per arm, timed blocks between CUDA events (frames/s, 12 frames per block) and one
   more block with CUDA events around every conv launch (conv time per block).
2. torch.cuda.max_memory_allocated of a decoder stream at 832x480 and 1280x720 for both arms.
Prints the GPU name, power limit and max SM clock with the numbers.

    python tools/vae_fp8_ab.py [--steps 8] [--warmup 3] [--rounds 2] [--out vae_fp8_ab.json]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from realtime_video_b200 import factory, ops  # noqa: E402
from tools.fp8_rowwise_ab import gpu_info  # noqa: E402


def vae_arm(dec, zs, steps, warmup):
    cache = [None] * 55
    with torch.no_grad():
        px, cache = dec(zs[0], *cache)                     # first block of the stream
        for i in range(warmup):
            px, cache = dec(zs[1 + i % 4], *cache)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(steps):
            px, cache = dec(zs[1 + i % 4], *cache)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / steps
        ops.profile_begin()
        px, cache = dec(zs[1], *cache)
        torch.cuda.synchronize()
        prof = ops.profile_end()
    conv = prof.get("vae_conv", {"ms": 0.0, "n": 0})
    return {"ms_per_block": ms, "frames_per_s": 12 / (ms / 1e3), "conv_ms_per_block": conv["ms"],
            "conv_launches": conv["n"], "conv_fp8_ms": prof.get("vae_conv/fp8", {"ms": 0.0})["ms"]}


def peak_memory(quant, H, W):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    dec = factory.synthetic_vae_decoder(device="cuda")
    dec.quant = quant
    z = torch.randn(1, 3, 16, H // 8, W // 8, device="cuda").half()
    with torch.no_grad():
        _, c = dec(z, *([None] * 55))
        _, c = dec(z, *c)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del dec, c
    torch.cuda.empty_cache()
    return peak / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    out = {"gpu": gpu_info(), "vae_decode_832x480": [], "peak_gib": {}}
    zs = [torch.randn(1, 3, 16, 60, 104, device="cuda").half() for _ in range(5)]
    decs = {None: factory.synthetic_vae_decoder(device="cuda"), "fp8": factory.synthetic_vae_decoder(device="cuda")}
    decs["fp8"].quant = "fp8"
    for r in range(args.rounds):
        for q in (None, "fp8"):
            res = vae_arm(decs[q], zs, args.steps, args.warmup)
            res.update(arm=q or "fp16", round=r)
            out["vae_decode_832x480"].append(res)
            print(json.dumps(res), flush=True)
    del decs
    for H, W in ((480, 832), (720, 1280)):
        for q in (None, "fp8"):
            out["peak_gib"][f"{W}x{H}/{q or 'fp16'}"] = peak_memory(q, H, W)
    print(json.dumps(out["peak_gib"]), flush=True)
    print(json.dumps(out["gpu"]))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
