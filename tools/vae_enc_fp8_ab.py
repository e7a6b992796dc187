"""A/B of the VAE encoder's FP8 (e4m3) conv tier against fp16, alternated in one process (fp16, FP8, fp16, FP8).

Workload: a webcam-style stream (the server's process_webcam_frames path): one fresh 1-frame chunk, then warm
stream=True calls of 4 pixel frames (48 timed per arm by default, about a second at 832x480) through the synthetic encoder, at 832x480 and 1280x720.  Per arm: timed calls
between CUDA events (encoded frames/s), one 12-frame block (three 4-frame calls) with CUDA events around every conv
launch (conv time per block: total and e4m3 convs), and torch.cuda.max_memory_allocated of an encoder stream.
Prints the GPU name, power limit and max SM clock with the numbers.

    python tools/vae_enc_fp8_ab.py [--steps 48] [--warmup 3] [--rounds 2] [--out vae_enc_fp8_ab.json]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from realtime_video_b200 import factory, ops  # noqa: E402
from tools.fp8_rowwise_ab import gpu_info  # noqa: E402


def clips(H, W, n=4):
    g = torch.Generator(device="cuda").manual_seed(0)
    return [(torch.rand(1, 3, 4, H, W, device="cuda", generator=g) * 2 - 1).half() for _ in range(n)]


def enc_arm(enc, xs, steps, warmup):
    with torch.no_grad():
        _, cache = enc(xs[0][:, :, :1], [None] * 55)                  # first chunk of the stream
        for i in range(warmup):
            _, cache = enc(xs[i % 4], cache, stream=True)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(steps):
            _, cache = enc(xs[i % 4], cache, stream=True)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / steps
        ops.profile_begin()
        for i in range(3):                                            # one 12-frame block
            _, cache = enc(xs[i], cache, stream=True)
        torch.cuda.synchronize()
        prof = ops.profile_end()
    conv = prof.get("vae_conv", {"ms": 0.0, "n": 0})
    return {"ms_per_call": ms, "frames_per_s": 4 / (ms / 1e3), "conv_ms_per_block": conv["ms"],
            "conv_launches_per_block": conv["n"], "conv_fp8_ms_per_block": prof.get("vae_conv/fp8", {"ms": 0.0})["ms"]}


def peak_memory(quant, H, W):
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    enc = factory.synthetic_vae_encoder(device="cuda")
    enc.quant = quant
    x = clips(H, W, 1)[0]
    with torch.no_grad():
        _, c = enc(x[:, :, :1], [None] * 55)
        _, c = enc(x, c, stream=True)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del enc, c
    torch.cuda.empty_cache()
    return peak / 2 ** 30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=48)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"gpu": gpu_info(), "peak_gib": {}}
    for H, W in ((480, 832), (720, 1280)):
        key = f"vae_encode_{W}x{H}"
        out[key] = []
        xs = clips(H, W)
        encs = {None: factory.synthetic_vae_encoder(device="cuda"), "fp8": factory.synthetic_vae_encoder(device="cuda")}
        encs["fp8"].quant = "fp8"
        for r in range(args.rounds):
            for q in (None, "fp8"):
                res = enc_arm(encs[q], xs, args.steps, args.warmup)
                res.update(arm=q or "fp16", round=r, size=f"{W}x{H}")
                out[key].append(res)
                print(json.dumps(res), flush=True)
        del encs, xs
        for q in (None, "fp8"):
            out["peak_gib"][f"{W}x{H}/{q or 'fp16'}"] = peak_memory(q, H, W)
    print(json.dumps(out["peak_gib"]), flush=True)
    print(json.dumps(out["gpu"]))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
