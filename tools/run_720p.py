"""BASELINE configs[3]: 1280x720, kv_cache_num_frames=5 (Lq 10800, Lkv up to 28800), 14B dims, on one GPU.

Runs ``--blocks`` blocks of the synthetic session (DiT, VAE decode, and the first-frame re-encode once the context
window has slid) and prints one JSON line: steady-block fps (the blocks after the slide), the peak
``torch.cuda.max_memory_allocated`` and the card it ran on (name, power limit, max SM clock, read in the same run).
``KR_VAE_FP8=1`` runs the VAE decoder's FP8 tier.  Per-block lines go to stderr."""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from realtime_video_b200 import factory  # noqa: E402
import harness  # noqa: E402
from harness import GenerateParams, GenerationSession  # noqa: E402

KV_FRAMES, FRAMES_PER_BLOCK = 5, 3


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(torch.cuda.current_device())], capture_output=True, text=True)
    fields = q.stdout.strip().split(", ") if q.returncode == 0 else []
    power, clock = (fields[1:] + ["unknown"] * 2)[:2]
    return {"gpu": torch.cuda.get_device_name(), "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--blocks", type=int, default=8, help="blocks to generate (the window slides at block 3)")
    args = ap.parse_args()
    slide = 1 + -(-KV_FRAMES // FRAMES_PER_BLOCK)          # first block that re-encodes its first context frame
    if args.blocks <= slide:
        ap.error(f"--blocks must exceed {slide}: the steady blocks are the ones after the window slides")
    w = factory.synthetic_transformer("14B")
    vae = factory.synthetic_vae_decoder()
    enc = factory.synthetic_vae_encoder()
    models = harness.build_models(w, vae_decoder=vae, vae_encoder=enc)
    pe = factory.synthetic_prompt_embeds()
    sess = GenerationSession(GenerateParams(width=1280, height=720, kv_cache_num_frames=KV_FRAMES,
                                            num_blocks=args.blocks), models, prompt_embeds=pe)
    steady_ms, steady_frames, finite = 0.0, 0, True
    for b in range(args.blocks):
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        px = sess.generate_block()
        e.record()
        torch.cuda.synchronize()
        ms = s.elapsed_time(e)
        ok = bool(torch.isfinite(px).all())
        finite &= ok
        if b >= slide:
            steady_ms, steady_frames = steady_ms + ms, steady_frames + px.shape[1]
        print(f"block {b}: {tuple(px.shape)} {ms:.1f} ms finite={ok} "
              f"peak {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB", file=sys.stderr, flush=True)
    line = {"metric": "frames_per_second_1280x720_kv5_steady", "value": steady_frames / (steady_ms / 1e3),
            "unit": "frames/s", "blocks": args.blocks, "steady_blocks": args.blocks - slide,
            "vae_quant": vae.quant or "fp16", "decoder_frame_tile": vae.engine.frame_tile,
            "max_memory_allocated_gib": torch.cuda.max_memory_allocated() / 2**30, "finite": finite, **gpu_info()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
