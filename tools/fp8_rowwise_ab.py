"""A/B of the two FP8 granularities on the bench's server-loop workload (Wan-14B dims, 832x480, 12 frames per block,
4 denoising steps, one GPU, one process): ``quantize_`` with PerTensor and with PerRow, alternated (T, R, T, R by
default).  Per arm: warm-up blocks, then timed blocks between CUDA events (fps = 12 frames per block), then ONE more
block with CUDA events around every quantise, LayerNorm and FP8 GEMM launch for the per-kernel totals of that block.
Prints the GPU name, power limit and max SM clock with the numbers.

    python tools/fp8_rowwise_ab.py [--steps 4] [--warmup 2] [--rounds 2] [--out fp8_rowwise_ab.json]
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import harness  # noqa: E402
from realtime_video_b200 import factory, fp8, ops  # noqa: E402

FRAMES_PER_BLOCK = 12
# kernel family -> the ops entry points of each granularity that launch it
FAMILIES = {"quantise": ("fp8_quantize", "fp8_quantize_rows"), "layernorm": ("ln_modulate", "ln_modulate_fp8"),
            "gemm_fp8": ("gemm_fp8", "gemm_fp8_rowwise")}


def gpu_info() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["power_limit_clock_max_sm"] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        info["power_limit_clock_max_sm"] = f"unavailable: {ex}"
    return info


class KernelEvents:
    """Wraps the ops entry points of FAMILIES with CUDA events on the current stream while active."""

    def __init__(self):
        self.events = {fam: [] for fam in FAMILIES}
        self.saved = {}

    def __enter__(self):
        for fam, names in FAMILIES.items():
            for name in names:
                fn = getattr(ops, name)
                self.saved[name] = fn

                def timed(*a, _fn=fn, _fam=fam, **k):
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    s.record()
                    out = _fn(*a, **k)
                    e.record()
                    self.events[_fam].append((s, e))
                    return out
                setattr(ops, name, timed)
        return self

    def __exit__(self, *exc):
        for name, fn in self.saved.items():
            setattr(ops, name, fn)
        return False

    def totals(self) -> dict:
        torch.cuda.synchronize()
        return {fam: {"ms": sum(s.elapsed_time(e) for s, e in ev), "launches": len(ev)}
                for fam, ev in self.events.items()}


def run_arm(transformer, models, pe, granularity, steps: int, warmup: int, seed: int) -> dict:
    fp8.quantize_(transformer, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=granularity))
    try:
        sess = harness.GenerationSession(harness.GenerateParams(num_blocks=warmup + steps + 1, seed=seed), models,
                                         prompt_embeds=pe, device="cuda")
        with torch.inference_mode():
            for _ in range(warmup):
                sess.generate_block()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                sess.generate_block()
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b)
            with KernelEvents() as kev:
                sess.generate_block()
            kernels = kev.totals()
    finally:
        fp8.dequantize_(transformer)
    return {"granularity": type(granularity).__name__, "fps": steps * FRAMES_PER_BLOCK / (ms / 1e3),
            "ms_per_block": ms / steps, "kernels_one_block": kernels}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4, help="timed blocks per arm")
    ap.add_argument("--warmup", type=int, default=2, help="warm-up blocks per arm")
    ap.add_argument("--rounds", type=int, default=2, help="PerTensor / PerRow pairs, alternated")
    ap.add_argument("--layers", type=int, default=None, help="DiT layers (default: all 40 of the 14B model)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fp8_rowwise_ab.py needs a CUDA device")
    torch.cuda.set_device(0)
    kw = {} if a.layers is None else {"num_layers": a.layers}
    transformer = factory.synthetic_transformer("14B", device="cuda", seed=0, **kw)
    models = harness.build_models(transformer, vae_decoder=factory.synthetic_vae_decoder(device="cuda"),
                                  device="cuda")
    pe = factory.synthetic_prompt_embeds(device="cuda")
    arms = []
    for r in range(a.rounds):
        for g in (fp8.PerTensor(), fp8.PerRow()):
            arms.append(run_arm(transformer, models, pe, g, a.steps, a.warmup, seed=4042 + r))
            print(json.dumps(arms[-1]), flush=True)
    res = {"gpu": gpu_info(), "workload": {"dims": "14B", "width": 832, "height": 480,
                                           "frames_per_block": FRAMES_PER_BLOCK, "denoising_steps": 4,
                                           "timed_blocks": a.steps, "warmup_blocks": a.warmup},
           "arms": arms}
    for name in ("PerTensor", "PerRow"):
        fps = [x["fps"] for x in arms if x["granularity"] == name]
        res[f"{name}_fps"] = fps
    res["PerRow_over_PerTensor"] = sum(res["PerRow_fps"]) / sum(res["PerTensor_fps"])
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        Path(a.out).write_text(text + "\n")


if __name__ == "__main__":
    main()
