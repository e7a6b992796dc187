"""A/B of the INT8 DiT linears (torchao Int8DynamicActivationInt8WeightConfig: s8 wgmma, exact s32 accumulation on a
128 x 256 tile) against the row-scaled FP8 ones, one command:

  gemm   the six DiT projections of one block at M = 4680 with their real epilogues and operand layouts:
         kr_gemm_i8_rowwise vs kr_gemm_fp8_rowwise (promoted) vs kr_gemm_fp8_rowwise_fast, alternated; CUDA-event
         medians and p10 / p90 of --reps launches after warm-up: ms, algorithmic TFLOP/s (2 M N K over the time) and
         its share of the 1979 TFLOP/s (TOPS for INT8) the H100 SXM data sheet gives for dense FP8 and INT8 (a
         data-sheet figure for a 700 W card, not a measured peak);
  loop   the bench's server-loop workload (Wan-14B dims, 832x480, 12 frames per block, 4 denoising steps) after
         ``quantize_`` with PerRow FP8 and fast accumulation vs INT8, arms alternated --rounds times in one process,
         per arm --warmup + --steps blocks and one further block with CUDA events around every kernel family
         (ops.profile_begin / profile_end).

Prints the GPU name, power limit and max SM clock with the numbers.

    python tools/int8_ab.py [--parts gemm,loop] [--reps 100] [--out int8_ab.json]
"""
import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import harness  # noqa: E402
from realtime_video_b200 import factory, fp8, ops  # noqa: E402

M, D, FFN, ROWS_PER_GATE = 4680, 5120, 13824, 1560
SHAPES = [("to_qkv", 3 * D, D, ops.EPI_BIAS), ("self_o", D, D, ops.EPI_BIAS_GATE_RES),
          ("cross_q", D, D, ops.EPI_BIAS), ("cross_o", D, D, ops.EPI_BIAS_RES),
          ("ffn0", FFN, D, ops.EPI_BIAS_GELU), ("ffn2", D, FFN, ops.EPI_BIAS_GATE_RES)]
DATA_SHEET_8BIT_TFLOPS = 1979.0
FRAMES_PER_BLOCK = 12
KERNELS = ("int8", "fp8_row", "fp8_row_fast")
ARMS = ("fp8_row_fast", "int8")


def gpu_info() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["name_power_limit_clock_max_sm"] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        info["name_power_limit_clock_max_sm"] = f"unavailable: {ex}"
    return info


def make_call(name: str, N: int, K: int, epi: int, kernel: str, g: torch.Generator):
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).bfloat16()
    b = (torch.randn(N, device="cuda", generator=g) * 0.1).bfloat16()
    if kernel == "int8":
        wq, sw = fp8.quantize_weight_int8_rows(w)
        a = ops.i8_quantize_rows(x)
        run = lambda **kw: ops.gemm_i8_rowwise(a, wq, sw, b, **kw)      # noqa: E731
    else:
        wq, sw = fp8.quantize_weight_rows(w)
        a = ops.fp8_quantize_rows(x)
        fast = kernel == "fp8_row_fast"
        run = lambda **kw: ops.gemm_fp8_rowwise(a, wq, sw, b, fast_accum=fast, **kw)    # noqa: E731
    del x, w
    if name == "to_qkv":
        qk = torch.empty(M, 2 * D, device="cuda", dtype=torch.bfloat16)
        v_cache = torch.empty(2 * M, D, device="cuda", dtype=torch.bfloat16)
        return lambda: run(out=qk, out2=v_cache[M:], n_split=2 * D)
    if epi in (ops.EPI_BIAS, ops.EPI_BIAS_GELU):
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        return lambda: run(epilogue=epi, out=out)
    r = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    if epi == ops.EPI_BIAS_RES:
        return lambda: run(epilogue=epi, residual=r, out=r)
    gate = (torch.randn(M // ROWS_PER_GATE, N, device="cuda", generator=g) * 0.1).bfloat16()
    return lambda: run(epilogue=epi, residual=r, gate=gate, rows_per_gate=ROWS_PER_GATE, out=r)


def timed_ms(fn, reps: int) -> list:
    ev = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        ev.append((s, e))
    torch.cuda.synchronize()
    return [s.elapsed_time(e) for s, e in ev]


def part_gemm(reps: int) -> dict:
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {}
    total = {k: 0.0 for k in KERNELS}
    for name, N, K, epi in SHAPES:
        calls = {k: make_call(name, N, K, epi, k, g) for k in KERNELS}
        for fn in calls.values():
            for _ in range(10):
                fn()
        torch.cuda.synchronize()
        ms = {k: [] for k in KERNELS}
        chunk = max(1, reps // 4)
        done = 0
        while done < reps:                                          # int8, fp8_row, fp8_row_fast, int8, ...
            for k in KERNELS:
                ms[k] += timed_ms(calls[k], min(chunk, reps - done))
            done += chunk
        row = {}
        for k in KERNELS:
            s = sorted(ms[k])
            t = s[len(s) // 2]
            tf = 2.0 * M * N * K / (t * 1e-3) / 1e12
            row[k] = {"ms": t, "ms_p10": s[len(s) // 10], "ms_p90": s[(9 * len(s)) // 10], "tflops": tf,
                      "share_of_data_sheet": tf / DATA_SHEET_8BIT_TFLOPS, "reps": len(s)}
            total[k] += t
        res[name] = dict(row, N=N, K=K, epilogue=epi)
        print(f"{name:8s} {N:5d}x{K:5d} " + " | ".join(
            f"{k} {row[k]['ms']:6.3f} ms [{row[k]['ms_p10']:6.3f}, {row[k]['ms_p90']:6.3f}] {row[k]['tflops']:6.1f}"
            for k in KERNELS), flush=True)
        del calls
        torch.cuda.empty_cache()
    res["sum_of_six_ms"] = total
    print("sum of the six:", json.dumps(total))
    return res


def _config(arm: str):
    if arm == "int8":
        return fp8.Int8DynamicActivationInt8WeightConfig()
    return fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow(),
                                                         mm_config=fp8.Float8MMConfig(use_fast_accum=True))


def run_arm(transformer, models, pe, arm: str, steps: int, warmup: int, seed: int) -> dict:
    fp8.quantize_(transformer, _config(arm))
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
            a.record()
            ops.profile_begin()
            sess.generate_block()
            b.record()
            torch.cuda.synchronize()
            prof = ops.profile_end()
            prof_ms = a.elapsed_time(b)
    finally:
        fp8.dequantize_(transformer)
    kernels = {k: {"ms": v["ms"], "launches": v["n"],
                   "tflops": v["flops"] / (v["ms"] * 1e-3) / 1e12 if v["ms"] > 0 and v["flops"] > 0 else None}
               for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}
    return {"arm": arm, "fps": steps * FRAMES_PER_BLOCK / (ms / 1e3), "ms_per_block": ms / steps,
            "profiled_block_ms": prof_ms, "kernels_one_block": kernels}


def part_loop(steps: int, warmup: int, rounds: int) -> dict:
    transformer = factory.synthetic_transformer("14B", device="cuda", seed=0)
    models = harness.build_models(transformer, vae_decoder=factory.synthetic_vae_decoder(device="cuda"),
                                  device="cuda")
    pe = factory.synthetic_prompt_embeds(device="cuda")
    arms = []
    for r in range(rounds):
        for arm in ARMS:
            arms.append(run_arm(transformer, models, pe, arm, steps, warmup, seed=4042 + r))
            print(json.dumps({k: v for k, v in arms[-1].items() if k != "kernels_one_block"}), flush=True)
    res = {"workload": {"dims": "14B", "width": 832, "height": 480, "frames_per_block": FRAMES_PER_BLOCK,
                        "denoising_steps": 4, "timed_blocks": steps, "warmup_blocks": warmup},
           "arms": arms}
    for arm in ARMS:
        res[f"{arm}_fps"] = [x["fps"] for x in arms if x["arm"] == arm]
    res["int8_over_fp8_row_fast"] = sum(res["int8_fps"]) / sum(res["fp8_row_fast_fps"])
    del transformer, models
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="gemm,loop")
    ap.add_argument("--reps", type=int, default=100, help="timed launches per shape and kernel (gemm)")
    ap.add_argument("--steps", type=int, default=4, help="timed blocks per arm (loop)")
    ap.add_argument("--warmup", type=int, default=2, help="warm-up blocks per arm (loop)")
    ap.add_argument("--rounds", type=int, default=2, help="FP8 fast / INT8 pairs, alternated (loop)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    parts = a.parts.split(",")
    if a.reps < 100 and "gemm" in parts:
        ap.error("--reps must be at least 100")
    if not torch.cuda.is_available():
        sys.exit("int8_ab.py needs a CUDA device")
    torch.cuda.set_device(0)
    res = {"gpu": gpu_info()}
    print(json.dumps(res["gpu"]), flush=True)
    if "gemm" in parts:
        res["gemm"] = part_gemm(a.reps)
    if "loop" in parts:
        res["loop"] = part_loop(a.steps, a.warmup, a.rounds)
    text = json.dumps(res, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        Path(a.out).write_text(text + "\n")
    else:
        print(text)


if __name__ == "__main__":
    main()
