"""The six bf16 DiT projections of one block at M = 4680 (the bench's 832x480 server loop, 3 frames of 1560 rows),
each with its real epilogue and operand layout, timed at their real K and again at K = 64, where the epilogue is most
of the kernel.  From the two: the exposed epilogue time per tile and its share of each shape's time.

  to_qkv   15360 x 5120   bias, columns >= 10240 (V) into a row slice of a V cache
  self o    5120 x 5120   bias + per-frame gate + in-place residual
  cross q   5120 x 5120   bias
  cross o   5120 x 5120   bias + in-place residual
  ffn.0    13824 x 5120   bias + GELU-tanh
  ffn.2     5120 x 13824  bias + per-frame gate + in-place residual

CUDA-event medians over --reps launches after warm-up.  Prints the GPU name, power limit and max SM clock with the
numbers.  `--ab N` instead runs the script N times per arm in subprocesses, alternating KR_GEMM_EPI_WARPS=0 / 1 (the
library reads the switch once per process), and prints both arms' per-shape times and TFLOP/s.

    python tools/gemm_epi_ab.py [--reps 100] [--ab 2] [--out gemm_epi_ab.json]
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
from realtime_video_b200 import _lib, ops  # noqa: E402

M, D, FFN, ROWS_PER_GATE = 4680, 5120, 13824, 1560
SHAPES = [("to_qkv", 3 * D, D, ops.EPI_BIAS), ("self_o", D, D, ops.EPI_BIAS_GATE_RES),
          ("cross_q", D, D, ops.EPI_BIAS), ("cross_o", D, D, ops.EPI_BIAS_RES),
          ("ffn0", FFN, D, ops.EPI_BIAS_GELU), ("ffn2", D, FFN, ops.EPI_BIAS_GATE_RES)]
KERNELS = {1: "gemm_tn_kernel", 2: "gemm2_tn_kernel", 3: "gemm_sk_kernel", 4: "gemm_flex_kernel"}


def gpu_info() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        info["name_power_limit_clock_max_sm"] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        info["name_power_limit_clock_max_sm"] = f"unavailable: {ex}"
    return info


def make_call(name: str, N: int, K: int, epi: int, g: torch.Generator):
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.02).bfloat16()
    b = (torch.randn(N, device="cuda", generator=g) * 0.1).bfloat16()
    if name == "to_qkv":
        qk = torch.empty(M, 2 * D, device="cuda", dtype=torch.bfloat16)
        v_cache = torch.empty(2 * M, D, device="cuda", dtype=torch.bfloat16)
        return lambda: ops.gemm(a, w, b, out=qk, out2=v_cache[M:], n_split=2 * D)
    if epi in (ops.EPI_BIAS, ops.EPI_BIAS_GELU):
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        return lambda: ops.gemm(a, w, b, epilogue=epi, out=out)
    x = torch.randn(M, N, device="cuda", generator=g).bfloat16()
    if epi == ops.EPI_BIAS_RES:
        return lambda: ops.gemm(a, w, b, epilogue=epi, residual=x, out=x)
    gate = torch.randn(M // ROWS_PER_GATE, N, device="cuda", generator=g).bfloat16()
    return lambda: ops.gemm(a, w, b, epilogue=epi, residual=x, gate=gate, rows_per_gate=ROWS_PER_GATE, out=x)


def median_ms(fn, reps: int) -> float:
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    ev = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        ev.append((s, e))
    torch.cuda.synchronize()
    ms = sorted(s.elapsed_time(e) for s, e in ev)
    return ms[len(ms) // 2]


def measure(reps: int) -> dict:
    lib = _lib.load()
    ops.stream_k = False   # the data-parallel kernels the bench runs (stream-K is opt-in, KR_GEMM_SK=1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"gpu": gpu_info(), "epi_warps_env": os.environ.get("KR_GEMM_EPI_WARPS"), "M": M, "reps": reps,
           "shapes": {}}
    tot_full = tot_epi = 0.0
    for name, N, K, epi in SHAPES:
        t_full = median_ms(make_call(name, N, K, epi, g), reps)
        t_k64 = median_ms(make_call(name, N, 64, epi, g), reps)
        torch.cuda.empty_cache()
        # the K = 64 kernel runs the fixed-width dispatch: 128 x 256 tiles where N % 256 == 0, else 128 x 128
        bn64 = 256 if N % 256 == 0 and ((M + 127) // 128) * (N // 256) >= sms else 128
        tiles64 = ((M + 127) // 128) * ((N + bn64 - 1) // bn64)
        waves64 = (tiles64 + sms - 1) // sms
        tf = 2.0 * M * N * K / (t_full * 1e-3) / 1e12
        res["shapes"][name] = {
            "N": N, "K": K, "epilogue": epi,
            "kernel": KERNELS[lib.kr_gemm_kernel_id_ws(epi, M, N, K, 0)],
            "ms": t_full, "tflops": tf, "ms_k64": t_k64,
            # one 64-wide k-block of mainloop and the launch are inside t_k64, so both are upper bounds
            "epi_us_per_tile_k64": t_k64 * 1e3 / waves64, "tile_n_k64": bn64,
            "epi_share": t_k64 / t_full}
        tot_full += t_full
        tot_epi += t_k64
        print(f"{name:8s} {N:5d}x{K:5d} {res['shapes'][name]['kernel']:16s} {t_full:7.3f} ms {tf:6.1f} TFLOP/s | "
              f"K=64 {t_k64:6.3f} ms, {t_k64 * 1e3 / waves64:5.2f} us/tile, share {t_k64 / t_full:6.1%}", flush=True)
    res["total_ms"], res["total_ms_k64"], res["epi_share_total"] = tot_full, tot_epi, tot_epi / tot_full
    print(f"sum of the six: {tot_full:.3f} ms, K=64 {tot_epi:.3f} ms, epilogue share {tot_epi / tot_full:.1%}")
    return res


def ab(n: int, reps: int) -> dict:
    runs = {"0": [], "1": []}
    for i in range(n):
        for arm in ("0", "1"):
            env = dict(os.environ, KR_GEMM_EPI_WARPS=arm)
            r = subprocess.run([sys.executable, __file__, "--reps", str(reps), "--json-only"], cwd=ROOT, env=env,
                               capture_output=True, text=True, timeout=1200)
            if r.returncode != 0:
                sys.exit(f"arm KR_GEMM_EPI_WARPS={arm} failed:\n{r.stdout[-2000:]}{r.stderr[-4000:]}")
            runs[arm].append(json.loads(r.stdout.strip().splitlines()[-1]))
    res = {"gpu": runs["1"][0]["gpu"], "repeats_per_arm": n, "reps": reps, "shapes": {}}
    print(f"{'shape':8s} | KR_GEMM_EPI_WARPS=0 ms (TFLOP/s) per repeat | =1 ms (TFLOP/s) per repeat | change")
    for name, N, K, _ in SHAPES:
        row = {}
        for arm in ("0", "1"):
            row[arm] = {"ms": [x["shapes"][name]["ms"] for x in runs[arm]],
                        "tflops": [x["shapes"][name]["tflops"] for x in runs[arm]],
                        "kernel": runs[arm][0]["shapes"][name]["kernel"]}
        m0, m1 = min(row["0"]["ms"]), min(row["1"]["ms"])
        row["change_best"] = m1 / m0 - 1
        res["shapes"][name] = row
        f = lambda arm: " ".join(f"{t:.3f} ({tf:.0f})" for t, tf in zip(row[arm]["ms"], row[arm]["tflops"]))  # noqa
        print(f"{name:8s} | {f('0')} | {f('1')} | {row['change_best']:+.1%}")
    for arm in ("0", "1"):
        res["total_ms_" + arm] = [x["total_ms"] for x in runs[arm]]
    print(f"sum      | {res['total_ms_0']} | {res['total_ms_1']}")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--ab", type=int, default=0, help="repeats per arm of KR_GEMM_EPI_WARPS=0 / 1, alternated")
    ap.add_argument("--out", default=None)
    ap.add_argument("--json-only", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.reps < 50:
        ap.error("--reps must be at least 50")
    if not torch.cuda.is_available():
        sys.exit("gemm_epi_ab.py needs a CUDA device")
    if a.json_only:
        sys.stdout = open(os.devnull, "w")
        res = measure(a.reps)
        sys.stdout = sys.__stdout__
        print(json.dumps(res))
        return
    res = ab(a.ab, a.reps) if a.ab > 0 else measure(a.reps)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
