"""GEMM A/B on one GPU: ours (planned kernel, with and without the stream-K workspace) vs cuBLAS (torch F.linear)
for the four DiT projections at M = 4680 and at the sequence-parallel shards M = 2340 / 1170 / 585.
    python tools/gemm_ab.py"""
import sys

import torch

sys.path.insert(0, ".")
from realtime_video_b200 import _lib, ops  # noqa: E402

dev = "cuda"


def timeit(fn, n=20, warm=5):
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


lib = _lib.load()
names = {1: "single", 2: "pair", 3: "streamK", 4: "flex"}
print("shape                      | ours(ws) kernel TF/s | ours(no ws) kernel TF/s | cuBLAS TF/s | ours/cuBLAS")
for M in (4680, 2340, 1170, 585):
    for (N, K, name) in [(15360, 5120, "qkv"), (5120, 5120, "proj"), (13824, 5120, "ffn1"), (5120, 13824, "ffn2")]:
        a = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
        w = torch.randn(N, K, device=dev, dtype=torch.bfloat16) * 0.02
        b = torch.zeros(N, device=dev, dtype=torch.bfloat16)
        o = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        fl = 2.0 * M * N * K
        ops.stream_k = True
        t_ws = timeit(lambda: ops.gemm(a, w, b, out=o))
        k_ws = lib.kr_gemm_kernel_id_ws(0, M, N, K, 1)
        ops.stream_k = False
        t_no = timeit(lambda: ops.gemm(a, w, b, out=o))
        k_no = lib.kr_gemm_kernel_id_ws(0, M, N, K, 0)
        ops.stream_k = True
        t_cb = timeit(lambda: torch.nn.functional.linear(a, w, b))
        print(f"{name:5s} {M:5d}x{N:5d}x{K:5d} | {names[k_ws]:8s} {fl / t_ws / 1e9:7.1f} | {names[k_no]:8s} {fl / t_no / 1e9:7.1f} | "
              f"{fl / t_cb / 1e9:7.1f} | {t_cb / t_ws:5.3f}", flush=True)
