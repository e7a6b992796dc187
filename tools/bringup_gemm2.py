"""2-CTA cluster GEMM (kr_gemm2.cu) against torch fp32; run with KR_GEMM2=2 to force it on every shape."""
import math
import sys

import torch

sys.path.insert(0, ".")
from realtime_video_b200 import ops  # noqa: E402
from tools.bringup import report, timeit  # noqa: E402

dev = "cuda"
torch.manual_seed(0)
ok = True
for dt in (torch.bfloat16, torch.float16):
    for (M, N, K) in [(256, 256, 64), (128, 256, 128), (300, 512, 256), (4680, 15360, 5120), (4680, 13824, 5120),
                      (77, 768, 192), (1000, 1024, 1000), (4680, 5120, 13824), (585, 5120, 5120)]:
        a = torch.randn(M, K, device=dev, dtype=dt)
        w = torch.randn(N, K, device=dev, dtype=dt) / math.sqrt(K)
        b = torch.randn(N, device=dev, dtype=dt)
        got = ops.gemm(a, w, b)
        torch.cuda.synchronize()
        ok &= report(f"gemm2 bias {dt} {M}x{N}x{K}", got, a.float() @ w.float().t() + b.float(), 6e-3)
M, N, K, F = 720, 1536, 1536, 3
a = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
w = torch.randn(N, K, device=dev, dtype=torch.bfloat16) / math.sqrt(K)
b = torch.randn(N, device=dev, dtype=torch.bfloat16)
res = torch.randn(M, N, device=dev, dtype=torch.bfloat16)
gate = torch.randn(F, 6, N, device=dev, dtype=torch.bfloat16)
y = a.float() @ w.float().t() + b.float()
ok &= report("gemm2 gelu", ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GELU), torch.nn.functional.gelu(y, approximate="tanh"), 8e-3)
ok &= report("gemm2 res", ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_RES, residual=res), res.float() + y, 8e-3)
g = gate[:, 2]
ok &= report("gemm2 gate res", ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=res, gate=g, rows_per_gate=M // F),
             res.float() + y * g.float().repeat_interleave(M // F, dim=0), 8e-3)
o1 = torch.empty(M, 1024, device=dev, dtype=torch.bfloat16); o2 = torch.empty(M + 5, 512, device=dev, dtype=torch.bfloat16)
ops.gemm(a, w, b, out=o1, out2=o2[5:], n_split=1024)
ok &= report("gemm2 split lo", o1, y[:, :1024], 6e-3)
ok &= report("gemm2 split hi", o2[5:], y[:, 1024:], 6e-3)
print("GEMM2", "PASS" if ok else "FAIL", flush=True)
L, D, FF = 4680, 5120, 13824
for (N, K, name) in [(15360, D, "qkv"), (FF, D, "ffn1"), (D, D, "proj"), (D, FF, "ffn2")]:
    a = torch.randn(L, K, device=dev, dtype=torch.bfloat16)
    w = torch.randn(N, K, device=dev, dtype=torch.bfloat16) * 0.02
    b = torch.zeros(N, device=dev, dtype=torch.bfloat16)
    o = torch.empty(L, N, device=dev, dtype=torch.bfloat16)
    ms = timeit(lambda: ops.gemm(a, w, b, out=o), n=20)
    ms_t = timeit(lambda: torch.nn.functional.linear(a, w, b), n=20)
    fl = 2.0 * L * N * K
    print(f"PERF gemm {name} {L}x{N}x{K}: {ms:.3f} ms {fl / ms / 1e9:.1f} TF/s | cuBLAS {ms_t:.3f} ms {fl / ms_t / 1e9:.1f} TF/s", flush=True)
