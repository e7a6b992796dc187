"""UMT5-XXL encoder (24 layers, dim 4096, 64 heads, ffn 10240, L = 512) on one GPU: time per prompt, kernel split.
    python tools/time_t5.py"""
import sys

import torch

sys.path.insert(0, ".")
from realtime_video_b200 import ops  # noqa: E402
from realtime_video_b200.t5 import umt5_xxl_encoder  # noqa: E402

torch.manual_seed(0)
m = umt5_xxl_encoder(device="cuda", dtype=torch.bfloat16, vocab=32128)     # full width / depth, smaller vocabulary table
with torch.no_grad():
    for p in m.parameters():
        if p.dim() == 2:
            p.normal_(std=0.02)
ids = torch.randint(0, 32128, (1, 512), device="cuda")
mask = torch.zeros(1, 512, dtype=torch.long, device="cuda")
mask[:, :60] = 1
for _ in range(3):
    y = m(ids, mask)
torch.cuda.synchronize()
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
n0 = ops.launch_count
s.record()
for _ in range(10):
    y = m(ids, mask)
e.record()
torch.cuda.synchronize()
ms = s.elapsed_time(e) / 10
launches = (ops.launch_count - n0) // 10
L, d, f, h = 512, 4096, 10240, 64
flops = 24 * (2 * L * d * d * 4 + 2 * L * d * f * 3 + 4 * L * L * d)
print(f"UMT5-XXL encoder, L=512, bf16: {ms:.2f} ms per prompt, {launches} launches, {flops / 1e12:.2f} TFLOP -> "
      f"{flops / ms / 1e9:.0f} TF/s; finite={bool(torch.isfinite(y).all())}")
ops.profile_begin()
y = m(ids, mask)
torch.cuda.synchronize()
for k, v in sorted(ops.profile_end().items()):
    print(f"  {k:28s} {v['n']:4d} launches {v['ms']:8.3f} ms {v['flops'] / max(v['ms'], 1e-9) / 1e9:8.0f} TF/s")
