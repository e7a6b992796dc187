"""The 2-CTA cluster GEMM (kr_gemm2.cu: W multicast to both CTAs of a cluster, stage release to both CTAs' barriers)
forced on every N % 256 == 0 shape with KR_GEMM2=2 in a subprocess (the planner reads the switch once per process), at
the bench shapes and an odd row-block count, every epilogue it serves, against an fp32 matmul of the same bf16
operands: rel-L2 <= 2e-3."""
import os
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent

SCRIPT = r'''
import torch
from realtime_video_b200 import _lib, ops
from tests.golden_io import rel_l2
lib = _lib.load()
for M, N, K, epi in [(4680, 5120, 5120, "gate_res"), (4680, 13824, 5120, "gelu"), (4680, 15360, 5120, "bias"),
                     (300, 512, 640, "res")]:
    assert lib.kr_gemm_kernel_id(0, M, N, K) == 2, (M, N, K)
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    ref = a.float() @ w.float().t() + b.float()
    if epi == "bias":
        out, want = ops.gemm(a, w, b), ref
    elif epi == "gelu":
        out = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GELU)
        want = torch.nn.functional.gelu(ref.bfloat16().float(), approximate="tanh")
    elif epi == "res":
        r = torch.randn(M, N, device="cuda").bfloat16()
        out = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_RES, residual=r)
        want = r.float() + ref.bfloat16().float()
    else:
        x = torch.ones(M, N, device="cuda").bfloat16()
        gate = torch.randn(3, N, device="cuda").bfloat16()
        rpg = (M + 2) // 3
        rows = torch.arange(M, device="cuda") // rpg
        want = x.float() + (ref.bfloat16().float() * gate.float()[rows]).bfloat16().float()
        out = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=x, gate=gate, rows_per_gate=rpg, out=x)
    torch.cuda.synchronize()
    r = rel_l2(out.float(), want)
    assert r < 2e-3, (M, N, K, epi, r)
print("cluster GEMM OK")
'''


def test_cluster_gemm_forced_on_every_eligible_shape():
    env = dict(os.environ, KR_GEMM2="2", KR_GEMM_SK="0")
    r = subprocess.run([sys.executable, "-c", SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "cluster GEMM OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
