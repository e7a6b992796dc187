"""The 16-bit GEMM epilogues run on the epilogue warps (KR_GEMM_EPI_WARPS=1, the default: consumers write
rnd16(acc + bias) to a shared C buffer, warps 9..11 apply the rest) against the in-register epilogue
(KR_GEMM_EPI_WARPS=0), each in a subprocess since the library reads the switch once per process.  The arithmetic and
its order are the same, so the outputs must be equal bit for bit: bf16 and fp16, every 16-bit epilogue, the fixed
widths 32 / 64 / 128 / 256 and the runtime widths 96..224 the planner picks (some with a narrower last column tile;
it never picks 256 there, which is the fixed-width tile), M in {4680, 1170, 200, 1}, the split output into a strided
cache slot, the in-place residual and a per-frame gate with a row offset."""
import os
import subprocess
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent

SCRIPT = r'''
import hashlib
import sys
import torch
from realtime_video_b200 import _lib, ops
lib = _lib.load()
ops.stream_k = False
E = ops
EPIS = [E.EPI_BIAS, E.EPI_BIAS_GELU, E.EPI_BIAS_GATE_RES, E.EPI_BIAS_RES, E.EPI_MUL]
# (M, N, K, kernel id): fixed widths at K = 256 (the runtime-width planner needs K >= 512); at M = 4680 N = 1280 / 640 /
# 320 / 352 take the 256 / 128 / 64 / 32 tiles, at smaller M the dispatch narrows them.  The K = 512 shapes are the
# planner's runtime widths on 132 SMs: 160 (N = 1024, last tile 64 wide), 192 (N = 512, last 128), 224 (N = 1536,
# last 192), 128 (N = 4096) at M = 4680; 96 (N = 512, last 32) and 224 (N = 2560, last 96) at M = 1170.
SHAPES = [(4680, 1280, 256, 1), (4680, 640, 256, 1), (4680, 320, 256, 1), (4680, 352, 256, 1),
          (1170, 1280, 256, 1), (200, 1280, 256, 1), (1, 1280, 256, 1), (200, 352, 256, 1),
          (4680, 1024, 512, 4), (4680, 512, 512, 4), (4680, 1536, 512, 4), (4680, 4096, 512, 4),
          (1170, 512, 512, 4), (1170, 2560, 512, 4), (200, 512, 512, 4), (1, 512, 512, 4)]
outs = []
for dt in (torch.bfloat16, torch.float16):
    for M, N, K, kid in SHAPES:
        assert lib.kr_gemm_kernel_id_ws(0, M, N, K, 0) == kid, (M, N, K)
        g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
        a = torch.randn(M, K, device="cuda", generator=g).to(dt)
        w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).to(dt)
        b = torch.randn(N, device="cuda", generator=g).to(dt)
        res = torch.randn(M, N, device="cuda", generator=g).to(dt)
        rpg, r0 = max(1, (M + 2) // 3), 37
        gate = torch.randn((M + r0) // rpg + 1, N, device="cuda", generator=g).to(dt)
        for epi in EPIS:
            if epi == E.EPI_BIAS_GATE_RES:
                x = res.clone()   # in place, as the DiT block updates its residual stream
                ops.gemm(a, w, b, epilogue=epi, residual=x, gate=gate, rows_per_gate=rpg, out=x, row_offset=r0)
                outs.append(x)
            elif epi == E.EPI_BIAS_RES:
                x = res.clone()
                ops.gemm(a, w, b, epilogue=epi, residual=x, out=x)
                outs.append(x)
            elif epi == E.EPI_MUL:
                outs.append(ops.gemm(a, w, None, epilogue=epi, residual=res))
            else:
                outs.append(ops.gemm(a, w, b, epilogue=epi))
        outs.append(ops.gemm(a, w, None))
        # split output: columns >= n_split into a row slice of a wider cache
        ns = 1024 if kid == 1 and N > 1024 else (N // 2 // 32 * 32 if kid == 4 else 0)
        if ns:
            lo = torch.empty(M, ns, device="cuda", dtype=dt)
            cache = torch.zeros(M + 64, N - ns + 64, device="cuda", dtype=dt)
            ops.gemm(a, w, b, out=lo, out2=cache[32:32 + M, :N - ns], n_split=ns)
            outs += [lo, cache]
torch.cuda.synchronize()
with open(sys.argv[1], "w") as f:
    for o in outs:
        f.write(f"{tuple(o.shape)} {o.dtype} {hashlib.sha256(o.cpu().view(torch.int16).numpy().tobytes()).hexdigest()}\n")
print("epi outputs", len(outs))
'''


def _run(arm: str, path: Path):
    env = dict(os.environ, KR_GEMM_EPI_WARPS=arm, KR_GEMM2="0", KR_GEMM_SK="0")
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(path)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and "epi outputs" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
    return path.read_text().splitlines()


def test_epilogue_warps_bit_identical_to_register_epilogue(tmp_path):
    # one line per output: shape, dtype and the SHA-256 of its bits
    new, old = _run("1", tmp_path / "new.txt"), _run("0", tmp_path / "old.txt")
    assert len(new) == len(old) > 0
    bad = [i for i, (x, y) in enumerate(zip(new, old)) if x != y]
    assert not bad, [(i, new[i], old[i]) for i in bad[:8]]
