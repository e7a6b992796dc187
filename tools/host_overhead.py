"""Host time per DiT block with the kernel launchers stubbed out (no GPU needed): the per-op Python schedule (14 ctypes
calls + temporaries) against ONE kr_dit_block_fwd call.  Builds the launch recorder of tests/kr_record_stubs.cu (the real
kr_api.cu / kr_dit_block.cu / kr_host.cu linked against recording stand-ins) and times both paths on this machine's CPU.
    python tools/host_overhead.py"""
import ctypes
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from realtime_video_b200 import _lib, ops  # noqa: E402

CSRC = ROOT / "realtime_video_b200" / "csrc"
so = Path(tempfile.mkdtemp()) / "libkrea_record.so"
nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
subprocess.run([nvcc, "-std=c++17", "-O2", "-shared", "-Xcompiler", "-fPIC", "-cudart", "static",
                "-Wno-deprecated-gpu-targets", str(CSRC / "kr_host.cu"), str(CSRC / "kr_api.cu"),
                str(CSRC / "kr_dit_block.cu"), str(ROOT / "tests" / "kr_record_stubs.cu"), "-o", str(so)], check=True)
lib = ctypes.CDLL(str(so))
for name, argtypes in _lib.SIGNATURES.items():
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = ctypes.c_int, argtypes
lib.kr_dit_block_workspace_bytes.restype = ctypes.c_size_t
lib.kr_dit_block_workspace_bytes.argtypes = [ctypes.c_int] * 4
lib.kr_gemm_workspace_bytes.restype = ctypes.c_size_t
lib.kr_last_error.restype = ctypes.c_char_p
ops._lib.load = lambda: lib
ops._req = lambda t, name, dtype=None: None
ops._stream = lambda: 0
ops.stream_k = False

from realtime_video_b200.dit import CausalWanModel  # noqa: E402

m = CausalWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=1, text_dim=128).to(torch.bfloat16).eval()
blk = m.blocks[0]
blk.self_attn.fuse_projections()
FS = 32
x, e0 = torch.randn(3 * FS, 256).bfloat16(), torch.randn(3, 6, 256).bfloat16()
kv = {"k": torch.zeros(1, 6 * FS, 2, 128, dtype=torch.bfloat16), "v": torch.zeros(1, 6 * FS, 2, 128, dtype=torch.bfloat16)}
ca = {"k": torch.randn(1, 512, 2, 128).bfloat16(), "v": torch.randn(1, 512, 2, 128).bfloat16(), "is_init": True}
print(f"host time per DiT block, kernel launchers stubbed out (cpu: {torch.get_num_threads()} threads, python "
      f"{sys.version.split()[0]}); independent of the tensor sizes")
for one_call in (False, True):
    m.use_block_fwd = one_call
    ts = []
    for _ in range(7):
        t0 = time.perf_counter()
        for _ in range(200):
            kv["global_end_index"] = kv["local_end_index"] = 0
            lib.kr_record_clear()
            with torch.no_grad():
                m._block(blk, x, e0, (3, 4, 8), None, kv, ca, 0, None)
        ts.append((time.perf_counter() - t0) / 200 * 1e6)
    ts.sort()
    print(f"{'one kr_dit_block_fwd call' if one_call else 'per-op schedule (14 calls)':<28} min {ts[0]:7.1f} us   "
          f"median {ts[3]:7.1f} us   -> {ts[3] * 200 / 1e3:6.1f} ms per 200-block step")
