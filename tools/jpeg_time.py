"""Time the device JPEG egress (kr_frames_to_jpeg) on one 12-frame 832x480 block of decoder-like frames and the
reference's host path (normalise + to_pil_image + Pillow save in a 24-thread pool, release_server.py:945-983) on
the same frames.  Writes out/jpeg_time.json."""
import io
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from realtime_video_b200 import ops  # noqa: E402
from tests.jpeg_cases import frames_fp32  # noqa: E402


def main():
    T, H, W = 12, 480, 832
    x = torch.from_numpy(frames_fp32(T, H, W, seed=1)).cuda()[None]
    out, sizes = ops.frames_to_jpeg(x, 90)
    torch.cuda.synchronize()
    files = ops.jpeg_files(out, sizes)
    jpeg_bytes = sum(len(f) for f in files)
    big = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")          # L2 flush between iterations
    ts = []
    for _ in range(10):
        big.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ops.frames_to_jpeg(x, 90, out=out, sizes=sizes)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    dev_ms = float(np.median(ts))
    # end to end: kernel + sizes + the used bytes to the host
    t0 = time.time()
    for _ in range(5):
        o, s = ops.frames_to_jpeg(x, 90, out=out, sizes=sizes)
        ops.jpeg_files(o, s)
    e2e_ms = (time.time() - t0) / 5 * 1e3
    # reference host path on the same frames
    import torchvision.transforms.functional as TF
    host = torch.empty(x.shape, dtype=torch.float32).pin_memory()
    pool = ThreadPoolExecutor(max_workers=24)

    def ref_once():
        host.copy_(x)
        norm = host.add_(1.0).mul_(0.5).clamp_(0.0, 1.0)

        def enc(i):
            buf = io.BytesIO()
            TF.to_pil_image(norm[0, i], "RGB").save(buf, format="JPEG", quality=90)
            return buf.getvalue()
        return list(pool.map(enc, range(T)))
    ref_files = ref_once()
    t0 = time.time()
    for _ in range(3):
        ref_once()
    ref_ms = (time.time() - t0) / 3 * 1e3
    res = {"frames": T, "height": H, "width": W, "quality": 90, "identical_to_pillow": files == ref_files,
           "jpeg_bytes_per_block": jpeg_bytes, "device_ms_per_block": dev_ms, "device_ms_all": ts,
           "device_e2e_ms_per_block_incl_d2h": e2e_ms, "reference_host_ms_per_block_24_threads": ref_ms,
           "host_cores": os.cpu_count(),
           "algorithmic_bytes": T * 3 * H * W * 4 + jpeg_bytes,
           "achieved_gbs": (T * 3 * H * W * 4 + jpeg_bytes) / (dev_ms * 1e-3) / 1e9}
    Path(ROOT / "out").mkdir(exist_ok=True)
    (ROOT / "out" / "jpeg_time.json").write_text(json.dumps(res))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
