"""Frame-tiled VAE stages on the H100 at 1280x720: tiled and untiled decode / encode are bit-identical, and the 14B
long-form session (kv_cache_num_frames=5) fits on one 80 GB card."""
import gc
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _decode_blocks(quant, tile, zs):
    from realtime_video_b200.factory import synthetic_vae_decoder
    m = synthetic_vae_decoder(device="cuda")
    m.quant = quant
    m.engine._tile_override = tile
    cache, outs = [None] * 55, []
    with torch.no_grad():
        for z in zs:
            px, cache = m(z, *cache)
            outs.append(px.cpu())
    tile_used = m.engine.frame_tile
    del m, cache
    torch.cuda.empty_cache()
    return outs, tile_used


@pytest.mark.parametrize("quant", [None, "fp8"], ids=["fp16", "fp8"])
def test_720p_tiled_decode_is_bit_identical_to_untiled(quant):
    gen = torch.Generator(device="cuda").manual_seed(0)
    zs = [torch.randn(1, 3, 16, 90, 160, generator=gen, device="cuda").half() for _ in range(3)]
    got, tile = _decode_blocks(quant, None, zs)
    want, untiled = _decode_blocks(quant, 12, zs)
    assert tile < untiled == 12
    assert [p.shape[1] for p in got] == [9, 12, 12]
    for a, b in zip(got, want):
        assert torch.isfinite(a).all() and torch.equal(a, b)


def test_720p_tiled_encode_is_bit_identical_to_untiled():
    from realtime_video_b200.factory import synthetic_vae_encoder
    gen = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(1, 3, 13, 720, 1280, generator=gen, device="cuda").half() * 2 - 1

    def run(tile):
        m = synthetic_vae_encoder(device="cuda")
        with torch.no_grad():
            m(x[:, :, :1], [None] * 55)                          # builds the engine
            m._engine._tile_override = tile
            cold, cache = m(x[:, :, :9], [None] * 55)            # 1 + 4 + 4 frames on a fresh cache
            warm, _ = m(x[:, :, 9:], cache, stream=True)         # a 4-frame webcam chunk
            one, _ = m(x[:, :, 12:13], [None] * 55)              # the one-frame re-encode
        t = m._engine.frame_tile
        del m, cache
        torch.cuda.empty_cache()
        return [cold.cpu(), warm.cpu(), one.cpu()], t

    got, tile = run(None)
    want, untiled = run(4)
    assert tile < untiled == 4
    for a, b in zip(got, want):
        assert torch.isfinite(a).all() and torch.equal(a, b)


def test_720p_long_form_session_fits_one_80gb_card():
    """Five blocks of the 14B session at 1280x720, kv_cache_num_frames=5, in a child process (nothing else on the
    card counts): blocks 3 and 4 re-encode their first context frame after the window slides."""
    free, total = torch.cuda.mem_get_info()
    if total < 79 * 2**30:
        pytest.skip("needs an 80 GB card")
    # this process's caching allocator still reserves what earlier GPU tests freed (several GiB after the 720p
    # geometry tests): hand it back to the driver so that the child gets the card
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    here = (f"this process: {torch.cuda.memory_allocated() / 2**30:.2f} GiB allocated, "
            f"{torch.cuda.memory_reserved() / 2**30:.2f} GiB reserved; card free before the child {free / 2**30:.2f} GiB")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_720p.py"), "--blocks", "5"], cwd=ROOT,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{here}\n{r.stderr[-4000:]}"
    line = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps(line))
    assert line["finite"] and line["steady_blocks"] == 2
    assert line["max_memory_allocated_gib"] <= 74.0, line
