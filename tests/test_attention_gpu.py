"""GPU parity of the wgmma attention kernel (kr_attn_fwd through the C ABI) against an fp32 torch
restatement of flash_attn_func / the FlexAttention block mask (wan/modules/attention.py:65-70,
wan/modules/causal_model.py:134-138, 339-348).  Floating point, bf16 inputs: P is rounded to bf16 before
P.V exactly like FlashAttention-2, so rel-L2 <= 1e-2 (observed 2.3e-3) and the tolerance is in the test.

The shapes are chosen to hit every scheduling mode of the kernel: two-tile CTAs, the single-tile CTA at the
end of a head (Lq % 256 <= 128), ragged Lkv, masked tiles, the local window, and scores that keep growing
along the key axis so the lazy O-rescale path runs on (almost) every tile."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
TOL = 1e-2


def attn_ref(q, k, v, heads, block_len=0, window=0):
    Lq, Lkv = q.shape[0], k.shape[0]
    d = q.shape[1] // heads
    q4 = q.float().view(Lq, heads, d).transpose(0, 1)
    k4 = k.float().view(Lkv, heads, d).transpose(0, 1)
    v4 = v.float().view(Lkv, heads, d).transpose(0, 1)
    s = q4 @ k4.transpose(1, 2) / math.sqrt(d)
    if block_len:
        qi = torch.arange(Lq, device=q.device)[:, None]
        ki = torch.arange(Lkv, device=q.device)[None, :]
        hi = (qi // block_len + 1) * block_len
        ok = ki < hi
        if window:
            ok &= ki >= (hi - window)
        s = s.masked_fill(~ok, float("-inf"))
    return (torch.softmax(s, dim=-1) @ v4).transpose(0, 1).reshape(Lq, heads * d)


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


@pytest.mark.parametrize("Lq,Lkv,heads,block_len,window", [
    (128, 128, 2, 0, 0), (300, 500, 2, 0, 0), (720, 1440, 3, 0, 0), (333, 77, 2, 0, 0),
    (100, 900, 1, 0, 0),                       # single-tile CTA only
    (720, 720, 2, 240, 0), (1200, 1200, 2, 480, 0), (1200, 1200, 2, 240, 480),
])
def test_attention_matches_fp32_reference(Lq, Lkv, heads, block_len, window):
    from realtime_video_b200 import ops
    torch.manual_seed(Lq * 7 + Lkv)
    D = heads * 128
    q = torch.randn(Lq, D, device="cuda").bfloat16()
    k = torch.randn(Lkv, D, device="cuda").bfloat16()
    v = torch.randn(Lkv, D, device="cuda").bfloat16()
    out = torch.empty(Lq, D, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, heads=heads, out=out, block_len=block_len, window=window)
    r = rel(out, attn_ref(q, k, v, heads, block_len, window))
    assert r < TOL, r


@pytest.mark.parametrize("Lq", [100, 256, 384, 700])   # 100/384: last CTA of a head runs the single-tile mode
def test_growing_scores_exercise_the_lazy_rescale(Lq):
    """Keys are scaled up along the sequence so the running row maximum jumps by far more than the
    2^8 rescale threshold from one 128-key tile to the next: O is rescaled in registers while the previous
    tile's P.V must already have retired (the ordering the o_done barrier / issue order guarantee)."""
    from realtime_video_b200 import ops
    torch.manual_seed(5)
    heads, Lkv = 2, 1300
    D = heads * 128
    q = torch.randn(Lq, D, device="cuda").abs().bfloat16()            # positive q . positive k -> monotone growth
    ramp = (1.0 + 10.0 * torch.arange(Lkv, device="cuda") / Lkv)[:, None]
    k = (torch.randn(Lkv, D, device="cuda").abs() * ramp).bfloat16()
    v = torch.randn(Lkv, D, device="cuda").bfloat16()
    out = torch.empty(Lq, D, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):                                                   # repeat: a race would be intermittent
        ops.attention(q, k, v, heads=heads, out=out)
        r = rel(out, attn_ref(q, k, v, heads))
        assert torch.isfinite(out).all() and r < TOL, r


def test_fp16_inputs():
    from realtime_video_b200 import ops
    torch.manual_seed(9)
    q = torch.randn(384, 256, device="cuda").half()
    k = torch.randn(640, 256, device="cuda").half()
    v = torch.randn(640, 256, device="cuda").half()
    out = torch.empty(384, 256, device="cuda", dtype=torch.float16)
    ops.attention(q, k, v, heads=2, out=out)
    assert rel(out, attn_ref(q, k, v, 2)) < TOL
