"""GPU parity of the wgmma attention kernel (kr_attn_fwd through the C ABI) against the float64 restatement
``kernel_refs.attention`` of flash_attn_func / the FlexAttention block mask (wan/modules/attention.py:65-70,
wan/modules/causal_model.py:134-138, 316-348), including the zero keys the recompute branch pads with (``pad_keys``).

The kernel runs one CTA per 128 query rows of one head: a TMA producer warpgroup streams 128-key K / V tiles through
a 4-stage ring, and two consumer warpgroups (64 query rows each) compute S = Q K^T with wgmma, mask it, run the online
softmax with lazy rescaling (O is rescaled only when the row maximum grows by more than 2^8), and accumulate P V with
P in registers.  Tiles past the block end are not visited, tiles below a local window are masked whole (m stays -inf),
and the padded keys are added to the softmax denominator in the epilogue.

Floating point, 16-bit inputs: P is rounded to 16 bits before P V, like FlashAttention-2, and O is rounded on the
store.  Tolerances: rel-L2 over the whole output <= 1e-2 (observed ~2.3e-3), and the relative L2 error of every
(row, head) 128-vector <= 8e-3 (measured max on an H100: 4.0e-3; the bound keeps a 2x margin), so one wrong head of
one row, an off-by-one in the padded-key count or at the window's lower edge fails.  Exact invariances (views, head
slices, masks that hide nothing) are checked with ``torch.equal``.  These checks hold for any correct schedule; the
element-wise check against a restatement of this kernel's own schedule is tests/test_attn_parity_gpu.py."""
import math

import pytest
import torch

from tests import kernel_refs as R

pytestmark = pytest.mark.gpu
TOL = 1e-2
PER_VECTOR_TOL = 8e-3


def attn_ref(q, k, v, heads, block_len=0, window=0, pad_keys=0, softmax_scale=None):
    return R.attention(q, k, v, heads, block_len, window, pad_keys, softmax_scale)


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


def _check(out, ref, heads, what=""):
    r = rel(out, ref)
    per = R.rel_rows_heads(out, ref, heads)
    worst = float(per.max())
    assert torch.isfinite(out).all()
    assert r < TOL and worst < PER_VECTOR_TOL, (what, r, worst, divmod(int(per.argmax()), heads))
    print(f"attention {what}: rel-L2 {r:.2e}, worst (row, head) {worst:.2e}")
    return worst


def _qkv(Lq, Lkv, heads, seed, dtype=torch.bfloat16, kind="randn"):
    g = torch.Generator(device="cuda").manual_seed(seed)
    D = heads * 128
    q = torch.randn(Lq, D, device="cuda", generator=g)
    k = torch.randn(Lkv, D, device="cuda", generator=g)
    v = torch.randn(Lkv, D, device="cuda", generator=g)
    if kind == "negative":
        # every real score ~ -4: the padded keys (score 0) carry a large share of each softmax row
        q, k = q.abs() * 0.75, -k.abs() * 0.75
    return q.to(dtype), k.to(dtype), v.to(dtype)


@pytest.mark.parametrize("Lq,Lkv,heads,block_len,window", [
    (128, 128, 2, 0, 0), (300, 500, 2, 0, 0), (720, 1440, 3, 0, 0), (333, 77, 2, 0, 0),
    (100, 900, 1, 0, 0),
    (720, 720, 2, 240, 0), (1200, 1200, 2, 480, 0), (1200, 1200, 2, 240, 480),
    (1, 1, 2, 0, 0), (1, 15, 2, 0, 0), (1, 129, 2, 0, 0), (129, 1, 2, 0, 0), (129, 15, 2, 0, 0),
    (129, 129, 2, 0, 0), (4680, 1, 2, 0, 0), (4680, 15, 2, 0, 0), (4680, 129, 2, 0, 0),
])
def test_attention_matches_fp32_reference(Lq, Lkv, heads, block_len, window):
    from realtime_video_b200 import ops
    q, k, v = _qkv(Lq, Lkv, heads, Lq * 7 + Lkv)
    out = torch.empty(Lq, heads * 128, device="cuda", dtype=torch.bfloat16)
    ops.attention(q, k, v, heads=heads, out=out, block_len=block_len, window=window)
    _check(out, attn_ref(q, k, v, heads, block_len, window), heads, f"{Lq}x{Lkv} bl {block_len} w {window}")


# recompute-branch shapes: L rows attend the first L keys block-causally, the keys padded with zeros up to a multiple
# of 128.  The padded keys are visible to the queries whose block end lies past L: min(end - L, pad) of them.
@pytest.mark.parametrize("L,block_len,window,kind", [
    (250, 84, 0, "negative"),       # last block end 252: 2 of the 6 padded keys visible
    (250, 84, 168, "negative"),     # ... with a 2-block window
    (480, 288, 0, "randn"),         # 5 frames of 96, blocks of 3 frames: 32 padded keys visible to frames 3-4
    (480, 288, 0, "negative"),
    (480, 288, 576, "negative"),    # window of 2 blocks: no key masked below
    (1200, 240, 480, "randn"),      # lower window edges 0, 0, 240, 480, 720: inside 128-key tiles
    (1560, 480, 480, "randn"),      # window of one block: rows of block 3 skip tiles 0-10 whole (m = -inf path)
    (4680, 1560 * 2, 1560 * 2, "negative"),   # bench frame length, block 2 frames: 3120 + 3120 > 4680 -> 56 padded keys
])
def test_attention_padded_keys_and_window(L, block_len, window, kind):
    from realtime_video_b200 import ops
    heads = 2
    pad = math.ceil(L / 128) * 128 - L
    q, k, v = _qkv(L, L, heads, L + block_len + window, kind=kind)
    out = ops.attention(q, k, v, heads=heads, block_len=block_len, window=window, pad_keys=pad)
    _check(out, attn_ref(q, k, v, heads, block_len, window, pad), heads,
           f"L {L} bl {block_len} w {window} pad {pad} {kind}")


def test_window_lower_edge_key_is_counted():
    """The key at each block's window lower edge (end - window) gets a score far above all others, so each row's
    output is essentially that key's value: dropping the edge key (an off-by-one at the window's lower edge) or
    admitting the key below it changes the whole row."""
    from realtime_video_b200 import ops
    heads, L, bl, window = 2, 1200, 240, 480
    q, k, v = _qkv(L, L, heads, 3)
    q = q.float().abs().bfloat16()
    k = k.float() * 0.1
    for end in range(bl, L + 1, bl):
        lo = end - window
        if lo > 0:
            k[lo] = 1.0            # q >= 0, so q . k[lo] >> q . k[j]
            k[lo - 1] = 1.0        # the key just below the edge is masked and must stay out
            v[lo - 1] = 50.0
    k = k.bfloat16()
    out = ops.attention(q, k, v, heads=heads, block_len=bl, window=window)
    _check(out, attn_ref(q, k, v, heads, bl, window), heads, "window edge")


@pytest.mark.parametrize("Lq", [100, 256, 384, 700])
def test_growing_scores_exercise_the_lazy_rescale(Lq):
    """Keys are scaled up along the sequence so the running row maximum jumps by far more than the 2^8 rescale
    threshold from one 128-key tile to the next: O is rescaled in registers between P.V accumulations."""
    from realtime_video_b200 import ops
    torch.manual_seed(5)
    heads, Lkv = 2, 1300
    D = heads * 128
    q = torch.randn(Lq, D, device="cuda").abs().bfloat16()            # positive q . positive k -> monotone growth
    ramp = (1.0 + 10.0 * torch.arange(Lkv, device="cuda") / Lkv)[:, None]
    k = (torch.randn(Lkv, D, device="cuda").abs() * ramp).bfloat16()
    v = torch.randn(Lkv, D, device="cuda").bfloat16()
    out = torch.empty(Lq, D, device="cuda", dtype=torch.bfloat16)
    ref = attn_ref(q, k, v, heads)
    for _ in range(3):                                                   # repeat: a race would be intermittent
        ops.attention(q, k, v, heads=heads, out=out)
        _check(out, ref, heads, f"lazy rescale {Lq}")


def test_fp16_inputs():
    from realtime_video_b200 import ops
    q, k, v = _qkv(384, 640, 2, 9, dtype=torch.float16)
    out = torch.empty(384, 256, device="cuda", dtype=torch.float16)
    ops.attention(q, k, v, heads=2, out=out)
    _check(out, attn_ref(q, k, v, 2), 2, "fp16")


def test_fp16_inputs_with_mask():
    """fp16 with the block-causal mask, a 2-block window and the padded keys (700 rows: 68 padded keys, 20 of them
    visible to the last block)."""
    from realtime_video_b200 import ops
    L, bl = 700, 240
    pad = math.ceil(L / 128) * 128 - L
    q, k, v = _qkv(L, L, 2, 19, dtype=torch.float16, kind="negative")
    out = ops.attention(q, k, v, heads=2, block_len=bl, window=2 * bl, pad_keys=pad)
    _check(out, attn_ref(q, k, v, 2, bl, 2 * bl, pad), 2, "fp16 masked")


def test_softmax_scale():
    from realtime_video_b200 import ops
    q, k, v = _qkv(300, 700, 2, 13)
    out = ops.attention(q, k, v, heads=2, softmax_scale=0.25)
    _check(out, attn_ref(q, k, v, 2, softmax_scale=0.25), 2, "scale 0.25")


# ---------------------------------------------------------------------------------------------
# exact invariances
# ---------------------------------------------------------------------------------------------
def test_strided_views_give_the_same_bits():
    """K / V as the row-offset cache view cache[lo:hi] (lo % 128 != 0), Q with a row pitch > heads*128 and out as a
    column slice of a wider buffer give the same bits as contiguous copies; out columns outside the slice and the
    rows around it are untouched."""
    from realtime_video_b200 import ops
    heads, Lq, Lkv, lo = 2, 300, 700, 77
    D = heads * 128
    qb = torch.randn(Lq, D + 64, device="cuda").bfloat16()
    kc = torch.randn(lo + Lkv + 50, D, device="cuda").bfloat16()
    vc = torch.randn(lo + Lkv + 50, D, device="cuda").bfloat16()
    q, k, v = qb[:, 32:32 + D], kc[lo:lo + Lkv], vc[lo:lo + Lkv]
    ob = torch.full((Lq + 2, D + 256), -3.0, device="cuda").bfloat16()
    o = ob[1:1 + Lq, 128:128 + D]
    ops.attention(q, k, v, heads=heads, out=o)
    want = ops.attention(q.contiguous(), k.contiguous(), v.contiguous(), heads=heads)
    assert torch.equal(o, want)
    mask = torch.ones_like(ob, dtype=torch.bool)
    mask[1:1 + Lq, 128:128 + D] = False
    assert bool((ob[mask] == -3.0).all())


def test_one_head_equals_head_slice():
    """A one-head call on head h's columns (row pitch of the whole tensor) equals head h of the multi-head call."""
    from realtime_video_b200 import ops
    heads = 3
    q, k, v = _qkv(500, 900, heads, 21)
    full = ops.attention(q, k, v, heads=heads)
    for h in range(heads):
        cs = slice(h * 128, (h + 1) * 128)
        assert torch.equal(ops.attention(q[:, cs], k[:, cs], v[:, cs], heads=1), full[:, cs]), h


def test_masks_that_hide_nothing_are_the_unmasked_call():
    """block_len >= Lkv with pad_keys = 0 equals no mask, and a window >= the block end equals no window."""
    from realtime_video_b200 import ops
    q, k, v = _qkv(600, 600, 2, 31)
    plain = ops.attention(q, k, v, heads=2)
    assert torch.equal(ops.attention(q, k, v, heads=2, block_len=600), plain)
    assert torch.equal(ops.attention(q, k, v, heads=2, block_len=1000), plain)
    masked = ops.attention(q, k, v, heads=2, block_len=200)
    assert torch.equal(ops.attention(q, k, v, heads=2, block_len=200, window=600), masked)
    assert torch.equal(ops.attention(q, k, v, heads=2, block_len=200, window=5000), masked)
