"""kr_dit_block_fwd on the GPU: one C-ABI call per DiT block must reproduce the per-op schedule BIT FOR BIT (it issues
the same launches with the same arguments — tests/test_block_fwd_cpu.py proves that on the host; this is the live
check), on the golden 2-layer model through cache, later-block and recompute passes, and on one 14B-width layer."""
import pytest
import torch

from tests import test_dit_gpu as T
from tests.golden_io import load_npz

pytestmark = pytest.mark.gpu
FS = 96


def run_sequence(m, g, one_call: bool):
    m.use_block_fwd = one_call
    for blk in m.blocks:
        blk.self_attn.fuse_projections()
    kv, ca = T.caches(m, 6 * FS)
    outs = [T.fwd(m, g, "in/x0", 1000, kv, ca, 0),            # first pass of the prompt: per-op on both sides
            T.fwd(m, g, "in/x1", 750, kv, ca, 0),             # warm prompt cache: the one-call path engages
            T.fwd(m, g, "in/x2", 1000, kv, ca, 3 * FS)]
    m.block_mask = m._prepare_blockwise_causal_attn_mask("cuda", num_frames=3, frame_seqlen=FS, num_frame_per_block=3,
                                                         local_attn_size=-1)
    for c in kv:
        c["global_end_index"] = c["local_end_index"] = 0
    outs.append(T.fwd(m, g, "in/x3", 0, kv, ca, 3 * FS))      # recompute branch
    m.block_mask = None
    outs.append(T.fwd(m, g, "in/x4", 1000, kv, ca, 3 * FS))
    return outs, kv


def test_one_call_per_block_is_bit_identical_to_the_per_op_schedule():
    from realtime_video_b200 import ops
    g = load_npz("dit_small.npz")
    ref, kv_ref = run_sequence(T.build(g), g, one_call=False)
    n0 = ops.launch_count
    got, kv_got = run_sequence(T.build(g), g, one_call=True)
    assert ops.launch_count - n0 > 0
    for i, (a, b) in enumerate(zip(got, ref)):
        assert torch.equal(a, b), f"pass {i} differs"
    for a, b in zip(kv_got, kv_ref):
        assert torch.equal(a["k"], b["k"]) and torch.equal(a["v"], b["v"])
        assert (a["global_end_index"], a["local_end_index"]) == (b["global_end_index"], b["local_end_index"])


def test_one_call_engages_and_matches_at_14b_width():
    """d 5120 / 40 heads / ffn 13824, 3 frames of 1560 tokens against a 6-frame cache: the bench's block shape."""
    from realtime_video_b200.dit import CausalWanModel
    torch.manual_seed(3)
    with torch.device("cuda"):                    # initialise on the device like tests/test_real_geometry_gpu.py
        m = CausalWanModel(dim=5120, ffn_dim=13824, num_heads=40, num_layers=1)
    m = m.to(dtype=torch.bfloat16).eval()
    m.blocks[0].self_attn.fuse_projections()
    blk = m.blocks[0]
    fs, L, D = 1560, 4680, 5120
    x0 = torch.randn(L, D, device="cuda").bfloat16()
    e0 = (torch.randn(3, 6, D, device="cuda") * 0.1).bfloat16()
    outs = []
    for one_call in (False, True):
        m.use_block_fwd = one_call
        kv = {"k": torch.randn(1, 6 * fs, 40, 128, device="cuda").bfloat16(),
              "v": torch.randn(1, 6 * fs, 40, 128, device="cuda").bfloat16(), "global_end_index": L, "local_end_index": L}
        torch.manual_seed(4)
        kv["k"].normal_(); kv["v"].normal_()
        ca = {"k": torch.randn(1, 512, 40, 128, device="cuda", generator=torch.Generator("cuda").manual_seed(5)).bfloat16(),
              "v": torch.randn(1, 512, 40, 128, device="cuda", generator=torch.Generator("cuda").manual_seed(6)).bfloat16(),
              "is_init": True}
        x = x0.clone()
        assert m._block_fwd_eligible(blk, x, ca)
        with torch.no_grad():
            m._block(blk, x, e0, (3, 30, 52), None, kv, ca, L, None)
        outs.append((x, kv["k"].clone(), kv["v"].clone()))
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    assert torch.isfinite(outs[1][0].float()).all()
