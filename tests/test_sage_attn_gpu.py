"""Quantised attention tier on the H100: kr_sage_quantize bit-exact against the oracle's quantisation, kr_sage_attn
against the oracle's attention on the kernel's own buffers, end to end against exact fp32 attention, determinism
(including CUDA-graph replay of the server loop), and the model-level tolerance of ``attn_quant="sage"``."""

import pytest
import torch

from oracle import sage_oracle as so
from tests.golden_io import ReplayRandn, load_npz, rel_l2, weights

pytestmark = pytest.mark.gpu

# (Lq, Lkv, heads, ld of the K/V cache, first K/V row)
SHAPES = [
    (4680, 9360, 40, 5120, 0),       # cache branch of the bench shape
    (4680, 512, 40, 5120, 0),        # cross-attention over the prompt
    (100, 1, 2, 256, 0),             # tails
    (100, 127, 2, 256, 0),
    (100, 129, 2, 256, 0),
    (100, 200, 2, 256, 0),
    (1560, 3120, 8, 5120, 1560),     # K/V views into a wider cache, starting at a non-zero row
    (4680, 9360, 5, 640, 0),         # sequence-parallel width: 5 heads per rank
]
IDS = [f"{a}x{b}x{c}_ld{d}_r{e}" for a, b, c, d, e in SHAPES]


def _inputs(Lq, Lkv, heads, ld, row0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = heads * 128
    q = torch.randn(Lq, W, device="cuda", generator=g).bfloat16()
    kc = torch.randn(row0 + Lkv, ld, device="cuda", generator=g)
    vc = torch.randn(row0 + Lkv, ld, device="cuda", generator=g)
    kc += torch.randn(ld, device="cuda", generator=g) * 2      # per-channel key offsets: what smoothing removes
    vc += torch.randn(ld, device="cuda", generator=g) * 0.5
    return q, kc.bfloat16()[row0:row0 + Lkv, :W], vc.bfloat16()[row0:row0 + Lkv, :W]


def _ordered_bits(x):
    u = x.view(torch.int16).int() & 0xFFFF
    return torch.where(u >= 0x8000, -(u & 0x7FFF), u)


@pytest.mark.parametrize("Lq,Lkv,heads,ld,row0", SHAPES, ids=IDS)
def test_quantizer_is_bit_exact_against_the_oracle(Lq, Lkv, heads, ld, row0):
    from realtime_video_b200 import ops
    q, k, v = _inputs(Lq, Lkv, heads, ld, row0)
    b = ops.sage_quantize(q, k, v, heads=heads)
    torch.cuda.synchronize()
    # k_mean: fixed-order fp32 sum on the device vs the fp64 mean, both rounded to bf16
    want_mean = so.k_mean_of(k)
    d = (_ordered_bits(b["k_mean"]) - _ordered_bits(want_mean)).abs()
    assert int(d.max()) <= 1 and float((d == 0).float().mean()) >= 0.999
    ref = so.quantize(q, k, v, heads, k_mean=b["k_mean"])
    for name in ("q_i8", "q_scale", "k_i8", "k_scale", "v_t8", "v_scale"):
        assert b[name].shape == ref[name].shape, name
        assert torch.equal(b[name], ref[name]), (name, int((b[name] != ref[name]).sum()))
    assert int(so.unpermute_keys(b["v_t8"])[:, Lkv:].sum()) == 0       # padded keys


@pytest.mark.parametrize("Lq,Lkv,heads,ld,row0", SHAPES, ids=IDS)
def test_kernel_matches_the_oracle_and_tracks_exact_attention(Lq, Lkv, heads, ld, row0):
    from realtime_video_b200 import ops
    q, k, v = _inputs(Lq, Lkv, heads, ld, row0, seed=1)
    out = ops.sage_attention(q, k, v, heads=heads)
    torch.cuda.synchronize()
    b = ops._sage_scratch[(q.device.index, Lq, Lkv, heads)]
    want = so.attention_from_quantized(b, Lq, Lkv, heads)
    r_oracle = rel_l2(out.float(), want.float())
    assert torch.isfinite(out.float()).all() and r_oracle <= 3e-3, r_oracle
    exact = so.exact_attention(q, k, v, heads)
    gap = rel_l2(so.sage_attention(q, k, v, heads).float(), exact)          # the oracle's own quantisation error
    r = rel_l2(out.float(), exact)
    cos = float(torch.nn.functional.cosine_similarity(out.double().flatten(), exact.double().flatten(), 0))
    print(f"sage {Lq}x{Lkv}x{heads}: vs oracle {r_oracle:.2e}, vs exact {r:.3e} (oracle {gap:.3e}), cos {cos:.5f}")
    assert r <= 1.1 * gap + 2e-3 and cos >= 0.998, (r, gap, cos)


def test_same_inputs_give_the_same_bytes():
    from realtime_video_b200 import ops
    q, k, v = _inputs(4680, 9360, 40, 5120, 0, seed=2)
    a = ops.sage_attention(q, k, v, heads=40).clone()
    qa = {n: t.clone() for n, t in ops._sage_scratch[(0, 4680, 9360, 40)].items()}
    b = ops.sage_attention(q, k, v, heads=40)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    for n, t in ops._sage_scratch[(0, 4680, 9360, 40)].items():
        assert torch.equal(t, qa[n]), n


def _layer_14b():
    from realtime_video_b200.dit import CausalWanModel
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = CausalWanModel(num_layers=1, dim=5120, ffn_dim=13824, num_heads=40, text_dim=4096)
    with torch.no_grad():
        m.head.head.weight.normal_(std=0.02)
    m = m.to(torch.bfloat16).eval()
    m.blocks[0].self_attn.fuse_projections()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 60, 104, generator=g).bfloat16().cuda()
    ctx = torch.randn(40, 4096, generator=g).bfloat16().cuda()

    def run():
        kv = [dict(k=torch.zeros(1, 4680, 40, 128, dtype=torch.bfloat16, device="cuda"),
                   v=torch.zeros(1, 4680, 40, 128, dtype=torch.bfloat16, device="cuda"), global_end_index=0,
                   local_end_index=0)]
        ca = [dict(k=torch.zeros(1, 512, 40, 128, dtype=torch.bfloat16, device="cuda"),
                   v=torch.zeros(1, 512, 40, 128, dtype=torch.bfloat16, device="cuda"), is_init=False)]
        with torch.no_grad():
            return m(x[None], t=torch.full((1, 3), 750.0, device="cuda"), context=ctx[None], seq_len=32760,
                     kv_cache=kv, crossattn_cache=ca, current_start=0)[0].float()
    return m, run


def test_sage_layer_vs_bf16_layer_at_14b_dims():
    """One Wan-14B-dim layer, Lq 4680: the quantised attention tier against the bf16 path, alone and together with the
    FP8 linears."""
    from realtime_video_b200 import fp8
    m, run = _layer_14b()
    ref = run()
    m.attn_quant = "sage"
    got = run()
    r = rel_l2(got, ref)
    fp8.quantize_(m)
    got8 = run()
    r8 = rel_l2(got8, ref)
    print(f"14B-dim layer: sage vs bf16 rel-L2 {r:.3e}; sage + fp8 linears vs bf16 {r8:.3e}")
    assert torch.isfinite(got).all() and r <= 8e-2, r
    assert torch.isfinite(got8).all() and r8 <= 8e-2, r8


def _server_models(sage: bool, graphs: bool = False):
    from realtime_video_b200.factory import synthetic_vae_params
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEEncoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    gd = load_npz("dit_small.npz")
    tr = WanDiffusionWrapper(model_name="synthetic", timestep_shift=5.0, is_causal=True,
                             model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    tr.model.load_state_dict(weights(gd, torch.bfloat16), strict=False)
    tr = tr.to(device="cuda", dtype=torch.bfloat16).eval().requires_grad_(False)
    for blk in tr.model.blocks:
        blk.self_attn.fuse_projections()
    tr.model.attn_quant = "sage" if sage else None
    tr.use_cuda_graphs = graphs
    dec = VAEDecoderWrapper()
    dec.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    dec = dec.to(device="cuda", dtype=torch.float16).eval()
    enc = VAEEncoderWrapper()
    enc.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
    enc = enc.to(device="cuda", dtype=torch.float16).eval()
    return tr, dec, enc


# measured 3.2e-3 on an H100 80GB HBM3 (400 W power limit); bound with 3x headroom
SERVER_LOOP_LATENT_BOUND = 1e-2


def test_server_loop_with_sage_stays_within_its_tier():
    import harness
    gold = load_npz("server_loop_small.npz")
    draws = [gold[f"keep/draw{i}"] for i in range(int(gold["keep/ndraws"]))]
    tr, dec, enc = _server_models(sage=True)
    models = harness.build_models(tr, vae_decoder=dec, vae_encoder=enc, device="cuda")
    params = harness.GenerateParams(width=96, height=64, seed=11, kv_cache_num_frames=3, num_blocks=4,
                                    num_denoising_steps=4, keep_first_frame=True)
    with ReplayRandn(draws):
        sess = harness.GenerationSession(params, models, prompt_embeds=gold["prompt_embeds"], device="cuda")
        for _ in range(4):
            sess.generate_block()
    lat = sess.all_latents.float().cpu()
    r = rel_l2(lat, gold["keep/latents"].float())
    print(f"server loop, 4 blocks, sage: latents rel-L2 {r:.3e} vs the reference-executed golden")
    assert torch.isfinite(lat).all() and r <= SERVER_LOOP_LATENT_BOUND, r


def test_cuda_graph_replay_with_sage_is_bit_identical_to_eager():
    import harness
    gold = load_npz("server_loop_small.npz")

    def run(graphs: bool):
        tr, dec, _ = _server_models(sage=True, graphs=graphs)
        models = harness.build_models(tr, vae_decoder=dec, device="cuda")
        params = harness.GenerateParams(width=96, height=64, seed=3, kv_cache_num_frames=3, num_blocks=5,
                                        num_denoising_steps=4, keep_first_frame=True)
        sess = harness.GenerationSession(params, models, prompt_embeds=gold["prompt_embeds"], device="cuda")
        px = [sess.generate_block().clone() for _ in range(5)]
        return px, sess.all_latents.clone(), tr

    px_e, lat_e, _ = run(False)
    px_g, lat_g, tr = run(True)
    assert sum("graph" in st for st in tr._graphs.values()) >= 3
    assert torch.equal(lat_e, lat_g)
    for a, b in zip(px_e, px_g):
        assert torch.equal(a, b)
