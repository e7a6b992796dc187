"""Row a1 on the GPU: the server's block loop (harness/server_loop.py — proven bit-equal to the unmodified
``release_server.GenerationSession`` on the same drop-in classes by tests/test_reference_callers_cpu.py) on the
sm_90a kernels, against ``tests/golden/server_loop_small.npz`` = the same loop executed by the reference's own
modules (bf16 DiT, fp16 VAE; tests/golden/make_server_loop_golden.py).  4 blocks: cache init, recompute under the
block-causal mask, 4 denoise passes with re-noising (recorded draws replayed), VAE decode, sliding context window,
first-frame re-encode.  Tolerances: both sides round to bf16/fp16 at different points and the error compounds over
4 dependent blocks: latents rel-L2 <= 3e-2, pixels mean|d| <= 1.5e-2 on [-1, 1]."""
import pytest
import torch

from tests.golden_io import ReplayRandn, load_npz, rel_l2, weights

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("keep", [True, False], ids=["keep_first_frame", "reencode_first_frame"])
def test_server_block_loop_vs_reference_executed_golden(keep):
    import harness
    from realtime_video_b200.factory import synthetic_vae_params
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEEncoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    gold, gd = load_npz("server_loop_small.npz"), load_npz("dit_small.npz")
    tag = "keep" if keep else "reenc"
    draws = [gold[f"{tag}/draw{i}"] for i in range(int(gold[f"{tag}/ndraws"]))]
    tr = WanDiffusionWrapper(model_name="synthetic", timestep_shift=5.0, is_causal=True,
                             model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    tr.model.load_state_dict(weights(gd, torch.bfloat16), strict=False)
    tr = tr.to(device="cuda", dtype=torch.bfloat16).eval().requires_grad_(False)
    for blk in tr.model.blocks:
        blk.self_attn.fuse_projections()
    dec = VAEDecoderWrapper()
    dec.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    dec = dec.to(device="cuda", dtype=torch.float16).eval()
    enc = VAEEncoderWrapper()
    enc.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
    enc = enc.to(device="cuda", dtype=torch.float16).eval()
    models = harness.build_models(tr, vae_decoder=dec, vae_encoder=enc, device="cuda")
    params = harness.GenerateParams(width=96, height=64, seed=11, kv_cache_num_frames=3, num_blocks=4,
                                    num_denoising_steps=4, keep_first_frame=keep)
    with ReplayRandn(draws):
        sess = harness.GenerationSession(params, models, prompt_embeds=gold["prompt_embeds"], device="cuda")
        px = [sess.generate_block().float().cpu() for _ in range(4)]
    r = rel_l2(sess.all_latents.float().cpu(), gold[f"{tag}/latents"].float())
    assert r < 3e-2, f"latents rel_l2={r:.3e}"
    for b in range(4):
        ref = gold[f"{tag}/px{b}_sub"].float()
        got = px[b][..., ::2, ::2]
        assert got.shape == ref.shape
        mad = (got - ref).abs().mean().item()
        assert mad < 1.5e-2, f"block {b}: mean|d|={mad:.3e}"


def test_cuda_graph_replay_of_the_dit_passes_is_bit_identical_to_eager():
    """``wrapper.use_cuda_graphs``: from the second occurrence of a pass signature on, the pass is replayed as a CUDA
    graph (static input buffers, Python-side cache indices restored).  5 blocks of the server loop: blocks 3-4 run
    entirely on replays; pixels and latents must equal the eager run bit for bit."""
    import harness
    from realtime_video_b200.factory import synthetic_vae_params
    from realtime_video_b200.vae import VAEDecoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    gold, gd = load_npz("server_loop_small.npz"), load_npz("dit_small.npz")

    def run(graphs: bool):
        tr = WanDiffusionWrapper(model_name="synthetic", timestep_shift=5.0, is_causal=True,
                                 model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
        tr.model.load_state_dict(weights(gd, torch.bfloat16), strict=False)
        tr = tr.to(device="cuda", dtype=torch.bfloat16).eval().requires_grad_(False)
        for blk in tr.model.blocks:
            blk.self_attn.fuse_projections()
        tr.use_cuda_graphs = graphs
        dec = VAEDecoderWrapper()
        dec.load_state_dict(synthetic_vae_params(seed=0), strict=False)
        dec = dec.to(device="cuda", dtype=torch.float16).eval()
        models = harness.build_models(tr, vae_decoder=dec, device="cuda")
        params = harness.GenerateParams(width=96, height=64, seed=3, kv_cache_num_frames=3, num_blocks=5,
                                        num_denoising_steps=4, keep_first_frame=True)
        sess = harness.GenerationSession(params, models, prompt_embeds=gold["prompt_embeds"], device="cuda")
        px = [sess.generate_block().clone() for _ in range(5)]
        return px, sess.all_latents.clone(), tr

    px_e, lat_e, _ = run(False)
    px_g, lat_g, tr = run(True)
    assert sum("graph" in st for st in tr._graphs.values()) >= 3      # recompute + first / later denoise passes
    assert torch.equal(lat_e, lat_g)
    for a, b in zip(px_e, px_g):
        assert torch.equal(a, b)
