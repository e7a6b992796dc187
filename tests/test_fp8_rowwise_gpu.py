"""Row-scaled FP8 (torchao ``granularity=PerRow()``) on the GPU, through the C ABI, against
oracle/fp8_rowwise_oracle.py.
  * kr_fp8_quantize_rows and kr_ln_modulate_fp8: e4m3 bytes and row scales BIT-EXACT vs the oracle (same fp32 divide
    and multiply, round-to-nearest-even saturating cast); the fused LayerNorm's bf16 output byte-identical to
    kr_ln_modulate's;
  * kr_gemm_fp8_rowwise: e4m3 products are exact in fp32, only the accumulation order and the order of the two scale
    multiplies differ -> rel-L2 <= 2e-3 on the bf16 output vs the oracle and vs torch._scaled_mm with row-wise scales;
  * model level: one 14B-dim layer against bf16 (<= 8e-2, the FP8 tier's bound), determinism, CUDA-graph replay."""
import pytest
import torch

from oracle import fp8_rowwise_oracle as F8
from tests.golden_io import rel_l2

pytestmark = pytest.mark.gpu


def _mixed_rows(rows, cols, gen):
    """Rows whose magnitudes span 1e-4 .. 1 (log-uniform) and one outlier element of 64 in the largest row: the
    outlier sets a tensor-wide scale that pushes the small rows into e4m3's subnormals or to zero."""
    mag = torch.logspace(-4, 0, rows)[torch.randperm(rows, generator=gen)]
    x = torch.randn(rows, cols, generator=gen) * mag[:, None]
    x[mag.argmax(), 0] = 64.0
    return x


@pytest.mark.parametrize("rows", [4680, 585, 7])
@pytest.mark.parametrize("cols", [1536, 5120, 8960, 13824])
def test_row_quantiser_is_bit_exact(rows, cols):
    from realtime_video_b200 import ops
    g = torch.Generator().manual_seed(rows + cols)
    x = (torch.randn(rows, cols, generator=g) * 2.5).bfloat16()
    x[0] = 0                                                    # zero row -> zeros, scale 1e-12 / 448
    if rows > 2:
        x[1] = 1e-3
        x[1, cols // 3] = 300.0                                 # single outlier
        x[2] = torch.randn(cols, generator=g).bfloat16() * 1e4  # large values: the amax still maps to 448 exactly
    xs = torch.zeros(rows, cols + 64).bfloat16()
    xs[:, 8:8 + cols] = x
    for src in (x.cuda(), xs.cuda()[:, 8:8 + cols]):          # contiguous and strided
        r = ops.fp8_quantize_rows(src)
        ref_q, ref_s = F8.quantize_per_row(x)
        assert torch.equal(r.q.cpu(), ref_q.view(torch.uint8))
        assert torch.equal(r.scale.cpu(), ref_s)
    assert int(r.q[0].cpu().abs().max()) == 0
    if rows > 2:
        assert float(r.q[1].cpu().view(torch.float8_e4m3fn).float().abs().max()) == 448.0


def test_row_quantiser_saturates_and_keeps_pitches():
    from realtime_video_b200 import ops
    x = torch.full((3, 256), 2.0).bfloat16()
    x[:, 5] = -8.0
    q = torch.full((3, 384), 0x55, dtype=torch.uint8, device="cuda")
    r = ops.fp8_quantize_rows(x.cuda(), q=q[:, :256])
    assert torch.equal(r.q.cpu(), F8.quantize_per_row(x)[0].view(torch.uint8))
    assert bool((q[:, 256:] == 0x55).all())                    # bytes past the row untouched
    assert float(r.q.cpu().view(torch.float8_e4m3fn).float()[:, 5].min()) == -448.0


@pytest.mark.parametrize("D", [1536, 5120])
@pytest.mark.parametrize("form", ["modulated", "affine"])
def test_ln_modulate_fp8_matches_ln_modulate_then_row_quantiser(D, form):
    from realtime_video_b200 import ops
    g = torch.Generator().manual_seed(D)
    rows, fs, r0 = 585, 195, 390
    x = (torch.randn(rows, D, generator=g) * 3 + 0.5).bfloat16().cuda()
    kw = dict(eps=1e-6, row_offset=r0)
    if form == "modulated":
        kw.update(mod=(torch.randn(6, 6, D, generator=g) * 0.3).bfloat16().cuda(), shift_idx=3, scale_idx=4,
                  rows_per_frame=fs)
    else:
        kw.update(weight=(1 + 0.2 * torch.randn(D, generator=g)).bfloat16().cuda(),
                  bias=(0.2 * torch.randn(D, generator=g)).bfloat16().cuda())
    want = ops.ln_modulate(x, **kw)
    out = torch.empty_like(want)
    r = ops.ln_modulate_fp8(x, out=out, **kw)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))               # byte-identical bf16 output
    ref_q, ref_s = F8.quantize_per_row(want.cpu())
    assert torch.equal(r.q.cpu(), ref_q.view(torch.uint8)) and torch.equal(r.scale.cpu(), ref_s)
    r2 = ops.ln_modulate_fp8(x, **kw)                                              # out = null: same bytes
    assert torch.equal(r2.q, r.q) and torch.equal(r2.scale, r.scale)


def _oracle_acc(x, w, b):
    xq, sx = F8.quantize_per_row(x.cpu())
    wq, sw = F8.quantize_per_row(w.cpu())
    return ((xq.float() @ wq.float().t()) * sx[:, None] * sw[None, :]).cuda() + b.float()


@pytest.mark.parametrize("M,N,K,epi", [(4680, 15360, 5120, "split"), (4680, 5120, 5120, "gate_res"),
                                       (4680, 13824, 5120, "gelu"), (4680, 5120, 13824, "res"), (585, 5120, 5120, "bias"),
                                       (100, 256, 512, "bias")])
def test_rowwise_gemm_vs_oracle(M, N, K, epi):
    from realtime_video_b200 import fp8, ops
    torch.manual_seed(M + N)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    wq, sw = fp8.quantize_weight_rows(w)
    assert torch.equal(wq.cpu(), F8.quantize_per_row(w.cpu())[0].view(torch.uint8))
    acc = _oracle_acc(x, w, b)
    if epi == "bias":
        out, want = ops.linear_fp8_rowwise(x, wq, sw, b), acc
    elif epi == "gelu":
        out = ops.linear_fp8_rowwise(x, wq, sw, b, epilogue=ops.EPI_BIAS_GELU)
        want = torch.nn.functional.gelu(acc.bfloat16().float(), approximate="tanh")
    elif epi == "res":
        r = torch.randn(M, N, device="cuda").bfloat16()
        out = ops.linear_fp8_rowwise(x, wq, sw, b, epilogue=ops.EPI_BIAS_RES, residual=r)
        want = r.float() + acc.bfloat16().float()
    elif epi == "gate_res":
        r = torch.ones(M, N, device="cuda").bfloat16()
        gate = torch.randn(3, N, device="cuda").bfloat16()
        want = r.float() + (acc.bfloat16().float() * gate.float().repeat_interleave(1560, 0)).bfloat16().float()
        out = ops.linear_fp8_rowwise(x, wq, sw, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, gate=gate,
                                     rows_per_gate=1560, out=r)
    else:
        out = torch.empty(M, 10240, device="cuda", dtype=torch.bfloat16)
        v = torch.zeros(M + 8, 5120, device="cuda", dtype=torch.bfloat16)
        ops.linear_fp8_rowwise(x, wq, sw, b, out=out, out2=v[4:4 + M], n_split=10240)
        assert rel_l2(v[4:4 + M].float(), acc[:, 10240:]) < 2e-3
        assert float(v[:4].abs().max()) == 0 and float(v[4 + M:].abs().max()) == 0      # guard rows untouched
        want = acc[:, :10240]
    torch.cuda.synchronize()
    assert rel_l2(out.float(), want) < 2e-3


@pytest.mark.parametrize("M,N,K", [(4680, 5120, 5120), (585, 13824, 5120), (100, 256, 512)])
def test_rowwise_gemm_vs_torch_scaled_mm(M, N, K):
    """The oracle's scaled matmul pinned on the GPU: torch._scaled_mm with scale_a [M, 1] and scale_b [1, N]."""
    from realtime_video_b200 import fp8, ops
    torch.manual_seed(K + N)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    wq, sw = fp8.quantize_weight_rows(w)
    xr = ops.fp8_quantize_rows(x)
    want = torch._scaled_mm(xr.q.view(torch.float8_e4m3fn), wq.view(torch.float8_e4m3fn).t(),
                            scale_a=xr.scale.reshape(M, 1), scale_b=sw.reshape(1, N), out_dtype=torch.bfloat16)
    got = ops.gemm_fp8_rowwise(xr, wq, sw)
    oracle = F8.linear_fp8_rowwise(x.cpu(), w.cpu())
    assert rel_l2(got.float(), want.float()) < 2e-3
    assert rel_l2(oracle.float().cuda(), want.float()) < 2e-3


def test_rowwise_beats_per_tensor_on_mixed_magnitude_rows():
    from realtime_video_b200 import fp8, ops
    g = torch.Generator().manual_seed(5)
    x = _mixed_rows(585, 5120, g).bfloat16().cuda()
    w = (torch.randn(5120, 5120, generator=g) * 0.02).bfloat16().cuda()
    exact = x.double() @ w.double().t()

    def per_row_err(y):
        return float(((y.double() - exact).norm(dim=1) / exact.norm(dim=1)).mean())
    wq_t, sw_t = fp8.quantize_weight(w)
    wq_r, sw_r = fp8.quantize_weight_rows(w)
    e_tensor = per_row_err(ops.linear_fp8(x, wq_t, sw_t))
    e_row = per_row_err(ops.linear_fp8_rowwise(x, wq_r, sw_r))
    assert e_row <= 0.5 * e_tensor, (e_row, e_tensor)


def _layer_model():
    from realtime_video_b200.dit import CausalWanModel
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = CausalWanModel(num_layers=1, dim=5120, ffn_dim=13824, num_heads=40, text_dim=4096)
    with torch.no_grad():
        m.head.head.weight.normal_(std=0.02)
    m = m.to(torch.bfloat16).eval()
    m.blocks[0].self_attn.fuse_projections()
    return m


def _layer_run(m, x, ctx):
    kv = [dict(k=torch.zeros(1, 4680, 40, 128, dtype=torch.bfloat16, device="cuda"),
               v=torch.zeros(1, 4680, 40, 128, dtype=torch.bfloat16, device="cuda"), global_end_index=0,
               local_end_index=0)]
    ca = [dict(k=torch.zeros(1, 512, 40, 128, dtype=torch.bfloat16, device="cuda"),
               v=torch.zeros(1, 512, 40, 128, dtype=torch.bfloat16, device="cuda"), is_init=False)]
    with torch.no_grad():
        return m(x[None], t=torch.full((1, 3), 750.0, device="cuda"), context=ctx[None], seq_len=32760,
                 kv_cache=kv, crossattn_cache=ca, current_start=0)[0].float()


def test_rowwise_layer_vs_bf16_layer_at_14b_dims():
    """One Wan-14B-dim layer, Lq 4680, as tests/test_fp8_gpu.py::test_fp8_layer_vs_bf16_layer_at_14b_dims, with the
    PerTensor value measured beside the PerRow one on the same weights / inputs (both recorded in DESIGN §5)."""
    from realtime_video_b200 import fp8
    m = _layer_model()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 60, 104, generator=g).bfloat16().cuda()
    ctx = torch.randn(40, 4096, generator=g).bfloat16().cuda()
    ref = _layer_run(m, x, ctx)
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerTensor()))
    r_tensor = rel_l2(_layer_run(m, x, ctx), ref)
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    got = _layer_run(m, x, ctx)
    again = _layer_run(m, x, ctx)
    r_row = rel_l2(got, ref)
    print(f"\n14B-dim layer rel-L2 vs bf16: PerRow {r_row:.4e}, PerTensor {r_tensor:.4e}")
    assert torch.isfinite(got).all() and r_row < 8e-2, r_row
    assert torch.equal(got, again)                                    # two PerRow runs are bit-identical


def test_server_loop_cuda_graph_replay_with_per_row_fp8_is_bit_identical_to_eager():
    import harness
    from realtime_video_b200 import fp8
    from realtime_video_b200.factory import synthetic_vae_params
    from realtime_video_b200.vae import VAEDecoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    from tests.golden_io import load_npz, weights
    gold, gd = load_npz("server_loop_small.npz"), load_npz("dit_small.npz")

    def run(graphs: bool):
        tr = WanDiffusionWrapper(model_name="synthetic", timestep_shift=5.0, is_causal=True,
                                 model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
        tr.model.load_state_dict(weights(gd, torch.bfloat16), strict=False)
        tr = tr.to(device="cuda", dtype=torch.bfloat16).eval().requires_grad_(False)
        for blk in tr.model.blocks:
            blk.self_attn.fuse_projections()
        fp8.quantize_(tr, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=[fp8.PerRow(), fp8.PerRow()]))
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
    assert sum("graph" in st for st in tr._graphs.values()) >= 3
    assert torch.isfinite(lat_e).all() and torch.equal(lat_e, lat_g)
    for a, b in zip(px_e, px_g):
        assert torch.equal(a, b)
