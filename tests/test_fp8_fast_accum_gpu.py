"""Fast accumulation for the FP8 linears (torchao ``Float8MMConfig(use_fast_accum=True)``) on the GPU, through the C
ABI.  kr_gemm_fp8_fast / kr_gemm_fp8_rowwise_fast read the same e4m3 bytes and scales as the promoted kernels and differ
only in where the sum over K is kept: inside the tensor core for the whole K instead of fp32 registers every 128 k.
  * against the exact product of the same quantised operands (fp32 matmul of the e4m3 values, scales, bias, epilogue;
    the arithmetic of oracle/fp8_oracle.py and oracle/fp8_rowwise_oracle.py), beside the promoted kernel on the same
    data; bounds and measured values: DESIGN.md section 5;
  * against torch._scaled_mm(use_fast_accum=True), the call the reference's torchao linears end in, with the gap of
    _scaled_mm fast vs slow on the same data beside it;
  * constructed same-sign data, where a short accumulator loses most;
  * model level: one 14B-dim layer against bf16 (<= 8e-2, the FP8 tier's bound), determinism, CUDA-graph replay, the
    server loop against the reference-executed golden latents."""
import pytest
import torch

from tests.golden_io import rel_l2

pytestmark = pytest.mark.gpu

# rel-L2 of the bf16 output against the exact product of the quantised operands (bf16 rounding alone is 1.6e-3).
# Promoted accumulation: <= 2e-3 (tests/test_fp8_gpu.py; measured here 1.39e-3 .. 1.85e-3).  Fast accumulation, measured
# on an H100 80GB HBM3 with N(0, 1) activations and N(0, 0.02) weights: 2.07e-3 .. 2.73e-3 at K = 5120 and 3.08e-3 ..
# 3.62e-3 at K = 13824, the same for both granularities (it grows with K; 1.65e-3 at K = 512).
PROMOTED_BOUND = 2e-3
FAST_BOUND = 5e-3


def _operands(M, N, K, rowwise, seed):
    """bf16 activation / weight / bias, their e4m3 bytes and scales from the library's own quantisers (bit-exact
    against the oracles: tests/test_fp8_gpu.py, tests/test_fp8_rowwise_gpu.py), and the exact fp32 accumulator."""
    from realtime_video_b200 import fp8, ops
    torch.manual_seed(seed)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    if rowwise:
        wq, sw = fp8.quantize_weight_rows(w)
        a = ops.fp8_quantize_rows(x)
        sa = a.scale[:M, None] * sw[None, :]
        aq = a.q
    else:
        wq, sw = fp8.quantize_weight(w)
        aq, state = ops.fp8_quantize(x)
        a, sa = (aq, state), state[1] * sw
    acc = (aq.view(torch.float8_e4m3fn).float() @ wq.view(torch.float8_e4m3fn).float().t()) * sa + b.float()
    return a, wq, sw, b, acc


def _gemm(a, wq, sw, b, rowwise, fast, **kw):
    from realtime_video_b200 import ops
    if rowwise:
        return ops.gemm_fp8_rowwise(a, wq, sw, b, fast_accum=fast, **kw)
    return ops.gemm_fp8(a[0], wq, a[1], sw, b, fast_accum=fast, **kw)


@pytest.mark.parametrize("rowwise", [False, True], ids=["PerTensor", "PerRow"])
@pytest.mark.parametrize("M,N,K,epi", [(4680, 15360, 5120, "split"), (4680, 5120, 5120, "gate_res"),
                                       (4680, 13824, 5120, "gelu"), (4680, 5120, 13824, "res"),
                                       (4680, 5120, 13824, "gate_res"), (585, 5120, 5120, "bias"),
                                       (585, 13824, 5120, "gelu"), (1000, 5120, 13824, "bias"), (100, 256, 512, "bias"),
                                       (7, 512, 144, "res")])
def test_fast_gemm_vs_exact_product_of_the_quantised_operands(M, N, K, epi, rowwise):
    from realtime_video_b200 import ops
    a, wq, sw, b, acc = _operands(M, N, K, rowwise, M + N)
    rel = {}
    for fast in (True, False):
        if epi == "bias":
            out, want = _gemm(a, wq, sw, b, rowwise, fast), acc
        elif epi == "gelu":
            out = _gemm(a, wq, sw, b, rowwise, fast, epilogue=ops.EPI_BIAS_GELU)
            want = torch.nn.functional.gelu(acc.bfloat16().float(), approximate="tanh")
        elif epi == "res":
            r = torch.randn(M, N, device="cuda", generator=torch.Generator("cuda").manual_seed(1)).bfloat16()
            out = _gemm(a, wq, sw, b, rowwise, fast, epilogue=ops.EPI_BIAS_RES, residual=r)
            want = r.float() + acc.bfloat16().float()
        elif epi == "gate_res":                                       # in place: the residual is the output
            r = torch.ones(M, N, device="cuda").bfloat16()
            gate = torch.randn(3, N, device="cuda", generator=torch.Generator("cuda").manual_seed(2)).bfloat16()
            want = r.float() + (acc.bfloat16().float() * gate.float().repeat_interleave(1560, 0)).bfloat16().float()
            out = _gemm(a, wq, sw, b, rowwise, fast, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, gate=gate,
                        rows_per_gate=1560, out=r)
        else:                                                         # to_qkv: V columns into a row slice of a cache
            out = torch.empty(M, 10240, device="cuda", dtype=torch.bfloat16)
            v = torch.zeros(M + 8, 5120, device="cuda", dtype=torch.bfloat16)
            _gemm(a, wq, sw, b, rowwise, fast, out=out, out2=v[4:4 + M], n_split=10240)
            assert rel_l2(v[4:4 + M].float(), acc[:, 10240:]) < (FAST_BOUND if fast else PROMOTED_BOUND)
            assert float(v[:4].abs().max()) == 0 and float(v[4 + M:].abs().max()) == 0      # guard rows untouched
            want = acc[:, :10240]
        torch.cuda.synchronize()
        rel[fast] = rel_l2(out.float(), want)
    print(f"\nrel-L2 vs exact, {'PerRow' if rowwise else 'PerTensor'} M={M} N={N} K={K} {epi}: "
          f"fast {rel[True]:.3e}, promoted {rel[False]:.3e}")
    assert rel[False] < PROMOTED_BOUND and rel[True] < FAST_BOUND, rel


def test_rows_past_m_are_neither_read_nor_written():
    """M = 200 on a 128-row tile grid: the output buffer's rows past M keep their fill, and the row scales past M
    (NaN here) do not reach any output."""
    from realtime_video_b200 import ops
    a, wq, sw, b, acc = _operands(256, 512, 1024, True, 3)
    a.scale[200:] = float("nan")
    out = torch.full((256, 512), 7.0, device="cuda", dtype=torch.bfloat16)
    ops.gemm_fp8_rowwise(ops.Fp8Rows(a.q[:200], a.scale, a.dtype), wq, sw, b, out=out[:200], fast_accum=True)
    assert bool((out[200:] == 7.0).all()) and torch.isfinite(out).all()
    assert rel_l2(out[:200].float(), acc[:200]) < FAST_BOUND


@pytest.mark.parametrize("M,N,K", [(4680, 5120, 5120), (585, 5120, 13824), (100, 256, 512)])
def test_fast_gemm_vs_torch_scaled_mm_fast_accum(M, N, K):
    """The reference's linears end in torch._scaled_mm(use_fast_accum=True).  Bit equality is not required (the order
    of the scale multiplies and of the k-blocks is the library's own); measured on an H100 80GB HBM3: per-tensor scales
    0 (bit-identical), row-wise scales 1.7e-5, while _scaled_mm fast vs slow and this package's fast vs promoted are
    both 2.53e-3 at K = 5120 and 3.62e-3 at K = 13824: the two fast kernels sit in the same place."""
    a, wq, sw, _, _ = _operands(M, N, K, True, K + N)
    mm = lambda fast: torch._scaled_mm(a.q.view(torch.float8_e4m3fn), wq.view(torch.float8_e4m3fn).t(),
                                       scale_a=a.scale.reshape(M, 1), scale_b=sw.reshape(1, N),
                                       out_dtype=torch.bfloat16, use_fast_accum=fast).float()
    ours = _gemm(a, wq, sw, None, True, True).float()
    ours_slow = _gemm(a, wq, sw, None, True, False).float()
    g_rows, g_lib, g_ours = rel_l2(ours, mm(True)), rel_l2(mm(True), mm(False)), rel_l2(ours, ours_slow)
    t, wq_t, sw_t, _, _ = _operands(M, N, K, False, K + N)
    one = torch.ones((), device="cuda")
    mm_t = lambda fast: torch._scaled_mm(t[0].view(torch.float8_e4m3fn), wq_t.view(torch.float8_e4m3fn).t(),
                                         scale_a=t[1][1] * one, scale_b=sw_t * one, out_dtype=torch.bfloat16,
                                         use_fast_accum=fast).float()
    g_tensor = rel_l2(_gemm(t, wq_t, sw_t, None, False, True).float(), mm_t(True))
    print(f"\nM={M} N={N} K={K}: ours fast vs _scaled_mm fast: PerRow {g_rows:.3e}, PerTensor {g_tensor:.3e}; "
          f"_scaled_mm fast vs slow {g_lib:.3e}; ours fast vs ours promoted {g_ours:.3e}")
    assert g_rows < 1e-3 and g_tensor < 1e-3
    assert g_ours < 2 * g_lib + PROMOTED_BOUND                       # the same place as cuBLASLt's fast accumulation


def test_same_sign_products_over_a_long_k():
    """The case a short accumulator handles worst: every product positive, so the running sum grows to K times one
    product and each late product loses its low bits when it is aligned to the sum; the tensor core truncates them, so
    the loss has one sign and adds up.  Measured on an H100 80GB HBM3 (K = 13824, e4m3 values in [1, 16)): fast
    accumulation 2.4e-1 below the exact sum, promoted 1.2e-3 (bf16 rounding), and torch._scaled_mm(use_fast_accum=True)
    loses what the fast kernel loses.  This documents the trade between the two modes on data built for it, not on
    activations (tests above and below); the bounds are loose."""
    from realtime_video_b200 import ops
    M, N, K = 256, 256, 13824
    g = torch.Generator("cuda").manual_seed(0)
    aq = (torch.rand(M, K, device="cuda", generator=g) * 15 + 1).to(torch.float8_e4m3fn)
    wq = (torch.rand(N, K, device="cuda", generator=g) * 15 + 1).to(torch.float8_e4m3fn)
    exact = aq.double() @ wq.double().t()
    sa, sw = torch.ones(M, device="cuda"), torch.full((N,), 2.0 ** -10, device="cuda")
    y = {fast: ops.gemm_fp8_rowwise(ops.Fp8Rows(aq.view(torch.uint8), sa, torch.bfloat16), wq.view(torch.uint8), sw,
                                    fast_accum=fast).double() * 2.0 ** 10 for fast in (True, False)}
    y["torch._scaled_mm fast"] = torch._scaled_mm(aq, wq.t(), scale_a=sa.reshape(M, 1), scale_b=sw.reshape(1, N),
                                                  out_dtype=torch.bfloat16, use_fast_accum=True).double() * 2.0 ** 10
    rel = {k: rel_l2(v, exact) for k, v in y.items()}
    for k, v in y.items():
        name = {True: "fast", False: "promoted"}.get(k, k)
        print(f"\nsame-sign K={K}: {name} rel-L2 {rel[k]:.3e}, mean signed error {float(((v - exact) / exact).mean()):+.3e}")
    assert rel[False] < PROMOTED_BOUND and rel[False] < rel[True] < 0.5, rel
    assert 0.5 * rel["torch._scaled_mm fast"] < rel[True] < 2 * rel["torch._scaled_mm fast"], rel


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


def test_fast_accum_layer_vs_bf16_layer_at_14b_dims():
    """One Wan-14B-dim layer, Lq 4680, as tests/test_fp8_rowwise_gpu.py::test_rowwise_layer_vs_bf16_layer_at_14b_dims
    (promoted: PerTensor 2.52e-2, PerRow 2.53e-2), both granularities with fast accumulation; the profile shows that
    the fast kernel and only the fast kernel ran."""
    from realtime_video_b200 import fp8, ops
    m = _layer_model()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 60, 104, generator=g).bfloat16().cuda()
    ctx = torch.randn(40, 4096, generator=g).bfloat16().cuda()
    ref = _layer_run(m, x, ctx)
    fastcfg = fp8.Float8MMConfig(use_fast_accum=True)
    for gran in (fp8.PerTensor, fp8.PerRow):
        fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=gran()))
        promoted = _layer_run(m, x, ctx)
        fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=gran(), mm_config=fastcfg))
        ops.profile_begin()
        got = _layer_run(m, x, ctx)
        torch.cuda.synchronize()
        prof = ops.profile_end()
        again = _layer_run(m, x, ctx)
        assert prof["gemm_fp8_fast"]["n"] == 8 and "gemm_fp8" not in prof
        r = rel_l2(got, ref)
        print(f"\n14B-dim layer rel-L2 vs bf16, {gran.__name__}: fast {r:.4e}, promoted {rel_l2(promoted, ref):.4e}, "
              f"fast vs promoted {rel_l2(got, promoted):.4e}")
        assert torch.isfinite(got).all() and r < 8e-2, r
        assert torch.equal(got, again)                                # two runs are bit-identical
    fp8.dequantize_(m)
    assert torch.equal(_layer_run(m, x, ctx), ref)                    # and the bf16 path is back


def _server_loop(graphs, config, blocks=5, seed=3, draws=None, encoder=False, keep=True):
    import harness
    from realtime_video_b200 import fp8
    from realtime_video_b200.factory import synthetic_vae_params
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEEncoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    from tests.golden_io import ReplayRandn, load_npz, weights
    import contextlib
    gold, gd = load_npz("server_loop_small.npz"), load_npz("dit_small.npz")
    tr = WanDiffusionWrapper(model_name="synthetic", timestep_shift=5.0, is_causal=True,
                             model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    tr.model.load_state_dict(weights(gd, torch.bfloat16), strict=False)
    tr = tr.to(device="cuda", dtype=torch.bfloat16).eval().requires_grad_(False)
    for blk in tr.model.blocks:
        blk.self_attn.fuse_projections()
    if config is not None:
        fp8.quantize_(tr, config)
    tr.use_cuda_graphs = graphs
    dec = VAEDecoderWrapper()
    dec.load_state_dict(synthetic_vae_params(seed=0), strict=False)
    dec = dec.to(device="cuda", dtype=torch.float16).eval()
    enc = None
    if encoder:
        enc = VAEEncoderWrapper()
        enc.load_state_dict(synthetic_vae_params(seed=0, encoder=True), strict=False)
        enc = enc.to(device="cuda", dtype=torch.float16).eval()
    models = harness.build_models(tr, vae_decoder=dec, vae_encoder=enc, device="cuda")
    params = harness.GenerateParams(width=96, height=64, seed=seed, kv_cache_num_frames=3, num_blocks=blocks,
                                    num_denoising_steps=4, keep_first_frame=keep)
    with (ReplayRandn(draws) if draws is not None else contextlib.nullcontext()):
        sess = harness.GenerationSession(params, models, prompt_embeds=gold["prompt_embeds"], device="cuda")
        px = [sess.generate_block().clone() for _ in range(blocks)]
    return px, sess.all_latents.clone(), tr


@pytest.mark.parametrize("gran", ["PerTensor", "PerRow"])
def test_server_loop_cuda_graph_replay_with_fast_accum_is_bit_identical_to_eager(gran):
    from realtime_video_b200 import fp8
    cfg = fp8.Float8DynamicActivationFloat8WeightConfig(granularity=getattr(fp8, gran)(),
                                                        mm_config=fp8.Float8MMConfig(use_fast_accum=True))
    px_e, lat_e, _ = _server_loop(False, cfg)
    px_g, lat_g, tr = _server_loop(True, cfg)
    assert sum("graph" in st for st in tr._graphs.values()) >= 3
    assert torch.isfinite(lat_e).all() and torch.equal(lat_e, lat_g)
    for a, b in zip(px_e, px_g):
        assert torch.equal(a, b)


def test_server_loop_latents_with_fast_accum_vs_reference_executed_golden():
    """tests/test_server_loop_gpu.py's loop (4 blocks, recorded noise draws replayed) with the block linears on FP8:
    latents against the bf16 golden of the reference's own modules, fast accumulation beside promoted for both
    granularities.  The bound is the FP8 tier's 8e-2; fast accumulation adds nothing visible to it."""
    from realtime_video_b200 import fp8
    from tests.golden_io import load_npz
    gold = load_npz("server_loop_small.npz")
    draws = [gold[f"keep/draw{i}"] for i in range(int(gold["keep/ndraws"]))]
    want = gold["keep/latents"].float()
    r = {}
    for gran in (fp8.PerTensor, fp8.PerRow):
        for fast in (False, True):
            cfg = fp8.Float8DynamicActivationFloat8WeightConfig(granularity=gran(),
                                                                mm_config=fp8.Float8MMConfig(use_fast_accum=fast))
            _, lat, _ = _server_loop(False, cfg, blocks=4, seed=11, draws=list(draws), encoder=True)
            r[gran.__name__, fast] = rel_l2(lat.float().cpu(), want)
    print("\nserver loop latents rel-L2 vs golden:", {f"{g} {'fast' if f else 'promoted'}": f"{v:.3e}"
                                                        for (g, f), v in r.items()})
    for (g, fast), v in r.items():
        assert v < 8e-2, (g, fast, v)
    for g in ("PerTensor", "PerRow"):
        assert r[g, True] < 1.25 * r[g, False] + 5e-3, r
