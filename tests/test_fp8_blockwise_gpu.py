"""Block-scaled FP8 (torchao ``granularity=[PerBlock([1, 128]), PerBlock([128, 128])]``) on the GPU, through the C ABI,
against oracle/fp8_blockwise_oracle.py.
  * kr_fp8_quantize_blocks and kr_ln_modulate_fp8_blocks: e4m3 bytes and group scales BIT-EXACT vs the oracle; the
    fused LayerNorm's bf16 output byte-identical to kr_ln_modulate's;
  * kr_gemm_fp8_blockwise: e4m3 products are exact in fp32, only the accumulation order and the scale multiplies
    differ -> rel-L2 <= 2e-3 vs the oracle's float64 product of the same operands, for every epilogue, the six DiT
    projections at M = 4680, an M tail and the split-V store; and vs torch._scaled_mm with block-wise scales where
    torch and cuBLAS run them;
  * the error advantage on channel outliers over PerRow; one 14B-dim layer vs bf16 (<= 8e-2); the server loop vs the
    reference-executed golden; determinism and CUDA-graph replay."""
import pytest
import torch

from oracle import fp8_blockwise_oracle as F8B
from tests.golden_io import rel_l2

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("rows", [4680, 585, 7])
@pytest.mark.parametrize("cols", [1536, 5120, 8960, 13824])
def test_group_quantiser_is_bit_exact(rows, cols):
    from realtime_video_b200 import ops
    g = torch.Generator().manual_seed(rows + cols)
    x = (torch.randn(rows, cols, generator=g) * 2.5).bfloat16()
    x[0] = 0                                                    # zero row -> zeros, scales 1e-12 / 448
    if rows > 2:
        x[1] = 1e-3
        x[1, cols // 3] = 300.0                                 # single outlier: only its group's scale moves
        x[2] = torch.randn(cols, generator=g).bfloat16() * 1e4
    xs = torch.zeros(rows, cols + 64).bfloat16()
    xs[:, 8:8 + cols] = x
    ref_q, ref_s = F8B.quantize_per_group(x)
    for src in (x.cuda(), xs.cuda()[:, 8:8 + cols]):          # contiguous and strided
        r = ops.fp8_quantize_blocks(src)
        assert torch.equal(r.q.cpu(), ref_q.view(torch.uint8))
        assert torch.equal(r.scale.cpu(), ref_s)
    # a scale pitch wider than the rows: the k-block-major layout the GEMM reads, padding untouched
    scale = torch.full((cols // 128, rows + 5), -1.0, device="cuda")
    r = ops.fp8_quantize_blocks(x.cuda(), scale=scale[:, :rows])
    assert torch.equal(scale[:, :rows].cpu(), ref_s) and bool((scale[:, rows:] == -1).all())


@pytest.mark.parametrize("D", [1536, 5120])
@pytest.mark.parametrize("form", ["modulated", "affine"])
def test_ln_modulate_fp8_blocks_matches_ln_modulate_then_group_quantiser(D, form):
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
    r = ops.ln_modulate_fp8_blocks(x, out=out, **kw)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))               # byte-identical bf16 output
    ref_q, ref_s = F8B.quantize_per_group(want.cpu())
    assert torch.equal(r.q.cpu(), ref_q.view(torch.uint8)) and torch.equal(r.scale.cpu(), ref_s)
    r2 = ops.ln_modulate_fp8_blocks(x, **kw)                                       # out = null: same bytes
    assert torch.equal(r2.q, r.q) and torch.equal(r2.scale, r.scale)


def _operands(M, N, K, seed):
    from realtime_video_b200 import fp8, ops
    torch.manual_seed(seed)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    wq, sw = fp8.quantize_weight_blocks(w)
    xb = ops.fp8_quantize_blocks(x)
    # the oracle's float64 product, evaluated on the device (the CPU would take minutes at these sizes)
    exact = F8B.matmul_blockwise(xb.q.view(torch.float8_e4m3fn), xb.scale, wq.view(torch.float8_e4m3fn), sw)
    return xb, wq, sw, b, exact


# the six DiT projections of the 14B model at M = 4680 (one 3-frame block at 832x480) with their real epilogues, the
# M tail, and every epilogue
SHAPES = [(4680, 15360, 5120, "split"), (4680, 5120, 5120, "gate_res"), (4680, 5120, 5120, "bias"),
          (4680, 5120, 5120, "res"), (4680, 13824, 5120, "gelu"), (4680, 5120, 13824, "gate_res"),
          (585, 5120, 5120, "f32"), (100, 256, 512, "bias"), (200, 384, 1536, "res")]


@pytest.mark.parametrize("M,N,K,epi", SHAPES)
def test_blockwise_gemm_vs_oracle(M, N, K, epi):
    from realtime_video_b200 import ops
    xb, wq, sw, b, exact = _operands(M, N, K, M + N + K)
    acc = exact + b.double()
    if epi == "bias":
        out, want = ops.gemm_fp8_blockwise(xb, wq, sw, b), acc
    elif epi == "f32":
        out, want = ops.gemm_fp8_blockwise(xb, wq, sw, b, epilogue=ops.EPI_F32), acc
        assert out.dtype == torch.float32
    elif epi == "gelu":
        out = ops.gemm_fp8_blockwise(xb, wq, sw, b, epilogue=ops.EPI_BIAS_GELU)
        want = torch.nn.functional.gelu(acc.bfloat16().double(), approximate="tanh")
    elif epi == "res":
        r = torch.randn(M, N, device="cuda").bfloat16()
        out = ops.gemm_fp8_blockwise(xb, wq, sw, b, epilogue=ops.EPI_BIAS_RES, residual=r)
        want = r.double() + acc.bfloat16().double()
    elif epi == "gate_res":
        r = torch.ones(M, N, device="cuda").bfloat16()
        gate = torch.randn(3, N, device="cuda").bfloat16()
        want = r.double() + (acc.bfloat16().double() * gate.double().repeat_interleave(1560, 0)).bfloat16().double()
        out = ops.gemm_fp8_blockwise(xb, wq, sw, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, gate=gate,
                                     rows_per_gate=1560, out=r)
    else:
        out = torch.empty(M, 10240, device="cuda", dtype=torch.bfloat16)
        v = torch.zeros(M + 8, 5120, device="cuda", dtype=torch.bfloat16)
        ops.gemm_fp8_blockwise(xb, wq, sw, b, out=out, out2=v[4:4 + M], n_split=10240)
        assert rel_l2(v[4:4 + M].double(), acc[:, 10240:]) < 2e-3
        assert float(v[:4].abs().max()) == 0 and float(v[4 + M:].abs().max()) == 0      # guard rows untouched
        want = acc[:, :10240]
    torch.cuda.synchronize()
    err = rel_l2(out.double(), want)
    print(f"\nblockwise M={M} N={N} K={K} {epi}: rel-L2 vs oracle {err:.3e}")
    assert err < 2e-3


@pytest.mark.parametrize("M,N,K", [(4680, 5120, 5120), (585, 13824, 5120), (256, 256, 512)])
def test_blockwise_gemm_vs_torch_scaled_mm(M, N, K):
    """torch._scaled_mm with BlockWise1x128 / BlockWise128x128 scales (scale_a [M, K/128], scale_b [K/128, N/128])
    where this torch and cuBLAS run it; otherwise the comparison is skipped with torch's error, and the oracle
    comparison above stays the binding one."""
    from realtime_video_b200 import ops
    xb, wq, sw, _, exact = _operands(M, N, K, 7 + M)
    got = ops.gemm_fp8_blockwise(xb, wq, sw)
    assert rel_l2(got.double(), exact) < 2e-3
    want, errors = None, []
    # the scales as stored (outer-dim-major views) first, then row-major copies
    for sa, sb in ((xb.scale.t(), sw.t()), (xb.scale.t().contiguous(), sw.t().contiguous())):
        try:
            want = torch._scaled_mm(xb.q.view(torch.float8_e4m3fn), wq.view(torch.float8_e4m3fn).t(),
                                    scale_a=sa, scale_b=sb, out_dtype=torch.bfloat16)
            torch.cuda.synchronize()
            break
        except (RuntimeError, NotImplementedError, ValueError, TypeError) as e:
            errors.append(str(e).splitlines()[0] if str(e) else type(e).__name__)
    if want is None:
        pytest.skip(f"torch._scaled_mm with block-wise scales is not available here: {errors}")
    d = rel_l2(got.float(), want.float())
    print(f"\nM={M} N={N} K={K}: ours vs _scaled_mm block-wise {d:.3e}, _scaled_mm vs oracle "
          f"{rel_l2(want.double(), exact):.3e}")
    assert d < 2e-3


def test_block_scaling_beats_per_row_on_channel_outliers():
    """N(0, 1) activations with 4 channels scaled by 1e5 in every token: one scale per row lets them set every row's
    scale and pushes the other channels into e4m3's subnormals; one scale per 128-channel group confines that to the
    four groups holding them.  Error of the output vs the exact matmul of the unquantised bf16 operands."""
    from realtime_video_b200 import fp8, ops
    g = torch.Generator().manual_seed(5)
    x = torch.randn(585, 5120, generator=g)
    x[:, [17, 1300, 2900, 4444]] *= 1e5
    x = x.bfloat16().cuda()
    w = (torch.randn(5120, 5120, generator=g) * 0.02).bfloat16().cuda()
    ok = torch.ones(5120, dtype=torch.bool)
    for c in (17, 1300, 2900, 4444):
        ok[c // 128 * 128:(c // 128 + 1) * 128] = False        # compare the product over the outlier-free groups
    xo, wo = x[:, ok.cuda()].contiguous(), w[:, ok.cuda()].contiguous()
    exact = xo.double() @ wo.double().t()
    wq_r, sw_r = fp8.quantize_weight_rows(wo)
    wq_b, sw_b = fp8.quantize_weight_blocks(wo)
    # the outliers' scales are what the full rows would give: quantise the full rows, keep the outlier-free groups
    xr = ops.fp8_quantize_rows(x)
    xr = ops.Fp8Rows(xr.q[:, ok.cuda()].contiguous(), xr.scale, xr.dtype)
    xb = ops.fp8_quantize_blocks(x)
    keep = ok.reshape(40, 128)[:, 0].cuda()
    xb = ops.Fp8Blocks(xb.q[:, ok.cuda()].contiguous(), xb.scale[keep].contiguous(), xb.dtype)
    e_row = rel_l2(ops.gemm_fp8_rowwise(xr, wq_r, sw_r).double(), exact)
    e_blk = rel_l2(ops.gemm_fp8_blockwise(xb, wq_b, sw_b).double(), exact)
    print(f"\nchannel outliers: rel-L2 vs exact, PerBlock {e_blk:.3e}, PerRow {e_row:.3e} "
          f"(ratio {e_row / e_blk:.1f})")
    assert e_blk < 5e-2 and e_blk < 0.25 * e_row, (e_blk, e_row)


def _layer_model():
    from tests.test_fp8_rowwise_gpu import _layer_model as lm
    return lm()


def test_blockwise_layer_vs_bf16_layer_at_14b_dims():
    """One Wan-14B-dim layer, Lq 4680, on the same weights and inputs as the PerRow test: bound 8e-2, the FP8 tier's;
    two runs bit-identical."""
    from realtime_video_b200 import fp8
    from tests.test_fp8_rowwise_gpu import _layer_run
    m = _layer_model()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 60, 104, generator=g).bfloat16().cuda()
    ctx = torch.randn(40, 4096, generator=g).bfloat16().cuda()
    ref = _layer_run(m, x, ctx)
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    r_row = rel_l2(_layer_run(m, x, ctx), ref)
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(
        granularity=[fp8.PerBlock([1, 128]), fp8.PerBlock([128, 128])]))
    got = _layer_run(m, x, ctx)
    again = _layer_run(m, x, ctx)
    r_blk = rel_l2(got, ref)
    print(f"\n14B-dim layer rel-L2 vs bf16: PerBlock {r_blk:.4e}, PerRow {r_row:.4e}")
    assert torch.isfinite(got).all() and r_blk < 8e-2, r_blk
    assert torch.equal(got, again)


def _cfg():
    from realtime_video_b200 import fp8
    return fp8.Float8DynamicActivationFloat8WeightConfig(granularity=[fp8.PerBlock([1, 128]),
                                                                      fp8.PerBlock([128, 128])])


def test_server_loop_cuda_graph_replay_with_per_block_fp8_is_bit_identical_to_eager():
    from tests.test_fp8_fast_accum_gpu import _server_loop
    px_e, lat_e, _ = _server_loop(False, _cfg())
    px_g, lat_g, tr = _server_loop(True, _cfg())
    assert sum("graph" in st for st in tr._graphs.values()) >= 3
    assert torch.isfinite(lat_e).all() and torch.equal(lat_e, lat_g)
    for a, b in zip(px_e, px_g):
        assert torch.equal(a, b)


def test_server_loop_latents_with_per_block_fp8_vs_reference_executed_golden():
    """The 4-block server loop (recorded noise draws replayed) with the block linears on block-scaled FP8: latents
    against the bf16 golden of the reference's own modules, within the FP8 tier's 8e-2 (PerRow measured beside it)."""
    from realtime_video_b200 import fp8
    from tests.golden_io import load_npz
    from tests.test_fp8_fast_accum_gpu import _server_loop
    gold = load_npz("server_loop_small.npz")
    draws = [gold[f"keep/draw{i}"] for i in range(int(gold["keep/ndraws"]))]
    want = gold["keep/latents"].float()
    r = {}
    for name, cfg in (("PerRow", fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow())),
                      ("PerBlock", _cfg())):
        _, lat, _ = _server_loop(False, cfg, blocks=4, seed=11, draws=list(draws), encoder=True)
        r[name] = rel_l2(lat.float().cpu(), want)
    print("\nserver loop latents rel-L2 vs golden:", {k: f"{v:.3e}" for k, v in r.items()})
    assert r["PerBlock"] < 8e-2, r
