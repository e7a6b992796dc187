"""INT8 linears (torchao ``Int8DynamicActivationInt8WeightConfig``) on the GPU, through the C ABI, against
oracle/int8_oracle.py.
  * kr_i8_quantize_rows and kr_ln_modulate_i8: s8 bytes and row scales BIT-EXACT vs the oracle; the fused LayerNorm's
    bf16 output byte-identical to kr_ln_modulate's;
  * kr_gemm_i8_rowwise: the s32 sums are exact, so EPI_F32 with unit scales equals torch._int_mm bit for bit, and with
    real scales equals the oracle's fp32 dequantisation bit for bit; the bf16 epilogues are held to the oracle's
    float64 epilogue on the same sums;
  * numerics against e4m3 PerRow on four activation families, and the model level: one 14B-dim layer against bf16,
    the server loop against the reference-executed golden, determinism, CUDA-graph replay."""
import pytest
import torch

from oracle import int8_oracle as I8
from tests.golden_io import rel_l2

pytestmark = pytest.mark.gpu

SHAPES = {"to_qkv": (15360, 5120), "self_o": (5120, 5120), "cross_q": (5120, 5120), "cross_o": (5120, 5120),
          "ffn0": (13824, 5120), "ffn2": (5120, 13824)}


@pytest.mark.parametrize("rows", [4680, 585, 7, 1])
@pytest.mark.parametrize("cols", [1536, 5120, 13824])
def test_row_quantiser_is_bit_exact(rows, cols):
    from realtime_video_b200 import ops
    g = torch.Generator().manual_seed(rows + cols)
    x = (torch.randn(rows, cols, generator=g) * 2.5).bfloat16()
    x[0, : cols // 2] = 0
    if rows > 3:
        x[1] = 0                                                # zero row -> zeros, scale 1e-12 / 127
        x[2] = 0
        x[2, cols // 3] = -300.0                                # a single nonzero value -> -127
        x[3, :6] = torch.tensor([127.0, 0.5, 1.5, 2.5, -0.5, -2.5])   # multiplier exactly 1: ties to even
        x[3, 6:] = 0
    xs = torch.zeros(rows, cols + 64).bfloat16()
    xs[:, 8:8 + cols] = x
    ref_q, ref_s = I8.quantize_act_rows(x)
    for src in (x.cuda(), xs.cuda()[:, 8:8 + cols]):          # contiguous and strided
        r = ops.i8_quantize_rows(src)
        assert r.q.dtype == torch.int8 and torch.equal(r.q.cpu(), ref_q)
        assert torch.equal(r.scale.cpu(), ref_s)
    if rows > 3:
        assert int(r.q[1].abs().max()) == 0 and int(r.q[2, cols // 3]) == -127
        assert r.q[3, :6].tolist() == [127, 0, 2, 2, 0, -2]


@pytest.mark.parametrize("D", [1536, 5120])
@pytest.mark.parametrize("form", ["modulated", "affine"])
def test_ln_modulate_i8_matches_ln_modulate_then_row_quantiser(D, form):
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
    r = ops.ln_modulate_i8(x, out=out, **kw)
    assert torch.equal(out.view(torch.int16), want.view(torch.int16))               # byte-identical bf16 output
    k = ops.i8_quantize_rows(want)
    assert torch.equal(r.q, k.q) and torch.equal(r.scale, k.scale)
    ref_q, ref_s = I8.quantize_act_rows(want.cpu())
    assert torch.equal(r.q.cpu(), ref_q) and torch.equal(r.scale.cpu(), ref_s)
    r2 = ops.ln_modulate_i8(x, **kw)                                               # out = null: same bytes
    assert torch.equal(r2.q, r.q) and torch.equal(r2.scale, r.scale)


def _operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8)
    w = torch.randint(-128, 128, (N, K), generator=g, dtype=torch.int8)
    return a.cuda(), w.cuda()


@pytest.mark.parametrize("M,N,K", [(4680, *SHAPES[k]) for k in SHAPES] +
                         [(1, 256, 5120), (127, 512, 5120), (129, 512, 5120), (4681, 256, 13824), (200, 512, 1040)])
def test_gemm_sums_are_exact(M, N, K):
    """EPI_F32 with unit scales and no bias: float(acc) of the exact s32 sums, equal to torch._int_mm bit for bit
    (K = 1040 is not a multiple of the 128-wide k-block: the TMA zero-fills the tail)."""
    from realtime_video_b200 import ops
    a, w = _operands(M, N, K, M + N + K)
    one_a, one_w = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    got = ops.gemm_i8_rowwise(ops.I8Rows(a, one_a, torch.bfloat16), w, one_w, epilogue=ops.EPI_F32)
    if M >= 17:
        want = torch._int_mm(a, w.t())
    else:                                                       # torch._int_mm needs M > 16
        want = torch._int_mm(torch.cat([a, a.new_zeros(17 - M, K)]), w.t())[:M]
    assert torch.equal(got, want.float())
    sa = torch.rand(M, device="cuda") * 0.1 + 1e-3
    sw = torch.rand(N, device="cuda") * 0.01 + 1e-4
    got = ops.gemm_i8_rowwise(ops.I8Rows(a, sa, torch.bfloat16), w, sw, epilogue=ops.EPI_F32)
    assert torch.equal(got, I8.dequantize(want.long(), sa, sw))   # (float(acc) * s_a) * s_w, bit for bit


def _epi_case(M, N, K, seed):
    from realtime_video_b200 import fp8, ops
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g).bfloat16().cuda()
    w = (torch.randn(N, K, generator=g) * 0.02).bfloat16().cuda()
    b = torch.randn(N, generator=g).bfloat16().cuda()
    wq, sw = fp8.quantize_weight_int8_rows(w)
    xr = ops.i8_quantize_rows(x)
    v = I8.dequantize(I8.int_mm(xr.q.cpu(), wq.cpu()), xr.scale.cpu(), sw.cpu())   # the kernel's fp32 values
    return xr, wq, sw, b, v


@pytest.mark.parametrize("M,N,K,epi", [(4680, 15360, 5120, "split"), (4680, 5120, 5120, "gate_res"),
                                       (4680, 13824, 5120, "gelu"), (4680, 5120, 13824, "res"),
                                       (585, 5120, 5120, "bias"), (129, 256, 512, "bias")])
def test_epilogues_vs_oracle(M, N, K, epi):
    from realtime_video_b200 import ops
    xr, wq, sw, b, v = _epi_case(M, N, K, M + N + K)
    acc = v.double() + b.double().cpu()
    r16 = lambda t: t.to(torch.bfloat16).double()
    if epi == "bias":
        out = ops.gemm_i8_rowwise(xr, wq, sw, b)
        want = acc
        # one bf16 rounding of the oracle's fp32 restatement: at most 1 ulp apart
        ref = (v + b.float().cpu()).to(torch.bfloat16).float()
        ulp = torch.finfo(torch.bfloat16).eps * ref.abs().clamp(min=2.0 ** -126)
        assert bool(((out.float().cpu() - ref).abs() <= ulp).all())
    elif epi == "gelu":
        out = ops.gemm_i8_rowwise(xr, wq, sw, b, epilogue=ops.EPI_BIAS_GELU)
        want = torch.nn.functional.gelu(r16(acc), approximate="tanh")
    elif epi == "res":
        r = torch.randn(M, N, device="cuda").bfloat16()
        out = ops.gemm_i8_rowwise(xr, wq, sw, b, epilogue=ops.EPI_BIAS_RES, residual=r)
        want = r.double().cpu() + r16(acc)
    elif epi == "gate_res":
        r = torch.ones(M, N, device="cuda").bfloat16()
        gate = torch.randn(3, N, device="cuda").bfloat16()
        want = r.double().cpu() + r16(r16(acc) * gate.double().cpu().repeat_interleave(1560, 0))
        out = ops.gemm_i8_rowwise(xr, wq, sw, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, gate=gate,
                                  rows_per_gate=1560, out=r)
    else:
        out = torch.empty(M, 10240, device="cuda", dtype=torch.bfloat16)
        vv = torch.zeros(M + 8, 5120, device="cuda", dtype=torch.bfloat16)
        ops.gemm_i8_rowwise(xr, wq, sw, b, out=out, out2=vv[4:4 + M], n_split=10240)
        assert rel_l2(vv[4:4 + M].double().cpu(), acc[:, 10240:]) < 2e-3
        assert float(vv[:4].abs().max()) == 0 and float(vv[4 + M:].abs().max()) == 0      # guard rows untouched
        want = acc[:, :10240]
    torch.cuda.synchronize()
    assert rel_l2(out.double().cpu(), want) < 2e-3


def test_rows_past_m_are_neither_read_nor_written():
    """M = 129 inside a 256-row buffer: a NaN activation scale and NaN operands past row M leave no trace, and the
    output rows past M keep their guard value."""
    from realtime_video_b200 import ops
    M, N, K = 129, 512, 1024
    a, w = _operands(256, N, K, 7)
    sa = torch.rand(256, device="cuda") + 0.5
    sa[M:] = float("nan")
    sw = torch.rand(N, device="cuda") * 0.01
    out = torch.full((256, N), 3.0, device="cuda", dtype=torch.bfloat16)
    ops.gemm_i8_rowwise(ops.I8Rows(a[:M], sa, torch.bfloat16), w, sw, out=out[:M])
    assert torch.isfinite(out[:M].float()).all() and bool((out[M:] == 3.0).all())
    ref = I8.dequantize(I8.int_mm(a[:M].cpu(), w.cpu()), sa[:M].cpu(), sw.cpu()).bfloat16()
    assert torch.equal(out[:M].cpu(), ref)


def _family(name, M, K, g):
    if name == "gauss":
        return torch.randn(M, K, generator=g)
    if name == "gelu":
        return torch.nn.functional.gelu(torch.randn(M, K, generator=g) * 2, approximate="tanh")
    if name == "student_t":
        return torch.distributions.StudentT(3.0).sample((M, K))
    x = torch.randn(M, K, generator=g)
    x[:, [11, 700, 2900, 4100]] = 100.0                       # 4 channels = 100 in every token
    return x


@pytest.mark.parametrize("family", ["gauss", "gelu", "student_t", "outlier_channels"])
def test_numerics_against_the_oracle_and_fp8_per_row(family):
    """Against the exact product of the bf16 operands: the kernel's error within 1.05x of the oracle's; on Gaussian
    activations below half of kr_gemm_fp8_rowwise's error on the same inputs."""
    from realtime_video_b200 import fp8, ops
    torch.manual_seed(3)
    g = torch.Generator().manual_seed(3)
    M, K, N = 512, 5120, 512
    x = _family(family, M, K, g).bfloat16()
    w = (torch.randn(N, K, generator=g) * 0.02).bfloat16()
    exact = x.double() @ w.double().t()
    e_oracle = rel_l2(I8.linear_int8(x, w).double(), exact)
    wq, sw = fp8.quantize_weight_int8_rows(w.cuda())
    e_kernel = rel_l2(ops.linear_i8(x.cuda(), wq, sw).double().cpu(), exact)
    wq8, sw8 = fp8.quantize_weight_rows(w.cuda())
    e_fp8 = rel_l2(ops.linear_fp8_rowwise(x.cuda(), wq8, sw8).double().cpu(), exact)
    print(f"\n{family}: INT8 kernel {e_kernel:.3e}, oracle {e_oracle:.3e}, FP8 PerRow {e_fp8:.3e}")
    assert e_kernel <= 1.05 * e_oracle, (e_kernel, e_oracle)
    if family == "gauss":
        assert e_kernel < 0.5 * e_fp8, (e_kernel, e_fp8)


def test_int8_layer_vs_bf16_layer_at_14b_dims():
    """One Wan-14B-dim layer, Lq 4680, against the bf16 path (the FP8 tier's bound), and two runs bit-identical."""
    from realtime_video_b200 import fp8
    from tests.test_fp8_rowwise_gpu import _layer_model, _layer_run
    m = _layer_model()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(16, 3, 60, 104, generator=g).bfloat16().cuda()
    ctx = torch.randn(40, 4096, generator=g).bfloat16().cuda()
    ref = _layer_run(m, x, ctx)
    fp8.quantize_(m, fp8.Int8DynamicActivationInt8WeightConfig())
    got = _layer_run(m, x, ctx)
    again = _layer_run(m, x, ctx)
    r = rel_l2(got, ref)
    print(f"\n14B-dim layer rel-L2 vs bf16: INT8 {r:.4e}")
    assert torch.isfinite(got).all() and r < 8e-2, r
    assert torch.equal(got, again)


def test_server_loop_latents_vs_golden():
    from realtime_video_b200 import fp8
    from tests.golden_io import load_npz
    from tests.test_fp8_fast_accum_gpu import _server_loop
    gold = load_npz("server_loop_small.npz")
    draws = [gold[f"keep/draw{i}"] for i in range(int(gold["keep/ndraws"]))]
    want = gold["keep/latents"].float()
    _, lat, _ = _server_loop(False, fp8.Int8DynamicActivationInt8WeightConfig(), blocks=4, seed=11,
                             draws=list(draws), encoder=True)
    r = rel_l2(lat.float().cpu(), want)
    print(f"\nserver loop latents rel-L2 vs golden: INT8 {r:.3e}")
    assert r < 8e-2, r


def test_server_loop_cuda_graph_replay_with_int8_is_bit_identical_to_eager():
    from realtime_video_b200 import fp8
    from tests.test_fp8_fast_accum_gpu import _server_loop
    cfg = fp8.Int8DynamicActivationInt8WeightConfig()
    px_e, lat_e, _ = _server_loop(False, cfg)
    px_g, lat_g, tr = _server_loop(True, cfg)
    assert sum("graph" in st for st in tr._graphs.values()) >= 3
    assert torch.isfinite(lat_e).all() and torch.equal(lat_e, lat_g)
    for a, b in zip(px_e, px_g):
        assert torch.equal(a, b)
