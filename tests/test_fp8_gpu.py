"""FP8 row (SURVEY.md 8f.4) on the GPU, through the C ABI, against oracle/fp8_oracle.py (torchao's published
per-tensor dynamic-activation algorithm; "parity unpinned": torchao is not in the image).
  * kr_fp8_quantize: e4m3 bytes and scale BIT-EXACT vs the oracle (same fp32 multiply, round-to-nearest-even cast);
  * kr_gemm_fp8 (e4m3 wgmma, fp32 promotion per k-block): products of e4m3 values are exact in fp32, only the accumulation order
    differs -> rel-L2 <= 2e-3 on the bf16 output, every fused epilogue, the DiT shapes;
  * FP8 tier vs the bf16 path on one 14B-dim layer: rel-L2 <= 8e-2 (e4m3 has 3 mantissa bits; stated, not hidden)."""
import pytest
import torch

from oracle import fp8_oracle as F8
from tests.golden_io import rel_l2

pytestmark = pytest.mark.gpu


def test_dynamic_activation_quantisation_is_bit_exact():
    from realtime_video_b200 import ops
    torch.manual_seed(0)
    x = (torch.randn(4680, 5120, device="cuda") * 2.5).bfloat16()
    x[17, 33] = 40.0                                      # a clear amax
    q, state = ops.fp8_quantize(x)
    ref_q, ref_s = F8.quantize_per_tensor(x.cpu())
    assert float(state[0]) == 40.0 and float(state[1]) == float(ref_s)
    assert torch.equal(q.cpu().view(torch.float8_e4m3fn).float(), ref_q.float())


@pytest.mark.parametrize("M,N,K,epi", [(4680, 15360, 5120, "split"), (4680, 5120, 5120, "gate_res"),
                                       (4680, 13824, 5120, "gelu"), (4680, 5120, 13824, "res"), (585, 5120, 5120, "bias"),
                                       (100, 256, 512, "bias")])
def test_fp8_gemm_vs_oracle(M, N, K, epi):
    from realtime_video_b200 import fp8, ops
    torch.manual_seed(M + N)
    x = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    wq, sw = fp8.quantize_weight(w)
    lin = F8.linear_fp8(x.cpu(), w.cpu(), None).float().cuda()          # bf16(x_q w_q^T s) without bias
    acc = (F8.quantize_per_tensor(x.cpu())[0].float() @ F8.quantize_per_tensor(w.cpu())[0].float().t()).cuda() * \
        (float(F8.quantize_per_tensor(x.cpu())[1]) * sw) + b.float()
    if epi == "bias":
        out, want = ops.linear_fp8(x, wq, sw, b), acc
    elif epi == "gelu":
        out = ops.linear_fp8(x, wq, sw, b, epilogue=ops.EPI_BIAS_GELU)
        want = torch.nn.functional.gelu(acc.bfloat16().float(), approximate="tanh")
    elif epi == "res":
        r = torch.randn(M, N, device="cuda").bfloat16()
        out = ops.linear_fp8(x, wq, sw, b, epilogue=ops.EPI_BIAS_RES, residual=r)
        want = r.float() + acc.bfloat16().float()
    elif epi == "gate_res":
        r = torch.ones(M, N, device="cuda").bfloat16()
        gate = torch.randn(3, N, device="cuda").bfloat16()
        want = r.float() + (acc.bfloat16().float() * gate.float().repeat_interleave(1560, 0)).bfloat16().float()
        out = ops.linear_fp8(x, wq, sw, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=r, gate=gate, rows_per_gate=1560, out=r)
    else:
        out = torch.empty(M, 10240, device="cuda", dtype=torch.bfloat16)
        v = torch.zeros(M + 8, 5120, device="cuda", dtype=torch.bfloat16)
        ops.linear_fp8(x, wq, sw, b, out=out, out2=v[4:4 + M], n_split=10240)
        assert rel_l2(v[4:4 + M].float(), acc[:, 10240:]) < 2e-3 and float(v[:4].abs().max()) == 0
        want = acc[:, :10240]
    torch.cuda.synchronize()
    assert rel_l2(out.float(), want) < 2e-3
    del lin


def test_fp8_layer_vs_bf16_layer_at_14b_dims():
    """One Wan-14B-dim layer, Lq 4680: FP8 linears (quantize_) against the bf16 path on the same weights / inputs —
    the FP8 tier's own tolerance, reported next to the bf16 headline and never replacing it."""
    from realtime_video_b200 import fp8
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
    ref = run()
    fp8.quantize_(m)
    got = run()
    r = rel_l2(got, ref)
    assert torch.isfinite(got).all() and r < 8e-2, r
