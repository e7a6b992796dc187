"""Stream-K GEMM (kr_gemm_sk.cu through kr_gemm_ws) against an fp32 matmul of the same bf16 operands, on the row
shards the multi-GPU mode produces (M = 4680/N rows: 2340, 1170, 585) for every DiT projection and epilogue, plus
ragged cases that put 1, 2 and 3+ contributors on a tile.  Each case runs several times on the same workspace: the
tile counters must return to zero and the result must be bit-identical from launch to launch (partials are summed
in CTA order).  Tolerance: bf16 outputs of a K <= 13824 dot product, rel-L2 <= 2e-3 (fp32 accumulation order differs
from torch's)."""
import os

os.environ.setdefault("KR_GEMM_SK", "1")     # the plan only considers stream-K when asked (read once at first use)

import pytest  # noqa: E402
import torch  # noqa: E402

from tests.golden_io import rel_l2  # noqa: E402

pytestmark = pytest.mark.gpu


def _case(M, N, K, epi, repeats=3):
    from realtime_video_b200 import _lib, ops
    lib = _lib.load()
    if lib.kr_gemm_kernel_id_ws({"bias": 0, "gelu": 1, "gate_res": 2, "split": 0}[epi], M, N, K, 1) != 3:
        pytest.skip("stream-K not selected (KR_GEMM_SK was read as 0 earlier in this process, or the shape is data-parallel)")
    torch.manual_seed(M + N + K)
    a = torch.randn(M, K, device="cuda").bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.02).bfloat16()
    b = torch.randn(N, device="cuda").bfloat16()
    ref = a.float() @ w.float().t() + b.float()
    gate = torch.randn(3, N, device="cuda").bfloat16()
    outs = []
    for _ in range(repeats):
        if epi == "bias":
            out, want = ops.gemm(a, w, b), ref
        elif epi == "gelu":
            out = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GELU)
            want = torch.nn.functional.gelu(ref.bfloat16().float(), approximate="tanh")
        elif epi == "gate_res":
            x = torch.ones(M, N, device="cuda").bfloat16()
            rpg = (M + 2) // 3
            rows = torch.arange(M, device="cuda") // rpg
            want = x.float() + (ref.bfloat16().float() * gate.float()[rows]).bfloat16().float()
            out = ops.gemm(a, w, b, epilogue=ops.EPI_BIAS_GATE_RES, residual=x, gate=gate, rows_per_gate=rpg, out=x)
        else:   # split output: last third straight into a strided "cache slot"
            out = torch.empty(M, N - N // 3, device="cuda", dtype=torch.bfloat16)
            v = torch.zeros(M + 64, N // 3, device="cuda", dtype=torch.bfloat16)
            ops.gemm(a, w, b, out=out, out2=v[32:32 + M], n_split=N - N // 3)
            assert rel_l2(v[32:32 + M].float(), ref[:, N - N // 3:]) < 2e-3
            assert float(v[:32].abs().max()) == 0 and float(v[32 + M:].abs().max()) == 0
            want = ref[:, :N - N // 3]
        torch.cuda.synchronize()
        assert rel_l2(out.float(), want) < 2e-3
        outs.append(out.clone())
    for o in outs[1:]:
        assert torch.equal(o, outs[0]), "stream-K result changed between launches on the same workspace"
    ws = ops._sk_ws[(torch.cuda.current_device(), torch.cuda.current_stream().cuda_stream)]
    assert int(ws[:65536].view(torch.int32).abs().sum()) == 0, "tile counters not reset"
    return lib.kr_gemm_kernel_id_ws({"bias": 0, "gelu": 1, "gate_res": 2, "split": 0}[epi], M, N, K, 1)


@pytest.mark.parametrize("M", [585, 1170, 2340])
@pytest.mark.parametrize("N,K,epi", [(15360, 5120, "split"), (5120, 5120, "gate_res"), (13824, 5120, "gelu"),
                                     (5120, 13824, "gate_res"), (5120, 5120, "bias")])
def test_streamk_on_the_sequence_parallel_shards(M, N, K, epi):
    _case(M, N, K, epi)


@pytest.mark.parametrize("M,N,K", [(100, 256, 512), (585, 512, 5120), (129, 768, 8192), (1000, 1024, 640),
                                   (4680, 2560, 5120)])
def test_streamk_ragged_shapes(M, N, K):
    """few tiles x many k-blocks (one tile shared by dozens of CTAs), M tails, K = 10 k-blocks (ranges shorter
    than a tile), and a many-tile shape with a bad wave count."""
    from realtime_video_b200 import _lib
    if not _lib.load().kr_gemm_kernel_id_ws(0, M, N, K, 1) == 3:
        pytest.skip("plan keeps the data-parallel kernel for this shape")
    _case(M, N, K, "bias")


def test_plan_keeps_data_parallel_kernels_where_they_fill_the_machine():
    from realtime_video_b200 import _lib
    lib = _lib.load()
    assert lib.kr_gemm_kernel_id_ws(0, 4680, 5120, 5120, 1) == 4        # 740 tiles = 5.6 waves: wave-fitted width
    assert lib.kr_gemm_kernel_id_ws(0, 4680, 15360, 5120, 1) == 1       # 2220 tiles = 16.8 waves: fixed-width kernel
    if os.environ.get("KR_GEMM_SK") == "1" and lib.kr_gemm_kernel_id_ws(0, 585, 5120, 5120, 1) == 3:
        pass                                                            # stream-K enabled in this process
    assert lib.kr_gemm_kernel_id_ws(0, 585, 5120, 5120, 0) in (1, 4)    # no workspace -> never stream-K (single-CTA family)
