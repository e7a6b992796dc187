"""Block-scaled FP8 (torchao ``granularity=[PerBlock([1, 128]), PerBlock([128, 128])]``) without a GPU: the oracle's
per-group invariants, config parsing, ``fp8.quantize_`` with PerBlock, the torchao import line served by the drop-in
finder, the DiT block schedule on stand-in kernels (one GPU and sequence-parallel on gloo ranks), argument validation
of the three C entry points, and the SASS / resource usage of their kernels."""
import ctypes
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from oracle import fp8_blockwise_oracle as F8B
from oracle import fp8_rowwise_oracle as F8R
from tests import cpu_ops_emulation_fp8 as emu
from tests.golden_io import rel_l2
from tests.test_fp8_rowwise_cpu import _run, _small_model

ROOT = Path(__file__).resolve().parent.parent


def _counting(monkeypatch, names):
    calls = {n: 0 for n in names}
    for n in names:
        real = getattr(emu, n)

        def counted(*a, _real=real, _n=n, **k):
            calls[_n] += 1
            return _real(*a, **k)
        monkeypatch.setattr(emu, n, counted)
    return calls


def _pair(a=(1, 128), w=(128, 128)):
    from realtime_video_b200 import fp8
    return [fp8.PerBlock(list(a)), fp8.PerBlock(list(w))]


def _outlier_channels(rows, cols, seed, big=1e5):
    """N(0, 1) activations whose channels 3 and 700 are `big` in every token: with one scale per row those two
    channels set every row's scale and push the other channels towards e4m3's subnormals."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, cols, generator=g)
    x[:, 3] *= big
    x[:, 700] *= big
    return x


def test_oracle_per_group_invariants():
    x = _outlier_channels(64, 1024, 0)
    x[5, 256:384] = 0
    q, s = F8B.quantize_per_group(x)
    assert q.dtype == torch.float8_e4m3fn and s.shape == (8, 64) and s.dtype == torch.float32
    amax = q.float().reshape(64, 8, 128).abs().amax(dim=-1)
    assert int(amax[5, 2]) == 0                                           # a zero group quantises to zeros
    amax[5, 2] = 448.0
    assert bool((amax == 448.0).all())                                    # every other group's amax maps onto 448
    back = F8B.dequantize_groups(q, s)
    qr, sr = F8R.quantize_per_row(x)
    ok = torch.ones(1024, dtype=torch.bool)
    ok[:128] = ok[640:768] = False                                        # the groups without an outlier channel
    e_blk = rel_l2(back[:, ok].float(), x[:, ok])
    e_row = rel_l2((qr.float() * sr[:, None])[:, ok], x[:, ok])
    assert e_blk < 4e-2 and e_blk < 0.25 * e_row, (e_blk, e_row)          # measured 2.6e-2 vs 1.6e-1
    w = torch.randn(256, 384) * 0.02
    w[128:, :128] = 0
    wq, sw = F8B.quantize_per_block(w)
    assert sw.shape == (2, 3) and float(sw[1, 0]) == pytest.approx(1e-12 / 448)
    assert int(wq[128:, :128].float().abs().max()) == 0


def test_config_accepts_exactly_the_1x128_128x128_pair(monkeypatch):
    from realtime_video_b200 import fp8
    c = fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair())
    assert isinstance(c.granularity, fp8.PerBlock) and c.granularity.block_size == (1, 128)
    c = fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair(),
                                                      mm_config=fp8.Float8MMConfig(use_fast_accum=False))
    assert isinstance(c.granularity, fp8.PerBlock)
    for bad in ([fp8.PerBlock([1, 64]), fp8.PerBlock([128, 128])], [fp8.PerBlock([1, 128]), fp8.PerBlock([64, 64])],
                [fp8.PerBlock([128, 128]), fp8.PerBlock([1, 128])]):
        with pytest.raises(NotImplementedError):
            fp8.Float8DynamicActivationFloat8WeightConfig(granularity=bad)
    for bad in (fp8.PerBlock([1, 128]), [fp8.PerBlock([1, 128])], [fp8.PerBlock([1, 128]), fp8.PerRow()],
                [fp8.PerRow(), fp8.PerBlock([128, 128])], [fp8.PerTensor(), fp8.PerBlock([128, 128])]):
        with pytest.raises(ValueError):
            fp8.Float8DynamicActivationFloat8WeightConfig(granularity=bad)
    with pytest.raises(NotImplementedError, match="fast_accum"):
        fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair(),
                                                      mm_config=fp8.Float8MMConfig(use_fast_accum=True))


def _wrapper():
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    w = WanDiffusionWrapper(model_name="synthetic", is_causal=True,
                            model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    for blk in w.model.blocks:
        blk.self_attn.fuse_projections()
    return w


def test_quantize_per_block_attaches_block_scaled_weights_to_the_block_linears_only(monkeypatch):
    """The environment switch for fast accumulation does not apply to PerBlock: the recorded mode stays promoted."""
    from realtime_video_b200 import fp8
    monkeypatch.setenv("KR_FP8_FAST_ACCUM", "1")
    w = _wrapper()
    keys = set(w.state_dict().keys())
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
    blk = w.model.blocks[0]
    lins = (blk.self_attn.to_qkv, blk.self_attn.o, blk.cross_attn.q, blk.cross_attn.k, blk.cross_attn.v,
            blk.cross_attn.o, blk.ffn[0], blk.ffn[2])
    for lin in lins:
        wq, sw = lin._kr_fp8
        assert fp8.is_blockwise(lin) and not fp8.is_rowwise(lin) and not fp8.is_fast_accum(lin)
        ref_q, ref_s = F8B.quantize_per_block(lin.weight.detach())
        N, K = lin.weight.shape
        assert wq.dtype == torch.uint8 and torch.equal(wq, ref_q.view(torch.uint8))
        assert sw.dtype == torch.float32 and sw.shape == (N // 128, K // 128) and torch.equal(sw, ref_s)
        q2, s2 = fp8.quantize_weight_blocks(lin.weight)
        assert torch.equal(q2, wq) and torch.equal(s2, sw)
    assert not hasattr(w.model.head.head, "_kr_fp8") and not hasattr(w.model.time_embedding[0], "_kr_fp8")
    assert set(w.state_dict().keys()) == keys
    fp8.dequantize_(w)
    for lin in lins:
        assert not any(hasattr(lin, a) for a in ("_kr_fp8", "_kr_fp8_granularity", "_kr_fp8_fast_accum"))
    # the switch still applies to the other granularities
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    assert fp8.is_fast_accum(blk.ffn[0])
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
    assert fp8.is_blockwise(blk.ffn[0]) and not fp8.is_fast_accum(blk.ffn[0])


def test_quantize_per_block_skips_linears_whose_k_is_not_whole_blocks():
    from realtime_video_b200 import fp8
    w = _wrapper()
    blk = w.model.blocks[0]
    blk.ffn[2] = torch.nn.Linear(448, 256)                  # K = 448: not a whole number of 128-wide blocks
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
    assert not hasattr(blk.ffn[2], "_kr_fp8") and fp8.is_blockwise(blk.ffn[0])
    with pytest.raises(ValueError):
        fp8.quantize_weight_blocks(torch.zeros(256, 448))


def test_server_per_block_import_line_resolves_through_the_dropin():
    code = ("import realtime_video_b200.dropin as d; d.install()\n"
            "from torchao.quantization.quant_api import quantize_, Float8DynamicActivationFloat8WeightConfig, PerBlock\n"
            "import realtime_video_b200.fp8 as f\n"
            "c = Float8DynamicActivationFloat8WeightConfig(granularity=[PerBlock([1, 128]), PerBlock([128, 128])])\n"
            "assert quantize_ is f.quantize_ and PerBlock is f.PerBlock and isinstance(c.granularity, f.PerBlock)\n"
            "print('OK')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                       env={"PYTHONPATH": str(ROOT), "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stderr[-2000:]


@pytest.mark.parametrize("fused", [True, False])
def test_block_schedule_with_per_block_fp8(monkeypatch, fused):
    """Host logic with stand-in kernels: per block, the three LayerNorms feeding FP8 linears cast to e4m3 per
    128-channel group themselves (to_qkv or q/k/v, cross q, ffn.0), the self- and cross-attention o and ffn.2 use the
    group quantiser, the prompt is cast once for both K/V projections, every quantised linear runs the block-scaled
    GEMM, and no per-tensor or per-row entry point runs.  The result equals the schedule with an unfused "LayerNorm,
    then quantise groups" stand-in bit for bit and stays within the toy FP8 bound of bf16."""
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    monkeypatch.setattr(dit, "ops", emu)
    monkeypatch.delenv("KR_FP8_FAST_ACCUM", raising=False)
    m, g = _small_model(fused)
    ref, _ = _run(m, g)
    calls = _counting(monkeypatch, ["linear_fp8", "linear_fp8_rowwise", "fp8_quantize_rows", "ln_modulate_fp8",
                                    "fp8_quantize_blocks", "ln_modulate_fp8_blocks", "gemm_fp8_blockwise"])
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
    got, kv = _run(m, g)
    n_qkv = 1 if fused else 3
    assert calls == {"linear_fp8": 0, "linear_fp8_rowwise": 0, "fp8_quantize_rows": 0, "ln_modulate_fp8": 0,
                     "ln_modulate_fp8_blocks": 2 * 3, "fp8_quantize_blocks": 2 * 4,
                     "gemm_fp8_blockwise": 2 * (n_qkv + 7)}, calls
    assert kv[0]["local_end_index"] == 3 * 96 and float(kv[0]["v"].abs().sum()) > 0
    assert rel_l2(got, ref) < 0.15

    def unfused(x, *, q=None, scale=None, out=None, **kw):
        return emu.fp8_quantize_blocks(emu.ln_modulate(x, out=out, **kw), q, scale)
    monkeypatch.setattr(emu, "ln_modulate_fp8_blocks", unfused)
    got2, _ = _run(m, g)
    assert torch.equal(got, got2)


def test_cross_q_without_norm3_uses_the_group_quantiser(monkeypatch):
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model(cross_attn_norm=False)
    calls = _counting(monkeypatch, ["fp8_quantize_blocks", "ln_modulate_fp8_blocks", "ln_modulate"])
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
    got, _ = _run(m, g)
    assert torch.isfinite(got).all()
    # per block: o, cross q, cross o, ffn.2, the prompt (first pass); LayerNorms: norm1 + norm2 fused, the head's
    assert calls == {"fp8_quantize_blocks": 2 * 5, "ln_modulate_fp8_blocks": 2 * 2, "ln_modulate": 1}, calls


def _sp_worker(rank, world, port, ret):
    import os

    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import realtime_video_b200.dit as dit
        from realtime_video_b200 import fp8
        from realtime_video_b200.parallel import SequenceParallel
        dit.ops = emu
        m, g = _small_model()
        fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
        m.sp = SequenceParallel()
        n = m.kv_cache_heads
        kv = [{"k": torch.zeros(1, 6 * 96, n, 128), "v": torch.zeros(1, 6 * 96, n, 128),
               "global_end_index": 0, "local_end_index": 0} for _ in m.blocks]
        ca = [{"k": torch.zeros(1, 512, 2, 128), "v": torch.zeros(1, 512, 2, 128), "is_init": False} for _ in m.blocks]
        outs = []
        with torch.no_grad():
            for name, t, start in (("in/x0", 1000.0, 0), ("in/x2", 1000.0, 3 * 96)):
                x = g[name].float()
                outs.append(m(x[None], t=torch.full((1, 3), t), context=g["in/ctx"].float()[None], seq_len=32760,
                              kv_cache=kv, crossattn_cache=ca, current_start=start)[0])
        ret[rank] = torch.stack(outs)
    finally:
        dist.destroy_process_group()


def test_sequence_parallel_per_block_fp8_equals_one_rank_gloo(monkeypatch):
    """No scale spans rows, so 2 gloo ranks give the one-rank result bit for bit with the PerBlock stand-ins."""
    import torch.multiprocessing as mp

    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    from tests.test_parallel import _free_port
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model()
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=_pair()))
    one, _ = _run(m, g, passes=(("in/x0", 1000.0, 0), ("in/x2", 1000.0, 3 * 96)))
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_sp_worker, args=(2, _free_port(), ret), nprocs=2, join=True)
    for r in range(2):
        assert torch.equal(ret[r], one), (r, rel_l2(ret[r], one))


@pytest.fixture(scope="module")
def lib():
    from realtime_video_b200 import _lib
    _lib.build()
    return _lib.load()


def test_argument_validation_of_the_block_fp8_entry_points(lib):
    """Rejected before any CUDA call, so no GPU is needed (pointers are never dereferenced)."""
    p = ctypes.c_void_p(4096)
    s = ctypes.c_void_p(8192)
    # group quantiser: widths not a multiple of 128, too wide, short pitches, scale pitch < rows; null scales
    for rows, cols, ldx, ldq, lds in ((4, 1536 - 8, 1536, 1536, 4), (4, 14336 + 128, 14464, 14464, 4),
                                      (4, 1536, 1528, 1536, 4), (4, 1536, 1536, 1528, 4), (4, 1536, 1536, 1536, 3),
                                      (0, 1536, 1536, 1536, 4)):
        assert lib.kr_fp8_quantize_blocks(p, ldx, rows, cols, p, ldq, s, lds, None) < 0
    assert lib.kr_fp8_quantize_blocks(p, 1536, 4, 1536, p, 1536, None, 4, None) == -1
    # fused LayerNorm: width not whole groups, short q pitch, scale pitch < rows, null scales, half an affine pair
    args = lambda D, ldq, scale, lds=4, w=None, b=None: (p, D, None, 0, 4, D, ctypes.c_float(1e-6), w, b, None, 0, 0,
                                                         1, 0, 0, p, ldq, scale, lds, None)
    assert lib.kr_ln_modulate_fp8_blocks(*args(1536 - 8, 1536, s)) == -1
    assert lib.kr_ln_modulate_fp8_blocks(*args(1536, 1024, s)) == -2
    assert lib.kr_ln_modulate_fp8_blocks(*args(1536, 1536, s, lds=3)) == -1
    assert lib.kr_ln_modulate_fp8_blocks(*args(1536, 1536, None)) == -1
    assert lib.kr_ln_modulate_fp8_blocks(*args(1536, 1536, s, w=p)) == -1

    def gemm(epi, scale_a, scale_w, N=256, K=512, ld_sa=128, residual=None):
        return lib.kr_gemm_fp8_blockwise(epi, p, 512, p, 512, scale_a, ld_sa, scale_w, None, p, N, 128, N, K,
                                         residual, 0, None, 0, 0, None, 0, 0, 0, None)
    assert gemm(0, None, s) == -1 and gemm(0, s, None) == -1
    assert gemm(3, s, s) == -1 and b"residual" in lib.kr_last_error()
    assert gemm(2, s, s) == -1
    assert gemm(5, s, s) == -1                               # EPI_MUL is not an FP8 epilogue
    assert gemm(0, s, s, N=200) == -1
    assert gemm(0, s, s, K=496) == -1                        # K not whole 128-wide blocks
    assert gemm(0, s, s, ld_sa=100) == -1                    # activation scale pitch < M


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_and_resources_of_the_block_scaled_gemm_instantiations():
    from tests.test_sass_cpu import _ops, resource_usage, sass_functions
    funcs, usage = sass_functions(), resource_usage()
    gemms = [f for f in funcs if re.search(r"gemm_fp8_kernelILi\dELi2ELb0E", f)]   # block scales, promoted
    assert len(gemms) == 5                                   # bias, GELU, gate + residual, residual, fp32
    for f in gemms:
        ops = {o.split(".")[0] for o in _ops(funcs[f])}
        assert {"QGMMA", "UTMALDG", "SYNCS"} <= ops, f       # e4m3 wgmma fed by TMA
        assert not ops & {"HMMA", "LDL", "STL"}, f           # no mma.sync, no local memory
        assert usage[f][1:] == (0, 0), (f, usage[f])         # no stack, no local memory
    rows = [f for f in funcs if "fp8_quantize_blocks_kernel" in f or "ln_modulate_fp8_blocks_kernel" in f]
    assert len(rows) == 15
    for f in rows:
        ops = {o.split(".")[0] for o in _ops(funcs[f])}
        assert "SHFL" in ops and "ATOMG" not in ops and "RED" not in ops, f
        assert not ops & {"LDL", "STL"} and usage[f][1:] == (0, 0), (f, usage[f])
