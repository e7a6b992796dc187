"""INT8 linears (torchao Int8DynamicActivationInt8WeightConfig) without a GPU: the oracle against torch._int_mm and
its own formulas, the config, quantize_ / dequantize_ across tiers, the block schedule's routing with the stand-ins
of tests/cpu_ops_emulation_int8.py, sequence parallelism, the C entry points' argument checks and the machine code."""
import ctypes
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from oracle import int8_oracle as I8
from tests import cpu_ops_emulation_int8 as emu
from tests.golden_io import load_npz, rel_l2, weights

ROOT = Path(__file__).resolve().parent.parent


def test_oracle_integer_product_equals_torch_int_mm():
    g = torch.Generator().manual_seed(0)
    for M, K, N in ((32, 64, 16), (48, 5120, 40), (17 * 8, 13824, 24)):
        a = torch.randint(-127, 128, (M, K), generator=g, dtype=torch.int8)
        w = torch.randint(-128, 128, (N, K), generator=g, dtype=torch.int8)
        ref = torch._int_mm(a, w.t().contiguous())
        assert ref.dtype == torch.int32 and torch.equal(I8.int_mm(a, w), ref.long())
    # the extreme sums of the overflow bound stay exact
    a = torch.full((32, 4096), -127, dtype=torch.int8)
    w = torch.full((8, 4096), -128, dtype=torch.int8)
    assert int(I8.int_mm(a, w)[0, 0]) == 127 * 128 * 4096 == int(torch._int_mm(a, w.t().contiguous())[0, 0])
    assert 127 * 128 * I8.I8_MAX_K < 2 ** 31 <= 127 * 128 * (I8.I8_MAX_K + 1)


def test_oracle_activation_formula_on_edge_rows():
    x = torch.zeros(6, 16)
    x[1, 3] = -0.75                                   # a single nonzero value
    x[2, :2] = torch.tensor([2.0, -2.0])              # +-amax
    amax = 127.0
    x[3, 0] = amax                                    # halfway ties: amax = 127 makes the multiplier exactly 1
    x[3, 1:6] = torch.tensor([0.5, 1.5, 2.5, -0.5, -2.5])
    x[4] = torch.linspace(-3, 5, 16)
    x[5, 0] = 1e-30                                   # below the amax floor
    q, s = I8.quantize_act_rows(x)
    assert q.dtype == torch.int8 and s.dtype == torch.float32
    assert torch.equal(q[0], torch.zeros(16, dtype=torch.int8)) and float(s[0]) == pytest.approx(1e-12 / 127)
    assert int(q[1, 3]) == -127 and int(q[1].abs().sum()) == 127 and float(s[1]) == torch.tensor(0.75) / 127
    assert q[2, :2].tolist() == [127, -127]
    assert q[3, :6].tolist() == [127, 0, 2, 2, 0, -2]     # round half to even
    mul = torch.tensor(127.0) / torch.tensor(5.0)         # a true fp32 division
    assert torch.equal(q[4], torch.round(x[4] * mul).clamp(-127, 127).to(torch.int8))
    assert int(q[5, 0]) == 0 and float(s[5]) == pytest.approx(1e-12 / 127)


def test_oracle_weight_formula_on_edge_rows():
    w = torch.zeros(4, 8)
    w[1, 2] = 1.0                                     # a single nonzero value: +amax -> round(127.5) = 128 -> 127
    w[2, :2] = torch.tensor([-1.0, 1.0])              # +-amax -> the ends of [-128, 127]
    w[3] = torch.tensor([127.5, 0.5, 1.5, 2.5, -0.5, -1.5, 63.75, 0.0])   # s_n = 1: ties to even
    q, s = I8.quantize_weight_rows(w)
    assert torch.equal(q[0], torch.zeros(8, dtype=torch.int8)) and float(s[0]) == torch.finfo(torch.float32).eps
    s1 = torch.tensor(1.0) / torch.tensor(127.5)
    assert int(q[1, 2]) == 127 and float(s[1]) == float(s1)
    assert q[2, :2].tolist() == [int(torch.round(torch.tensor(-1.0) / s1)), 127]
    assert int(q[2, 0]) in (-128, -127)
    assert float(s[3]) == 1.0 and q[3].tolist() == [127, 0, 2, 2, 0, -2, 64, 0]
    from realtime_video_b200 import fp8
    wq, ws = fp8.quantize_weight_int8_rows(w)
    assert torch.equal(wq, q) and torch.equal(ws, s)


def test_config_arguments():
    from realtime_video_b200 import fp8
    c = fp8.Int8DynamicActivationInt8WeightConfig()
    assert c.layout is None and c.act_mapping_type is fp8.MappingType.SYMMETRIC and not c.weight_only_decode
    fp8.Int8DynamicActivationInt8WeightConfig(layout=fp8.PlainLayout(), act_mapping_type=fp8.MappingType.SYMMETRIC,
                                              weight_only_decode=False, set_inductor_config=False)
    with pytest.raises(NotImplementedError):
        fp8.Int8DynamicActivationInt8WeightConfig(act_mapping_type=fp8.MappingType.ASYMMETRIC)
    with pytest.raises(NotImplementedError):
        fp8.Int8DynamicActivationInt8WeightConfig(weight_only_decode=True)
    with pytest.raises(NotImplementedError):
        fp8.Int8DynamicActivationInt8WeightConfig(layout=object())


def _wrapper():
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    w = WanDiffusionWrapper(model_name="synthetic", is_causal=True,
                            model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    for blk in w.model.blocks:
        blk.self_attn.fuse_projections()
    return w


def _block_linears(blk):
    return (blk.self_attn.to_qkv, blk.self_attn.o, blk.cross_attn.q, blk.cross_attn.k, blk.cross_attn.v,
            blk.cross_attn.o, blk.ffn[0], blk.ffn[2])


def test_quantize_attaches_int8_weights_and_replaces_the_other_tier():
    from realtime_video_b200 import fp8
    w = _wrapper()
    keys = set(w.state_dict().keys())
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    fp8.quantize_(w, fp8.Int8DynamicActivationInt8WeightConfig())
    blk = w.model.blocks[0]
    for lin in _block_linears(blk):
        wq, sw = lin._kr_i8
        assert fp8.is_int8(lin) and not hasattr(lin, "_kr_fp8") and not hasattr(lin, "_kr_fp8_granularity")
        ref_q, ref_s = I8.quantize_weight_rows(lin.weight.detach())
        assert wq.dtype == torch.int8 and torch.equal(wq, ref_q)
        assert sw.dtype == torch.float32 and sw.shape == (lin.weight.shape[0],) and torch.equal(sw, ref_s)
    assert not hasattr(w.model.head.head, "_kr_i8") and not hasattr(w.model.time_embedding[0], "_kr_i8")
    assert set(w.state_dict().keys()) == keys
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(
        granularity=fp8.PerRow(), mm_config=fp8.Float8MMConfig(use_fast_accum=True)))
    assert all(not fp8.is_int8(m) and fp8.is_rowwise(m) and fp8.is_fast_accum(m) for m in _block_linears(blk))
    fp8.quantize_(w, fp8.Int8DynamicActivationInt8WeightConfig())
    assert all(fp8.is_int8(m) and not fp8.is_fast_accum(m) for m in _block_linears(blk))
    fp8.dequantize_(w)
    assert not any(hasattr(m, a) for m in _block_linears(blk) for a in ("_kr_i8", "_kr_fp8", "_kr_fp8_fast_accum"))


def test_server_int8_import_line_resolves_through_the_dropin():
    code = ("import realtime_video_b200.dropin as d; d.install()\n"
            "from torchao.quantization.quant_api import quantize_, Int8DynamicActivationInt8WeightConfig\n"
            "import realtime_video_b200.fp8 as f\n"
            "assert quantize_ is f.quantize_\n"
            "assert isinstance(Int8DynamicActivationInt8WeightConfig(), f.Int8DynamicActivationInt8WeightConfig)\n"
            "print('OK')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                       env={"PYTHONPATH": str(ROOT), "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stderr[-2000:]


def _small_model(fused=True, cross_attn_norm=True):
    import realtime_video_b200.dit as dit
    g = load_npz("dit_small.npz")
    m = dit.CausalWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128,
                           cross_attn_norm=cross_attn_norm)
    m.load_state_dict(weights(g, torch.float32), strict=False)
    m = m.float().eval()
    if fused:
        for blk in m.blocks:
            blk.self_attn.fuse_projections()
    return m, g


def _run(m, g, passes=(("in/x0", 750.0, 0),)):
    kv = [dict(k=torch.zeros(1, 6 * 96, 2, 128), v=torch.zeros(1, 6 * 96, 2, 128), global_end_index=0,
               local_end_index=0) for _ in range(2)]
    ca = [dict(k=torch.zeros(1, 512, 2, 128), v=torch.zeros(1, 512, 2, 128), is_init=False) for _ in range(2)]
    outs = []
    with torch.no_grad():
        for name, t, start in passes:
            x = g[name].float()
            outs.append(m(x[None], t=torch.full((1, 3), t), context=g["in/ctx"].float()[None], seq_len=32760,
                          kv_cache=kv, crossattn_cache=ca, current_start=start)[0])
    return torch.stack(outs), kv


def _counting(monkeypatch, names):
    calls = {n: 0 for n in names}
    for n in names:
        real = getattr(emu, n)

        def counted(*a, _real=real, _n=n, **k):
            calls[_n] += 1
            return _real(*a, **k)
        monkeypatch.setattr(emu, n, counted)
    return calls


@pytest.mark.parametrize("fused", [True, False])
def test_block_schedule_with_int8(monkeypatch, fused):
    """Per block, the three LayerNorms feeding INT8 linears cast to s8 themselves (to_qkv or q/k/v, cross q, ffn.0),
    the self- and cross-attention o and ffn.2 use the row quantiser, the prompt is cast once for both K/V
    projections, and no FP8 entry point runs.  The result equals the schedule with an unfused "LayerNorm, then
    quantise rows" stand-in bit for bit and stays within the toy tolerance of the unquantised model."""
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model(fused)
    ref, _ = _run(m, g)
    calls = _counting(monkeypatch, ["i8_quantize_rows", "ln_modulate_i8", "gemm_i8_rowwise", "linear_fp8",
                                    "linear_fp8_rowwise", "ln_modulate_fp8", "gemm"])
    fp8.quantize_(m, fp8.Int8DynamicActivationInt8WeightConfig())
    emu.entry_points.clear()
    got, kv = _run(m, g)
    n_qkv = 1 if fused else 3
    # gemm: the bf16 linears outside the blocks (patch embedding, time / text MLPs, head) only
    assert {k: v for k, v in calls.items() if k != "gemm"} == {
        "i8_quantize_rows": 2 * 4, "ln_modulate_i8": 2 * 3, "gemm_i8_rowwise": 2 * (n_qkv + 7), "linear_fp8": 0,
        "linear_fp8_rowwise": 0, "ln_modulate_fp8": 0}, calls
    # every linear fed by a LayerNorm or by the prompt cast receives its input already cast
    pre_cast = sum(1 for _, cast in emu.entry_points if cast)
    assert len(emu.entry_points) == 2 * (n_qkv + 7) and pre_cast == 2 * (n_qkv + 1 + 1 + 2)
    assert kv[0]["local_end_index"] == 3 * 96 and float(kv[0]["v"].abs().sum()) > 0
    assert rel_l2(got, ref) < 0.15

    def unfused(x, *, q=None, scale=None, out=None, **kw):
        return emu.i8_quantize_rows(emu.ln_modulate(x, out=out, **kw), q, scale)
    monkeypatch.setattr(emu, "ln_modulate_i8", unfused)
    got2, _ = _run(m, g)
    assert torch.equal(got, got2)


def test_int8_linears_refuse_the_one_call_block(monkeypatch):
    """KR_BLOCK_FWD=1: the one-call block (kr_dit_block_fwd) issues bf16 GEMMs, so a block with INT8 linears must
    take the per-op schedule."""
    monkeypatch.setenv("KR_BLOCK_FWD", "1")
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    m = dit.CausalWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128).to(torch.bfloat16).eval()
    for blk in m.blocks:
        blk.self_attn.fuse_projections()
    assert m.use_block_fwd
    x = torch.zeros(96, 256, dtype=torch.bfloat16)
    cache = {"is_init": True}
    assert m._block_fwd_eligible(m.blocks[0], x, cache)
    fp8.quantize_(m, fp8.Int8DynamicActivationInt8WeightConfig())
    assert not m._block_fwd_eligible(m.blocks[0], x, cache)
    fp8.dequantize_(m)
    assert m._block_fwd_eligible(m.blocks[0], x, cache)


def _sp_worker(rank, world, port, ret):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        import realtime_video_b200.dit as dit
        from realtime_video_b200 import fp8
        from realtime_video_b200.parallel import SequenceParallel
        dit.ops = emu
        m, g = _small_model()
        fp8.quantize_(m, fp8.Int8DynamicActivationInt8WeightConfig())
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


def test_sequence_parallel_int8_equals_one_rank_gloo(monkeypatch):
    """No INT8 scale spans rows, so 2 gloo ranks give the one-rank result bit for bit with the stand-ins."""
    import torch.multiprocessing as mp

    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    from tests.test_parallel import _free_port
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model()
    fp8.quantize_(m, fp8.Int8DynamicActivationInt8WeightConfig())
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


def test_int8_header_symbols_are_exported_and_bound(lib):
    from realtime_video_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "krea_b200_int8.h").read_text(), flags=re.S)
    names = set(re.findall(r"\b(kr_[a-z0-9_]+)\s*\(", text))
    assert names == set(_lib.INT8_SIGNATURES) == {"kr_i8_quantize_rows", "kr_ln_modulate_i8", "kr_gemm_i8_rowwise"}
    assert all(hasattr(lib, n) for n in names)
    assert '#include "krea_b200_int8.h"' in (ROOT / "include" / "krea_b200.h").read_text()


def test_argument_validation_of_the_int8_entry_points(lib):
    """Rejected before any CUDA call, so no GPU is needed (pointers are never dereferenced)."""
    p = ctypes.c_void_p(4096)
    s = ctypes.c_void_p(8192)
    for rows, cols, ldx, ldq in ((4, 1532, 1532, 1536), (4, 14344, 14344, 14344), (4, 1536, 1528, 1536),
                                 (4, 1536, 1536, 1530), (0, 1536, 1536, 1536)):
        assert lib.kr_i8_quantize_rows(p, ldx, rows, cols, p, ldq, s, None) == -2
        assert b"i8_quantize_rows" in lib.kr_last_error()
    assert lib.kr_i8_quantize_rows(p, 1536, 4, 1536, p, 1536, None, None) == -1
    args = lambda D, ldq, scale, w=None, b=None: (p, D, None, 0, 4, D, ctypes.c_float(1e-6), w, b, None, 0, 0, 1, 0, 0,
                                                  p, ldq, scale, None)
    assert lib.kr_ln_modulate_i8(*args(1532, 1536, s)) == -2
    assert lib.kr_ln_modulate_i8(*args(8200, 8200, s)) == -2
    assert lib.kr_ln_modulate_i8(*args(1536, 1024, s)) == -2
    assert lib.kr_ln_modulate_i8(*args(1536, 1536, None)) == -1
    assert lib.kr_ln_modulate_i8(*args(1536, 1536, s, w=p)) == -1

    def gemm(epi, scale_a, scale_w, N=256, K=512, residual=None):
        return lib.kr_gemm_i8_rowwise(epi, p, K, p, K, scale_a, scale_w, None, p, N, 128, N, K, residual, 0,
                                      None, 0, 0, None, 0, 0, 0, None)
    assert gemm(0, None, s) == -1 and gemm(0, s, None) == -1
    assert gemm(3, s, s) == -1 and b"residual" in lib.kr_last_error()
    assert gemm(2, s, s) == -1
    assert gemm(0, s, s, N=384) == -1                                  # the 256-wide tile
    assert gemm(0, s, s, K=520) == -1                                  # K % 16
    assert gemm(0, s, s, K=132112) == -1 and b"132104" in lib.kr_last_error()   # the s32 bound
    assert gemm(0, s, ctypes.c_void_p(8196)) == -1 and b"aligned" in lib.kr_last_error()
    assert gemm(5, s, s) == -1                                         # EPI_MUL


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_and_resources_of_the_int8_kernels():
    from tests.test_sass_cpu import _ops, resource_usage, sass_functions
    funcs, usage = sass_functions(), resource_usage()
    gemms = [f for f in funcs if "gemm_i8_kernel" in f]
    assert len(gemms) == 5                                             # bias, GELU, gate + residual, residual, fp32
    for f in gemms:
        ops = {o.split(".")[0] for o in _ops(funcs[f])}
        assert {"IGMMA", "UTMALDG", "SYNCS"} <= ops and not ops & {"QGMMA", "HGMMA", "LDL", "STL"}, f
        assert usage[f][1:] == (0, 0), (f, usage[f])                   # no stack, no local memory
    quant = [f for f in funcs if "i8_quantize_rows_kernel" in f or "ln_modulate_i8_kernel" in f]
    assert len(quant) == 15
    for f in quant:
        ops = {o.split(".")[0] for o in _ops(funcs[f])}
        assert not ops & {"LDL", "STL"} and usage[f][1:] == (0, 0), (f, usage[f])
