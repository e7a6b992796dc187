"""Row-scaled FP8 (torchao ``granularity=PerRow()``) without a GPU: the oracle's per-row quantisation invariants,
``fp8.quantize_`` with PerRow, the torchao import line served by the drop-in finder, the DiT block schedule on stand-in
kernels (one GPU and sequence-parallel on gloo ranks), argument validation of the three C entry points, and the SASS /
resource usage of their kernels."""
import ctypes
import os
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from oracle import fp8_oracle as F8T
from oracle import fp8_rowwise_oracle as F8
from tests import cpu_ops_emulation_fp8 as emu
from tests.golden_io import load_npz, rel_l2, weights

ROOT = Path(__file__).resolve().parent.parent


def _mixed_rows(rows, cols, seed):
    """Rows whose magnitudes span 1e-4 .. 1 (log-uniform) and one outlier element of 64 in the largest row: the
    outlier sets a tensor-wide scale that pushes the small rows into e4m3's subnormals or to zero."""
    g = torch.Generator().manual_seed(seed)
    mag = torch.logspace(-4, 0, rows)[torch.randperm(rows, generator=g)]
    x = torch.randn(rows, cols, generator=g) * mag[:, None]
    x[mag.argmax(), 0] = 64.0
    return x


def _row_rel_l2(a, b):
    return float(((a - b).norm(dim=1) / b.norm(dim=1)).mean())


def test_oracle_per_row_invariants():
    x = _mixed_rows(64, 512, 0)
    x[5] = 0
    q, s = F8.quantize_per_row(x)
    assert q.dtype == torch.float8_e4m3fn and s.shape == (64,) and s.dtype == torch.float32
    amax = q.float().abs().amax(dim=1)
    nz = torch.arange(64) != 5
    assert bool((amax[nz] == 448.0).all())                       # every nonzero row's amax maps onto +-448
    assert int(q[5].float().abs().max()) == 0                    # a zero row quantises to zeros ...
    b = torch.randn(32)
    y = F8.linear_fp8_rowwise(x, torch.randn(32, 512) * 0.02, b.bfloat16())
    assert torch.equal(y[5], b.bfloat16())                       # ... and its output is the bias
    back = q.float() * s[:, None]
    qt, st = F8T.quantize_per_tensor(x)
    e_row, e_tensor = _row_rel_l2(back[nz], x[nz]), _row_rel_l2(qt.float()[nz] * st, x[nz])
    assert e_row < 4e-2 and e_row < 0.3 * e_tensor, (e_row, e_tensor)    # magnitudes 1e-4 .. 1: per row wins


def _wrapper():
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    w = WanDiffusionWrapper(model_name="synthetic", is_causal=True,
                            model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    for blk in w.model.blocks:
        blk.self_attn.fuse_projections()
    return w


@pytest.mark.parametrize("gran", ["single", "pair"])
def test_quantize_per_row_attaches_channel_scaled_weights_to_the_block_linears_only(gran):
    from realtime_video_b200 import fp8
    w = _wrapper()
    keys = set(w.state_dict().keys())
    g = fp8.PerRow() if gran == "single" else [fp8.PerRow(), fp8.PerRow()]
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=g))
    blk = w.model.blocks[0]
    for lin in (blk.self_attn.to_qkv, blk.self_attn.o, blk.cross_attn.q, blk.cross_attn.k, blk.cross_attn.v,
                blk.cross_attn.o, blk.ffn[0], blk.ffn[2]):
        wq, sw = lin._kr_fp8
        assert fp8.is_rowwise(lin)
        ref_q, ref_s = F8.quantize_per_row(lin.weight.detach())
        assert wq.dtype == torch.uint8 and torch.equal(wq, ref_q.view(torch.uint8))
        assert sw.dtype == torch.float32 and sw.shape == (lin.weight.shape[0],) and torch.equal(sw, ref_s)
    assert not hasattr(w.model.head.head, "_kr_fp8") and not hasattr(w.model.time_embedding[0], "_kr_fp8")
    assert set(w.state_dict().keys()) == keys
    fp8.dequantize_(w)
    assert not hasattr(blk.ffn[0], "_kr_fp8") and not hasattr(blk.ffn[0], "_kr_fp8_granularity")


def test_granularity_pairs_must_be_of_one_kind():
    from realtime_video_b200 import fp8
    assert isinstance(fp8.Float8DynamicActivationFloat8WeightConfig(granularity=(fp8.PerTensor(), fp8.PerTensor()))
                      .granularity, fp8.PerTensor)
    with pytest.raises(ValueError):
        fp8.Float8DynamicActivationFloat8WeightConfig(granularity=[fp8.PerRow(), fp8.PerTensor()])
    with pytest.raises(ValueError):
        fp8.Float8DynamicActivationFloat8WeightConfig(granularity=[fp8.PerRow()])
    with pytest.raises(NotImplementedError):
        fp8.Float8DynamicActivationFloat8WeightConfig(granularity=object())


def test_server_per_row_import_line_resolves_through_the_dropin():
    code = ("import realtime_video_b200.dropin as d; d.install()\n"
            "from torchao.quantization.quant_api import quantize_, Float8DynamicActivationFloat8WeightConfig, PerRow\n"
            "import realtime_video_b200.fp8 as f\n"
            "c = Float8DynamicActivationFloat8WeightConfig(granularity=PerRow())\n"
            "assert quantize_ is f.quantize_ and PerRow is f.PerRow and isinstance(c.granularity, f.PerRow)\n"
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
def test_block_schedule_with_per_row_fp8(monkeypatch, fused):
    """Host logic with stand-in kernels: per block, the three LayerNorms feeding FP8 linears cast to e4m3 themselves
    (no separate quantise launch for to_qkv or q/k/v, cross q, ffn.0), the self- and cross-attention o and ffn.2 use
    the row quantiser, the prompt is cast once for both K/V projections, and no per-tensor quantise runs.  The result
    equals the schedule with an unfused "LayerNorm, then quantise rows" stand-in bit for bit and stays within the toy
    tolerance of bf16."""
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model(fused)
    ref, _ = _run(m, g)
    calls = _counting(monkeypatch, ["linear_fp8", "fp8_quantize_rows", "ln_modulate_fp8", "gemm_fp8_rowwise"])
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    got, kv = _run(m, g)
    n_qkv = 1 if fused else 3
    assert calls == {"linear_fp8": 0, "ln_modulate_fp8": 2 * 3, "fp8_quantize_rows": 2 * 4,
                     "gemm_fp8_rowwise": 2 * (n_qkv + 7)}, calls
    assert kv[0]["local_end_index"] == 3 * 96 and float(kv[0]["v"].abs().sum()) > 0
    assert rel_l2(got, ref) < 0.15

    def unfused(x, *, q=None, scale=None, out=None, **kw):
        return emu.fp8_quantize_rows(emu.ln_modulate(x, out=out, **kw), q, scale)
    monkeypatch.setattr(emu, "ln_modulate_fp8", unfused)
    got2, _ = _run(m, g)
    assert torch.equal(got, got2)


def test_cross_q_without_norm3_uses_the_row_quantiser(monkeypatch):
    """cross_attn_norm=False: cross q reads the residual stream itself, so it is cast by the row quantiser."""
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model(cross_attn_norm=False)
    calls = _counting(monkeypatch, ["fp8_quantize_rows", "ln_modulate_fp8", "ln_modulate"])
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    got, _ = _run(m, g)
    assert torch.isfinite(got).all()
    # per block: o, cross q, cross o, ffn.2, the prompt (first pass); LayerNorms: norm1 + norm2 fused, the head's
    assert calls == {"fp8_quantize_rows": 2 * 5, "ln_modulate_fp8": 2 * 2, "ln_modulate": 1}, calls


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
        fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
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


def test_sequence_parallel_per_row_fp8_equals_one_rank_gloo(monkeypatch):
    """Per-row scales do not depend on the row shard: 2 gloo ranks (harness of tests/test_parallel.py) give the
    one-rank result bit for bit with the PerRow stand-ins."""
    import torch.multiprocessing as mp

    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    from tests.test_parallel import _free_port
    monkeypatch.setattr(dit, "ops", emu)
    m, g = _small_model()
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
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


def test_argument_validation_of_the_row_fp8_entry_points(lib):
    """Rejected before any CUDA call, so no GPU is needed (pointers are never dereferenced)."""
    p = ctypes.c_void_p(4096)
    s = ctypes.c_void_p(8192)
    # row quantiser: widths not a multiple of 8, wider than 14336, short pitches; null scales
    for rows, cols, ldx, ldq in ((4, 1532, 1532, 1536), (4, 14344, 14344, 14344), (4, 1536, 1528, 1536),
                                 (4, 1536, 1536, 1530), (0, 1536, 1536, 1536)):
        assert lib.kr_fp8_quantize_rows(p, ldx, rows, cols, p, ldq, s, None) == -2
        assert b"fp8_quantize_rows" in lib.kr_last_error()
    assert lib.kr_fp8_quantize_rows(p, 1536, 4, 1536, p, 1536, None, None) == -1
    # fused LayerNorm: bad width, D beyond the row kernels, short q pitch, null scales, half an affine pair
    args = lambda D, ldq, scale, w=None, b=None: (p, D, None, 0, 4, D, ctypes.c_float(1e-6), w, b, None, 0, 0, 1, 0, 0,
                                                  p, ldq, scale, None)
    assert lib.kr_ln_modulate_fp8(*args(1532, 1536, s)) == -2
    assert lib.kr_ln_modulate_fp8(*args(8200, 8200, s)) == -2
    assert lib.kr_ln_modulate_fp8(*args(1536, 1024, s)) == -2
    assert lib.kr_ln_modulate_fp8(*args(1536, 1536, None)) == -1
    assert lib.kr_ln_modulate_fp8(*args(1536, 1536, s, w=p)) == -1
    # row-scaled GEMM: null scales, residual epilogue without residual, N not a multiple of 128, misaligned scales

    def gemm(epi, scale_a, scale_w, N=256, residual=None):
        return lib.kr_gemm_fp8_rowwise(epi, p, 512, p, 512, scale_a, scale_w, None, p, N, 128, N, 512, residual, 0,
                                       None, 0, 0, None, 0, 0, 0, None)
    assert gemm(0, None, s) == -1 and gemm(0, s, None) == -1
    assert gemm(3, s, s) == -1 and b"residual" in lib.kr_last_error()
    assert gemm(2, s, s) == -1
    assert gemm(0, s, s, N=200) == -2
    assert gemm(0, s, ctypes.c_void_p(8196)) == -1 and b"aligned" in lib.kr_last_error()


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_and_resources_of_the_row_scaled_gemm_instantiations():
    from tests.test_sass_cpu import _ops, resource_usage, sass_functions
    funcs, usage = sass_functions(), resource_usage()
    rowwise = [f for f in funcs if re.search(r"gemm_fp8_kernelILi\dELi1ELb0E", f)]   # row scales, promoted
    assert len(rowwise) == 4                                          # bias, GELU, gate + residual, residual
    for f in rowwise:
        ops = set(_ops(funcs[f]))
        assert {"QGMMA", "UTMALDG", "SYNCS"} <= {o.split(".")[0] for o in ops}, f
        assert usage[f][1] == 0, (f, usage[f])                        # no stack
    rows = [f for f in funcs if "fp8_quantize_rows_kernel" in f or "ln_modulate_fp8_kernel" in f]
    assert len(rows) >= 10
    for f in rows:
        ops = {o.split(".")[0] for o in _ops(funcs[f])}
        assert not ops & {"LDL", "STL"} and usage[f][1:] == (0, 0), (f, usage[f])   # no local memory
