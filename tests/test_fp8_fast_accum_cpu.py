"""Fast accumulation for the FP8 linears (torchao ``Float8MMConfig(use_fast_accum=True)``) without a GPU: the config
surface, the two torchao import paths served by the drop-in finder, the routing of the DiT block schedule on stand-in
kernels, argument validation of the two C entry points, and the SASS / resource usage of the new kernel."""
import ctypes
import re
import shutil
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from tests import cpu_ops_emulation_fp8 as emu
from tests.golden_io import load_npz, rel_l2, weights

ROOT = Path(__file__).resolve().parent.parent


def test_mm_config_fields_and_defaults():
    from realtime_video_b200 import fp8
    c = fp8.Float8MMConfig()
    assert (c.emulate, c.use_fast_accum, c.pad_inner_dim) == (False, False, False)
    assert fp8.Float8MMConfig(use_fast_accum=True).use_fast_accum is True
    assert fp8.Float8MMConfig(False, True, False).use_fast_accum is True          # torchao's positional order
    with pytest.raises(NotImplementedError):
        fp8.Float8MMConfig(emulate=True)
    with pytest.raises(NotImplementedError):
        fp8.Float8MMConfig(pad_inner_dim=True)
    cfg = fp8.Float8DynamicActivationFloat8WeightConfig(granularity=[fp8.PerRow(), fp8.PerRow()],
                                                        mm_config=fp8.Float8MMConfig(use_fast_accum=True))
    assert isinstance(cfg.granularity, fp8.PerRow) and cfg.mm_config.use_fast_accum
    assert fp8.Float8DynamicActivationFloat8WeightConfig().mm_config is None
    with pytest.raises(TypeError):
        fp8.Float8DynamicActivationFloat8WeightConfig(mm_config={"use_fast_accum": True})


def _wrapper():
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper
    w = WanDiffusionWrapper(model_name="synthetic", is_causal=True,
                            model_config=dict(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128))
    for blk in w.model.blocks:
        blk.self_attn.fuse_projections()
    return w


def _flags(w):
    from realtime_video_b200 import fp8
    lins = [m for m in w.modules() if isinstance(m, torch.nn.Linear)]
    return ({id(m) for m in lins if hasattr(m, "_kr_fp8")}, {id(m) for m in lins if fp8.is_fast_accum(m)})


@pytest.mark.parametrize("gran", ["PerTensor", "PerRow"])
def test_quantize_records_the_accumulation_mode_on_the_quantised_linears_only(gran, monkeypatch):
    from realtime_video_b200 import fp8
    monkeypatch.delenv("KR_FP8_FAST_ACCUM", raising=False)
    w = _wrapper()
    g = getattr(fp8, gran)
    cfg = lambda **kw: fp8.Float8DynamicActivationFloat8WeightConfig(granularity=g(), **kw)
    for slow in (cfg(), cfg(mm_config=fp8.Float8MMConfig()), cfg(mm_config=fp8.Float8MMConfig(use_fast_accum=False))):
        fp8.quantize_(w, slow)
        quantised, fast = _flags(w)
        assert len(quantised) >= 2 * 8 and not fast
    before = [(m._kr_fp8[0].clone(), m._kr_fp8[1]) for m in w.modules() if hasattr(m, "_kr_fp8")]
    fp8.quantize_(w, cfg(mm_config=fp8.Float8MMConfig(use_fast_accum=True)))
    quantised, fast = _flags(w)
    assert len(quantised) >= 2 * 8 and fast == quantised
    assert not fp8.is_fast_accum(w.model.head.head)
    after = [m._kr_fp8 for m in w.modules() if hasattr(m, "_kr_fp8")]
    for (q0, s0), (q1, s1) in zip(before, after):                  # same bytes and scales in both modes
        assert torch.equal(q0, q1) and (torch.equal(s0, s1) if torch.is_tensor(s0) else s0 == s1)
    fp8.quantize_(w, cfg())                                        # quantising again without the flag clears it
    assert not _flags(w)[1]
    fp8.quantize_(w, cfg(mm_config=fp8.Float8MMConfig(use_fast_accum=True)))
    fp8.dequantize_(w)
    assert _flags(w) == (set(), set())
    assert not any(hasattr(m, "_kr_fp8_fast_accum") or hasattr(m, "_kr_fp8_granularity") for m in w.modules())


def test_environment_switch_only_decides_calls_without_an_mm_config(monkeypatch):
    from realtime_video_b200 import fp8
    w = _wrapper()
    monkeypatch.setenv("KR_FP8_FAST_ACCUM", "1")
    fp8.quantize_(w)                                               # the reference's and the benchmark's call
    quantised, fast = _flags(w)
    assert len(quantised) >= 2 * 8 and fast == quantised
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=fp8.PerRow()))
    assert _flags(w)[1] == _flags(w)[0]
    fp8.quantize_(w, fp8.Float8DynamicActivationFloat8WeightConfig(mm_config=fp8.Float8MMConfig(use_fast_accum=False)))
    assert not _flags(w)[1]                                        # an explicit mm_config wins
    for off in ("0", ""):
        monkeypatch.setenv("KR_FP8_FAST_ACCUM", off)
        fp8.quantize_(w)
        assert not _flags(w)[1]


def test_both_torchao_import_paths_resolve_through_the_dropin():
    code = ("import realtime_video_b200.dropin as d; d.install()\n"
            "from torchao.quantization.quant_api import (quantize_, Float8DynamicActivationFloat8WeightConfig,\n"
            "                                            Float8MMConfig as A, PerRow)\n"
            "from torchao.float8.inference import Float8MMConfig as B\n"
            "import realtime_video_b200.fp8 as f\n"
            "assert A is B is f.Float8MMConfig and quantize_ is f.quantize_\n"
            "c = Float8DynamicActivationFloat8WeightConfig(granularity=PerRow(), mm_config=B(use_fast_accum=True))\n"
            "assert c.mm_config.use_fast_accum and isinstance(c.granularity, f.PerRow)\n"
            "import importlib\n"
            "try:\n"
            "    importlib.import_module('torchao.float8.config')\n"
            "    raise SystemExit('a torchao module that is not served resolved')\n"
            "except ImportError:\n"
            "    pass\n"
            "print('OK')\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                       env={"PYTHONPATH": str(ROOT), "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stderr[-2000:]


def _small_model(fused=True):
    import realtime_video_b200.dit as dit
    g = load_npz("dit_small.npz")
    m = dit.CausalWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128)
    m.load_state_dict(weights(g, torch.float32), strict=False)
    m = m.float().eval()
    if fused:
        for blk in m.blocks:
            blk.self_attn.fuse_projections()
    return m, g


def _run(m, g):
    kv = [dict(k=torch.zeros(1, 6 * 96, 2, 128), v=torch.zeros(1, 6 * 96, 2, 128), global_end_index=0,
               local_end_index=0) for _ in range(2)]
    ca = [dict(k=torch.zeros(1, 512, 2, 128), v=torch.zeros(1, 512, 2, 128), is_init=False) for _ in range(2)]
    x = g["in/x0"].float()
    with torch.no_grad():
        return m(x[None], t=torch.full((1, 3), 750.0), context=g["in/ctx"].float()[None], seq_len=32760,
                 kv_cache=kv, crossattn_cache=ca, current_start=0)[0]


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("gran", ["PerTensor", "PerRow"])
def test_block_schedule_routes_every_quantised_linear_to_the_fast_entry_points(monkeypatch, gran, fused):
    """Host logic with stand-in kernels: with ``use_fast_accum=True`` every quantised Linear of the two blocks (to_qkv
    or q/k/v, o, cross q/k/v/o, ffn.0, ffn.2) runs the fast entry point of its granularity and no other Linear does;
    PerRow keeps the LayerNorm -> Fp8Rows hand-off (to_qkv or q/k/v, cross q, ffn.0 and the prompt's k/v arrive already
    cast).  Without the flag the same schedule runs the promoted entry points, and the stand-in results are equal."""
    import realtime_video_b200.dit as dit
    from realtime_video_b200 import fp8
    monkeypatch.setattr(dit, "ops", emu)
    monkeypatch.setattr(emu, "entry_points", [])
    monkeypatch.delenv("KR_FP8_FAST_ACCUM", raising=False)
    m, g = _small_model(fused)
    ref = _run(m, g)
    assert emu.entry_points == []                                   # bf16 model: no FP8 entry point at all
    n_lin = 2 * (8 if fused else 10)
    granularity = getattr(fp8, gran)()
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(granularity=granularity))
    slow = _run(m, g)
    promoted, emu.entry_points[:] = list(emu.entry_points), []
    fp8.quantize_(m, fp8.Float8DynamicActivationFloat8WeightConfig(
        granularity=granularity, mm_config=fp8.Float8MMConfig(use_fast_accum=True)))
    fast = _run(m, g)
    if gran == "PerTensor":
        assert promoted == ["kr_gemm_fp8"] * n_lin and emu.entry_points == ["kr_gemm_fp8_fast"] * n_lin
    else:
        assert [n for n, _ in promoted] == ["kr_gemm_fp8_rowwise"] * n_lin
        assert [n for n, _ in emu.entry_points] == ["kr_gemm_fp8_rowwise_fast"] * n_lin
        assert [c for _, c in emu.entry_points] == [c for _, c in promoted]
        assert sum(c for _, c in emu.entry_points) == 2 * ((1 if fused else 3) + 4)   # already-cast inputs
    assert torch.equal(fast, slow) and rel_l2(fast, ref) < 0.15


@pytest.fixture(scope="module")
def lib():
    from realtime_video_b200 import _lib
    _lib.build()
    return _lib.load()


def test_fast_entry_points_are_exported_and_validate_their_arguments(lib):
    """Rejected before any CUDA call, so no GPU is needed (pointers are never dereferenced)."""
    p, s = ctypes.c_void_p(4096), ctypes.c_void_p(8192)
    assert hasattr(lib, "kr_gemm_fp8_fast") and hasattr(lib, "kr_gemm_fp8_rowwise_fast")

    def tensor(epi=0, a=p, scale_a=s, N=256, K=512, lda=512, ldw=512, ldc=None, residual=None):
        return lib.kr_gemm_fp8_fast(epi, a, lda, p, ldw, scale_a, ctypes.c_float(1.0), None, p, N if ldc is None else ldc,
                                    128, N, K, residual, 0, None, 0, 0, None, 0, 0, 0, None)

    def rows(epi=0, a=p, scale_a=s, scale_w=s, N=256, K=512, lda=512, ldw=512, ldc=None, residual=None):
        return lib.kr_gemm_fp8_rowwise_fast(epi, a, lda, p, ldw, scale_a, scale_w, None, p, N if ldc is None else ldc,
                                            128, N, K, residual, 0, None, 0, 0, None, 0, 0, 0, None)
    for fn, name in ((tensor, b"gemm_fp8_fast"), (rows, b"gemm_fp8_rowwise_fast")):
        for bad in (dict(a=None), dict(scale_a=None), dict(N=128), dict(N=384), dict(K=520), dict(lda=504),
                    dict(ldw=500), dict(lda=256), dict(ldc=260), dict(epi=3), dict(epi=2), dict(epi=4), dict(epi=9)):
            assert fn(**bad) == -1, bad                             # KR_ERR_INVALID_ARG
            assert name in lib.kr_last_error(), (bad, lib.kr_last_error())
    assert tensor(N=128) == -1 and b"256" in lib.kr_last_error()
    assert rows(scale_w=None) == -1
    assert rows(scale_w=ctypes.c_void_p(8196)) == -1 and b"aligned" in lib.kr_last_error()


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")
def test_sass_and_resources_of_the_fast_accum_gemm_instantiations():
    """gemm_fp8_kernel<kFast = true> is e4m3 wgmma (QGMMA) fed by TMA through mbarriers, in four epilogues for each scale mode,
    for sm_90a only, without a legacy tensor-core path, stack or local memory, and within the 168 registers that 384
    threads per SM allow at launch (the consumers raise theirs to 232 with setmaxnreg)."""
    from tests.test_sass_cpu import _ops, cuobjdump, resource_usage, sass_functions
    assert set(re.findall(r"sm_\d+a?", cuobjdump("-lelf"))) == {"sm_90a"}
    funcs, usage = sass_functions(), resource_usage()
    for rowwise in (0, 1):
        kern = [f for f in funcs if re.search(rf"gemm_fp8_kernelILi\dELi{rowwise}ELb1E", f)]   # fast accumulation
        assert len(kern) == 4, kern                                 # bias, GELU, gate + residual, residual
        for f in kern:
            ops = _ops(funcs[f])
            assert {"QGMMA", "UTMALDG", "SYNCS"} <= {o.split(".")[0] for o in ops}, f
            assert any(o.startswith("QGMMA.64x256x32") for o in ops), f     # the 256-wide instruction
            assert not any(o.startswith(("HMMA", "IMMA", "HGMMA", "LDL", "STL")) for o in ops), f
            reg, stack, local = usage[f]
            assert reg <= 168 and stack == 0 and local == 0, (f, usage[f])
