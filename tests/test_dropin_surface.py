"""The drop-in boundary (SURVEY.md §8b): ``realtime_video_b200.dropin.install()`` serves exactly the four module
names the reference's callers import the hot path through, leaves every other reference module importable, and
the served classes keep the reference's call signatures.  The reference-checkout-dependent half (unmodified
release_server.py / pipeline on the drop-ins) is tests/test_reference_callers_cpu.py."""
import inspect
import subprocess
import sys
import textwrap
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def run_py(code: str, *argv, cwd=None):
    return subprocess.run([sys.executable, "-c", textwrap.dedent(code), *argv], capture_output=True, text=True,
                          cwd=cwd, env={"PYTHONPATH": str(ROOT), "PATH": "/usr/bin:/bin"})


def test_aliased_names_resolve_to_the_b200_classes_without_a_reference_checkout():
    r = run_py("""
        import realtime_video_b200.dropin as d
        d.install()
        from utils.wan_wrapper import WanDiffusionWrapper, WanTextEncoder, WanVAEWrapper   # release_server.py:134,156
        from demo_utils.vae_block3 import VAEDecoderWrapper, VAEEncoderWrapper              # release_server.py:196-197
        from demo_utils.vae import VAEDecoderWrapperSingle
        from wan.modules.causal_model import CausalWanModel
        import realtime_video_b200.dit as dit, realtime_video_b200.vae as vae, realtime_video_b200.wan_wrapper as ww
        import utils.wan_wrapper, demo_utils.vae_block3
        assert utils.wan_wrapper is ww and demo_utils.vae_block3 is vae          # one module object, two names
        assert CausalWanModel is dit.CausalWanModel and VAEDecoderWrapper is vae.VAEDecoderWrapper
        assert WanDiffusionWrapper is ww.WanDiffusionWrapper
        import realtime_video_b200.t5 as t5
        te = WanTextEncoder(model_config=dict(vocab=8, dim=64, dim_attn=64, dim_ffn=64, num_heads=1, num_layers=1,
                                              num_buckets=32), device='cpu')
        assert isinstance(te.text_encoder, t5.T5Encoder)
        try:
            import utils.misc
        except ImportError:
            pass                        # no reference checkout here: nothing else under utils.* exists
        else:
            raise SystemExit("utils.misc must not exist without the reference")
        print("OK")
    """)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stderr[-3000:]


def test_other_reference_modules_stay_importable(tmp_path):
    """A stand-in checkout (namespace packages ``utils`` / ``demo_utils``, regular packages ``wan`` / ``pipeline``
    like the reference) AFTER or BEFORE the repo on sys.path: the finder overrides only its four names."""
    ref = tmp_path / "ref"
    for rel, body in {
        "utils/misc.py": "AtomicCounter = 'ref-misc'\n",
        "utils/wan_wrapper.py": "raise ImportError('the reference wrapper must be shadowed')\n",
        "utils/scheduler.py": "class FlowMatchScheduler: tag = 'ref-scheduler'\nclass SchedulerInterface: pass\n",
        "demo_utils/memory.py": "gpu = 'ref-memory'\n",
        "demo_utils/constant.py": "ZERO_VAE_CACHE = ['ref-cache']\nALL_INPUTS_NAMES = ['z']\n",
        "demo_utils/vae_block3.py": "raise ImportError('shadowed')\n",
        "wan/__init__.py": "from . import modules\n",
        "wan/modules/__init__.py": "from .vae import WanVAE\n",
        "wan/modules/vae.py": "WanVAE = 'ref-vae'\n",
        "wan/modules/tokenizers.py": "HuggingfaceTokenizer = 'ref-tok'\n",
        "wan/modules/causal_model.py": "raise ImportError('shadowed')\n",
        "pipeline/__init__.py": "from .causal_inference import CausalInferencePipeline\n",
        "pipeline/causal_inference.py": "from utils.wan_wrapper import WanDiffusionWrapper\n"
                                        "class CausalInferencePipeline: gen = WanDiffusionWrapper\n",
    }.items():
        f = ref / rel
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(body)
    code = """
        import sys
        ref = sys.argv[1]
        sys.path.insert(0 if sys.argv[2] == "first" else len(sys.path), ref)
        import realtime_video_b200.dropin as d
        d.install()
        from utils.misc import AtomicCounter                    # release_server.py:37
        from wan.modules.vae import WanVAE                      # release_server.py:54
        from wan.modules.tokenizers import HuggingfaceTokenizer  # utils/wan_wrapper.py:9
        from demo_utils.memory import gpu                       # pipeline/causal_inference.py:6
        from utils.scheduler import FlowMatchScheduler          # release_server.py:7
        assert (AtomicCounter, WanVAE, HuggingfaceTokenizer, gpu, FlowMatchScheduler.tag) == \\
            ('ref-misc', 'ref-vae', 'ref-tok', 'ref-memory', 'ref-scheduler')
        from pipeline import CausalInferencePipeline            # the reference's own class ...
        import realtime_video_b200.wan_wrapper as ww
        assert CausalInferencePipeline.gen is ww.WanDiffusionWrapper      # ... built on this package's wrapper
        assert ww.FlowMatchScheduler is FlowMatchScheduler      # the wrapper uses the reference's scheduler when it exists
        from demo_utils.vae import ZERO_VAE_CACHE, VAEDecoderWrapperSingle
        assert ZERO_VAE_CACHE == ['ref-cache']
        from wan.modules.causal_model import CausalWanModel
        import realtime_video_b200.dit as dit
        assert CausalWanModel is dit.CausalWanModel
        print("OK")
    """
    for order in ("first", "last"):
        r = run_py(code, str(ref), order)
        assert r.returncode == 0 and r.stdout.strip().endswith("OK"), (order, r.stderr[-3000:])


def test_launcher_runs_a_script_with_the_finder_installed(tmp_path):
    script = tmp_path / "entry.py"
    script.write_text("import sys\nfrom utils.wan_wrapper import WanDiffusionWrapper\n"
                      "print(WanDiffusionWrapper.__module__, sys.argv[1:])\n")
    r = subprocess.run([sys.executable, "-m", "realtime_video_b200.dropin", str(script), "--flag", "7"],
                       capture_output=True, text=True, env={"PYTHONPATH": str(ROOT), "PATH": "/usr/bin:/bin"})
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.strip() == "realtime_video_b200.wan_wrapper ['--flag', '7']"


def test_call_signatures_match_the_reference():
    from realtime_video_b200.vae import VAEDecoderWrapper, VAEDecoderWrapperSingle, VAEEncoderWrapper
    from realtime_video_b200.wan_wrapper import WanDiffusionWrapper, WanTextEncoder, WanVAEWrapper
    # utils/wan_wrapper.py:230-242
    fwd = list(inspect.signature(WanDiffusionWrapper.forward).parameters)
    assert fwd[:7] == ["self", "noisy_image_or_video", "conditional_dict", "timestep", "kv_cache",
                       "crossattn_cache", "current_start"]
    assert "cache_start" in fwd
    # utils/wan_wrapper.py:122-131
    init = inspect.signature(WanDiffusionWrapper.__init__).parameters
    for k in ("model_name", "timestep_shift", "is_causal", "local_attn_size", "sink_size", "meta_init"):
        assert k in init
    assert list(inspect.signature(WanTextEncoder.forward).parameters) == ["self", "text_prompts"]
    assert list(inspect.signature(WanVAEWrapper.decode_to_pixel).parameters) == ["self", "latent", "use_cache"]
    assert list(inspect.signature(WanVAEWrapper.encode_to_latent).parameters) == ["self", "pixel"]
    # demo_utils/vae_block3.py:195-199, :141-146 ; demo_utils/vae.py:167-172
    assert list(inspect.signature(VAEDecoderWrapper.forward).parameters) == ["self", "z", "feat_cache"]
    assert list(inspect.signature(VAEEncoderWrapper.forward).parameters) == ["self", "z", "feat_cache", "stream"]
    assert list(inspect.signature(VAEDecoderWrapperSingle.forward).parameters) == \
        ["self", "z", "is_first_frame", "feat_cache"]


def test_missing_checkpoints_raise_like_the_reference(tmp_path, monkeypatch):
    """The reference constructors read MODEL_FOLDER files and fail without them (utils/wan_wrapper.py:30-33,
    :73-77, :135-141); silently random weights would render garbage."""
    import pytest

    import realtime_video_b200.wan_wrapper as ww
    monkeypatch.setattr(ww, "MODEL_FOLDER", str(tmp_path))
    with pytest.raises(FileNotFoundError):
        ww.WanVAEWrapper()
    with pytest.raises(FileNotFoundError):
        ww.WanTextEncoder(device="cpu")
    with pytest.raises(FileNotFoundError):
        ww.WanDiffusionWrapper(model_name="Wan2.1-T2V-1.3B", is_causal=True)
    ww.WanVAEWrapper(load_pretrained=False)


def test_harness_context_frame_selection_matches_reference_rule():
    """release_server.py:563-576: first frame + last kv-1 frames while (block_idx-1)*3 < kv, afterwards
    the re-encoded oldest pixel frame replaces the first latent frame."""
    import torch
    from harness import GenerateParams, GenerationSession
    s = GenerationSession.__new__(GenerationSession)
    s.params = GenerateParams(kv_cache_num_frames=3, keep_first_frame=True)
    s.models = type("M", (), {"pipeline": type("P", (), {"num_frame_per_block": 3})(), "vae_encoder": None})()
    s.decode_enabled = True
    s.all_latents = torch.arange(12.0).view(1, 12, 1, 1, 1)
    for block_idx, start, expect in [(1, 3, [0, 1, 2]), (2, 6, [0, 4, 5]), (3, 9, [0, 7, 8])]:
        s.block_idx, s.current_start_frame = block_idx, start
        assert s.get_clean_context_frames().flatten().tolist() == expect
