"""Drop-in boundary: make the reference's import names resolve to this package's classes (SURVEY.md §8b).

The reference has no FFI; its callers (``release_server.py``, ``sample.py``, ``pipeline/causal_inference.py``)
reach the hot path through four module names.  :func:`install` puts ONE finder in front of ``sys.meta_path``
that serves exactly those names and nothing else — every other ``utils.*`` / ``demo_utils.*`` / ``wan.*`` /
``pipeline.*`` module (``utils.misc``, ``utils.scheduler``, ``wan.modules.vae``, ``wan.modules.tokenizers``,
``demo_utils.memory``, ``demo_utils.constant``, the reference's own ``pipeline.causal_inference`` …) keeps
resolving to the reference checkout, independent of the ``sys.path`` order:

    utils.wan_wrapper          -> realtime_video_b200.wan_wrapper   (WanDiffusionWrapper, WanTextEncoder, WanVAEWrapper;
                                                                     reference utils/wan_wrapper.py:20-323)
    demo_utils.vae_block3      -> realtime_video_b200.vae           (VAEDecoderWrapper, VAEEncoderWrapper; vae_block3.py:116-230)
    demo_utils.vae             -> realtime_video_b200.vae           (VAEDecoderWrapperSingle, ZERO_VAE_CACHE, ...; demo_utils/vae.py:150-195)
    wan.modules.causal_model   -> realtime_video_b200.dit           (CausalWanModel; wan/modules/causal_model.py:526)
    torchao.quantization.quant_api -> realtime_video_b200.fp8       (quantize_, Float8DynamicActivationFloat8WeightConfig,
                                                                     PerTensor: the `enable_fp8` lines release_server.py:179-182;
                                                                     PerRow: the same lines with granularity=PerRow() also resolve;
                                                                     PerBlock: granularity=[PerBlock([1, 128]), PerBlock([128, 128])];
                                                                     Int8DynamicActivationInt8WeightConfig: the W8A8 INT8 config)
    torchao.float8.inference   -> realtime_video_b200.fp8           (Float8MMConfig, where torchao defines it: the same lines
                                                                     with mm_config=Float8MMConfig(use_fast_accum=True))

The served module IS the product module (same object under both names), so ``isinstance`` checks and class
identity hold across the two spellings.  The reference's ``CausalInferencePipeline`` and ``GenerationSession``
are NOT replaced: they run unmodified on top of these classes (tests/test_reference_callers_cpu.py).

Use (caller unchanged):

    python -m realtime_video_b200.dropin /path/to/realtime-video/sample.py <args>
    python -m realtime_video_b200.dropin -m uvicorn release_server:app
or, in an embedding program, ``import realtime_video_b200.dropin as d; d.install()`` before the reference imports.
"""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.machinery
import sys
import types

ALIASES = {
    "utils.wan_wrapper": "realtime_video_b200.wan_wrapper",
    "demo_utils.vae_block3": "realtime_video_b200.vae",
    "demo_utils.vae": "realtime_video_b200.vae",
    "wan.modules.causal_model": "realtime_video_b200.dit",
    # `enable_fp8: true` (release_server.py:179-182): quantize_ / Float8DynamicActivationFloat8WeightConfig / PerTensor
    # (or PerRow, or PerBlock), and Int8DynamicActivationInt8WeightConfig
    "torchao.quantization.quant_api": "realtime_video_b200.fp8",
    # Float8MMConfig, the mm_config argument of the config above, under the module torchao defines it in
    "torchao.float8.inference": "realtime_video_b200.fp8",
}


class _AliasLoader(importlib.abc.Loader):
    def __init__(self, target: str):
        self.target = target

    def create_module(self, spec):
        return importlib.import_module(self.target)       # the product module itself

    def exec_module(self, module):                         # already executed under its own name
        return None


class _NamespaceLoader(importlib.abc.Loader):
    """Empty parent package for an alias whose reference package is absent (stand-alone use on a box
    without the reference checkout)."""

    def create_module(self, spec):
        m = types.ModuleType(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        return None


class DropInFinder(importlib.abc.MetaPathFinder):
    """Serves the names in :data:`ALIASES`; for their parent packages it steps aside whenever any other finder can
    import them (the reference checkout) and synthesises an empty package otherwise."""

    def __init__(self):
        self._busy = False

    def find_spec(self, fullname, path=None, target=None):
        if fullname in ALIASES:
            return importlib.machinery.ModuleSpec(fullname, _AliasLoader(ALIASES[fullname]), origin=ALIASES[fullname])
        if self._busy or not any(a.startswith(fullname + ".") for a in ALIASES):
            return None
        self._busy = True
        try:
            for finder in sys.meta_path:
                if finder is self or not hasattr(finder, "find_spec"):
                    continue
                spec = finder.find_spec(fullname, path, target)
                if spec is not None:
                    return spec
        finally:
            self._busy = False
        return importlib.machinery.ModuleSpec(fullname, _NamespaceLoader(), is_package=True)


_finder = None


def install() -> DropInFinder:
    """Idempotent.  Modules already imported under an aliased name are replaced, so call it first."""
    global _finder
    if _finder is None:
        _finder = DropInFinder()
    if _finder not in sys.meta_path:
        sys.meta_path.insert(0, _finder)
    for name in ALIASES:
        sys.modules.pop(name, None)
    return _finder


def uninstall() -> None:
    if _finder is not None and _finder in sys.meta_path:
        sys.meta_path.remove(_finder)
    for name in ALIASES:
        sys.modules.pop(name, None)
