"""The reference's ``utils/wan_wrapper.py`` on the sm_90a kernels (the L2 boundary, SURVEY.md §8b).

Same class names, constructor arguments, attributes and call conventions as
utils/wan_wrapper.py:20-323; the DiT underneath is ``realtime_video_b200.dit.CausalWanModel``, the text
encoder ``realtime_video_b200.t5.T5Encoder`` and the VAE ``realtime_video_b200.vae`` (hand-written sm_90a
kernels behind the C ABI).  ``realtime_video_b200.dropin.install()`` serves this module under the name
``utils.wan_wrapper``, so the reference's own ``pipeline/causal_inference.py`` and ``release_server.py``
construct and call these classes unchanged.

Checkpoints: like the reference, the constructors load ``MODEL_FOLDER/...`` files and RAISE when they are
missing; pass ``model_config=...`` (dims for a synthetic / caller-loaded model) to build without files.
"""
from __future__ import annotations

import json
import os
import types
from typing import List, Optional

import torch
from torch import nn

from realtime_video_b200 import ops
from realtime_video_b200.dit import CausalWanModel

try:   # dropped into the reference: its own pure-torch scheduler (utils/scheduler.py:5-194)
    from utils.scheduler import FlowMatchScheduler, SchedulerInterface  # type: ignore
except ImportError:   # stand-alone (bench / tests on a box without the reference checkout)
    from realtime_video_b200.flow_match import FlowMatchSchedule as FlowMatchScheduler
    SchedulerInterface = None

try:  # reference settings.py:1-5
    from settings import MODEL_FOLDER  # type: ignore
except Exception:  # noqa: BLE001
    MODEL_FOLDER = os.environ.get("MODEL_FOLDER", "wan_models")

# Wan 2.1 T2V dimensions (reference wan/configs/wan_t2v_14B.py:21-28, wan_t2v_1_3B.py:21-28)
KNOWN_CONFIGS = {
    "14B": dict(dim=5120, ffn_dim=13824, num_heads=40, num_layers=40),
    "1.3B": dict(dim=1536, ffn_dim=8960, num_heads=12, num_layers=30),
}


class _PromptTokenizer:
    """The reference's HuggingfaceTokenizer(name, seq_len=512, clean='whitespace') (wan/modules/tokenizers.py:38-83):
    ftfy.fix_text (when ftfy is installed) -> html.unescape twice -> collapse whitespace -> AutoTokenizer with
    padding='max_length', truncation, max_length=seq_len -> (input_ids, attention_mask)."""

    def __init__(self, name: str, seq_len: int = 512):
        from transformers import AutoTokenizer
        self.seq_len = seq_len
        self.tokenizer = AutoTokenizer.from_pretrained(name)

    @staticmethod
    def clean(text: str) -> str:
        import html
        import re
        try:
            import ftfy
            text = ftfy.fix_text(text)
        except ImportError:       # not in this image; only matters for mojibake in the prompt
            pass
        text = html.unescape(html.unescape(text)).strip()
        return re.sub(r"\s+", " ", text).strip()

    def __call__(self, sequence, return_mask: bool = True, **_):
        if isinstance(sequence, str):
            sequence = [sequence]
        enc = self.tokenizer([self.clean(u) for u in sequence], return_tensors="pt", padding="max_length",
                             truncation=True, max_length=self.seq_len, add_special_tokens=True)
        return (enc.input_ids, enc.attention_mask) if return_mask else enc.input_ids


class WanTextEncoder(nn.Module):
    """utils/wan_wrapper.py:20-56: UMT5-XXL encoder + tokenizer -> ``{"prompt_embeds": [B, 512, 4096]}`` with the
    rows past each prompt's length zeroed.  The encoder underneath is ``realtime_video_b200.t5.T5Encoder`` (same
    state-dict keys as the reference's ``umt5_xxl(encoder_only=True)``).  Extra keyword arguments (not in the
    reference) allow construction without the checkpoint / tokenizer files: ``model_config`` (dims),
    ``tokenizer`` (any callable ``(prompts, return_mask=True, add_special_tokens=True) -> (ids, mask)``),
    ``device``.  As in the reference the module is built in fp32 and the caller casts it
    (release_server.py:139-142 ``.to(dtype=torch.bfloat16)``)."""

    def __init__(self, model_config: Optional[dict] = None, tokenizer=None, device=None) -> None:
        super().__init__()
        from realtime_video_b200.t5 import umt5_xxl_encoder
        dev = device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu")
        ckpt = os.path.join(MODEL_FOLDER, "Wan2.1-T2V-1.3B", "models_t5_umt5-xxl-enc-bf16.safetensors")
        if model_config is None and not os.path.isfile(ckpt):
            # reference :30-33 loads unconditionally and fails without the file
            raise FileNotFoundError(f"{ckpt} not found; pass model_config=... to build without a checkpoint")
        self.text_encoder = umt5_xxl_encoder(device=dev, dtype=torch.float32, **(model_config or {}))
        if model_config is None:
            from safetensors.torch import load_file
            self.text_encoder.load_state_dict(load_file(ckpt, device=str(dev)))
        self.tokenizer = tokenizer
        self._tokenizer_path = os.path.join(MODEL_FOLDER, "Wan2.1-T2V-1.3B", "google", "umt5-xxl/")

    @property
    def device(self):
        return self.text_encoder.token_embedding.weight.device

    def forward(self, text_prompts: List[str]) -> dict:
        if self.tokenizer is None:
            if not os.path.isdir(self._tokenizer_path):
                raise FileNotFoundError(f"UMT5 tokenizer files not found under {self._tokenizer_path}; pass "
                                        f"tokenizer=... to WanTextEncoder")
            self.tokenizer = _PromptTokenizer(self._tokenizer_path, seq_len=512)
        ids, mask = self.tokenizer(text_prompts, return_mask=True, add_special_tokens=True)
        ids, mask = ids.to(self.device), mask.to(self.device)
        seq_lens = mask.gt(0).sum(dim=1).long()
        context = self.text_encoder(ids, mask)
        for u, v in zip(context, seq_lens):
            u[v:] = 0.0                              # set padding to 0.0 (wan_wrapper.py:52-53)
        return {"prompt_embeds": context}


class WanDiffusionWrapper(nn.Module):
    """utils/wan_wrapper.py:121-323.  Extra keyword arguments (not in the reference) let the
    model be built without a checkpoint on disk: ``model_config`` (dims), ``device``, ``dtype``."""

    def __init__(self, model_name="Wan2.1-T2V-1.3B", timestep_shift=8.0, is_causal=False,
                 local_attn_size=-1, sink_size=0, meta_init=False, model_config: Optional[dict] = None,
                 device=None, dtype=None):
        super().__init__()
        if not is_causal:
            raise NotImplementedError("the bidirectional WanModel is outside the hot path (SURVEY.md §2 row 2)")
        cfg = dict(model_config) if model_config else self._find_config(model_name)
        shards = [] if (model_config is not None or meta_init) else self._checkpoint_shards(model_name)
        cfg.update(local_attn_size=local_attn_size, sink_size=sink_size)
        ctx = torch.device("meta") if meta_init else (torch.device(device) if device is not None else None)
        prev = torch.get_default_dtype()
        try:
            if dtype is not None:
                torch.set_default_dtype(dtype)
            if ctx is not None:
                with ctx:
                    self.model = CausalWanModel(**cfg)
            else:
                self.model = CausalWanModel(**cfg)
        finally:
            torch.set_default_dtype(prev)
        if shards:
            self._load_pretrained(shards)
        self.model.eval()
        self.uniform_timestep = not is_causal
        self.scheduler = FlowMatchScheduler(shift=timestep_shift, sigma_min=0.0, extra_one_step=True)
        self.scheduler.set_timesteps(1000, training=True)
        self.seq_len = 32760
        self._sched_dev = None
        self.use_cuda_graphs = os.environ.get("KR_CUDA_GRAPH", "0") not in ("", "0")
        self._graphs = {}
        self.post_init()

    # -- construction helpers ---------------------------------------------------------------
    @staticmethod
    def _find_config(model_name: str) -> dict:
        path = os.path.join(MODEL_FOLDER, model_name, "config.json")
        keys = ("model_type", "patch_size", "text_len", "in_dim", "dim", "ffn_dim", "freq_dim",
                "text_dim", "out_dim", "num_heads", "num_layers", "qk_norm", "cross_attn_norm", "eps")
        if os.path.isfile(path):
            with open(path) as f:
                raw = json.load(f)
            cfg = {k: raw[k] for k in keys if k in raw}
            if "patch_size" in cfg:
                cfg["patch_size"] = tuple(cfg["patch_size"])
            return cfg
        for tag, dims in KNOWN_CONFIGS.items():
            if tag in model_name:
                return dict(dims)
        raise FileNotFoundError(f"no config.json under {os.path.join(MODEL_FOLDER, model_name)} and "
                                f"'{model_name}' names no known Wan 2.1 size")

    @staticmethod
    def _checkpoint_shards(model_name: str) -> list:
        """``CausalWanModel.from_pretrained(MODEL_FOLDER/model_name)`` (:135-141) reads the diffusers-format
        safetensors shards and fails without them; checked before the model is built."""
        folder = os.path.join(MODEL_FOLDER, model_name)
        files = sorted(os.path.join(folder, f) for f in os.listdir(folder)
                       if f.startswith("diffusion_pytorch_model") and f.endswith(".safetensors")) \
            if os.path.isdir(folder) else []
        if not files:
            raise FileNotFoundError(f"no diffusion_pytorch_model*.safetensors under {folder}; pass "
                                    f"model_config=... to build the model without a checkpoint")
        return files

    def _load_pretrained(self, shards: list) -> None:
        """strict load; the server overwrites these weights right afterwards with its self-forcing
        checkpoint (release_server.py:160-171)."""
        from safetensors.torch import load_file
        sd = {}
        for f in shards:
            sd.update(load_file(f))
        self.model.load_state_dict(sd, strict=True)

    # -- utils/wan_wrapper.py:181-228 ---------------------------------------------------------
    def _sigma_table(self, device):
        """float64 device copies of the scheduler's tables, rebuilt whenever the scheduler swaps its tensors
        (set_timesteps / ``.to``).  The source tensors are held and compared by identity, so a recycled
        address can never serve stale sigmas."""
        sig, ts = self.scheduler.sigmas, self.scheduler.timesteps
        c = self._sched_dev
        if c is None or c[0] is not sig or c[1] is not ts or c[2] != device:
            c = self._sched_dev = (sig, ts, device, sig.double().to(device), ts.double().to(device))
        return c[3], c[4]

    def _sigma_of(self, timestep: torch.Tensor, device) -> torch.Tensor:
        sigmas, timesteps = self._sigma_table(device)
        idx = torch.argmin((timesteps.unsqueeze(0) - timestep.to(device).unsqueeze(1)).abs(), dim=1)
        return sigmas[idx]

    def _convert_flow_pred_to_x0(self, flow_pred, xt, timestep):
        """x0 = xt - sigma_t * flow in float64 (:181-205); [B*, C, H, W] inputs."""
        sigma = self._sigma_of(timestep, flow_pred.device).reshape(-1, 1, 1, 1)
        return (xt.double() - sigma * flow_pred.double()).to(flow_pred.dtype)

    @staticmethod
    def _convert_x0_to_flow_pred(scheduler, x0_pred, xt, timestep):
        """(:207-228)"""
        dt = x0_pred.dtype
        sig, ts = scheduler.sigmas.double().to(x0_pred.device), scheduler.timesteps.double().to(x0_pred.device)
        idx = torch.argmin((ts.unsqueeze(0) - timestep.unsqueeze(1)).abs(), dim=1)
        return ((xt.double() - x0_pred.double()) / sig[idx].reshape(-1, 1, 1, 1)).to(dt)

    # -- utils/wan_wrapper.py:230-301 ---------------------------------------------------------
    # The server may wrap this module in torch.compile (release_server.py:753-755, DO_COMPILE=true).  The pass is a
    # fixed, hand-fused schedule of C-ABI launches: there is nothing for a tracing compiler to fuse, so the frame is
    # marked opaque — torch.compile(module) returns a module that runs this forward eagerly (tests/test_compile_cpu.py).
    @torch.compiler.disable
    def forward(self, noisy_image_or_video: torch.Tensor, conditional_dict: dict,
                timestep: torch.Tensor, kv_cache: Optional[List[dict]] = None,
                crossattn_cache: Optional[List[dict]] = None, current_start: Optional[int] = None,
                classify_mode: Optional[bool] = False, concat_time_embeddings: Optional[bool] = False,
                clean_x: Optional[torch.Tensor] = None, aug_t: Optional[torch.Tensor] = None,
                cache_start: Optional[int] = None):
        """noisy [B, F, 16, h, w], timestep [B, F] -> (flow_pred, pred_x0) of the same shape/dtype;
        mutates the cache dicts in place like the reference."""
        if kv_cache is None or clean_x is not None or classify_mode:
            raise NotImplementedError("only the KV-cached causal forward is on the hot path")
        prompt_embeds = conditional_dict["prompt_embeds"]
        B, Fr, C, H, W = noisy_image_or_video.shape
        model = self.model
        if self.use_cuda_graphs and B == 1 and noisy_image_or_video.is_cuda:
            out = self._graphed_forward(noisy_image_or_video, prompt_embeds, timestep, kv_cache, crossattn_cache,
                                        int(current_start or 0))
            if out is not None:
                return out
        entry = (int(kv_cache[0]["global_end_index"]), int(kv_cache[0]["local_end_index"])) if self._graphs else None
        flows, x0s = [], []
        for b in range(B):
            kv_b = kv_cache if B == 1 else [
                {"k": c["k"][b:b + 1], "v": c["v"][b:b + 1], "global_end_index": c["global_end_index"],
                 "local_end_index": c["local_end_index"]} for c in kv_cache]
            ca_b = crossattn_cache if B == 1 else None   # per-sample prompts: no shared cache
            head_out, _ = model.forward_tokens(noisy_image_or_video[b].permute(1, 0, 2, 3),
                                               timestep[b], prompt_embeds[b], kv_b, ca_b,
                                               int(current_start or 0))
            xt = noisy_image_or_video[b].to(head_out.dtype).contiguous()
            sigma = self._sigma_of(timestep[b].flatten(), head_out.device)
            flow, x0 = ops.unpatchify_x0(head_out, xt, sigma, model.out_dim, Fr, H, W)
            flows.append(flow)
            x0s.append(x0)
            if B > 1 and b == B - 1:
                for c, cb in zip(kv_cache, kv_b):
                    c["global_end_index"], c["local_end_index"] = cb["global_end_index"], cb["local_end_index"]
        if entry is not None and B == 1:
            self._note_exit_indices(noisy_image_or_video, timestep, kv_cache, crossattn_cache,
                                    int(current_start or 0), entry)
        return torch.stack(flows), torch.stack(x0s)

    # -- CUDA-graph replay of a whole DiT pass -------------------------------------------------------------------
    # A pass is ~2400 kernel launches issued from Python through ctypes (~10 us of host time each).  On one GPU the
    # device is the bottleneck and the host runs ahead; in the multi-GPU single-stream mode the kernels are N times
    # shorter and the host would limit the step.  In the server's steady state every block repeats the same two pass
    # shapes with the same cache indices (one recompute pass, four denoise passes into the same slot), so a pass is
    # captured once per (shape, start, mask, cache indices) signature — on its SECOND occurrence, the first runs
    # eagerly — and replayed afterwards: inputs are copied into static buffers, the Python-side cache indices are set
    # to the values the eager run produced.  Signatures that never repeat (the classic loop's growing indices) stay
    # eager.  Off by default (KR_CUDA_GRAPH=1 or ``wrapper.use_cuda_graphs = True``).
    _MAX_GRAPHS = 6

    def _graphed_forward(self, noisy, prompt_embeds, timestep, kv_cache, crossattn_cache, current_start):
        model = self.model
        if crossattn_cache is None or not all(c["is_init"] for c in crossattn_cache) or ops._prof is not None:
            return None                         # text K/V still to be computed / per-launch profiling: eager
        mask = model.block_mask
        mkey = None if mask is None else (mask.num_frames, mask.frame_seqlen, mask.num_frame_per_block,
                                          mask.local_attn_size)
        entry = (int(kv_cache[0]["global_end_index"]), int(kv_cache[0]["local_end_index"]))
        key = (tuple(noisy.shape), noisy.dtype, tuple(timestep.shape), timestep.dtype, current_start, mkey, entry,
               kv_cache[0]["k"].data_ptr(), crossattn_cache[0]["k"].data_ptr(), id(self.scheduler.sigmas),
               None if model.sp is None else model.sp.world)
        st = self._graphs.get(key)
        if st is None:                          # first occurrence: eager, remember what it did to the indices
            if len(self._graphs) >= self._MAX_GRAPHS:
                return None
            self._graphs[key] = {"pending": True}     # this eager run records its exit indices
            return None
        if "graph" not in st:
            if "exit" not in st:                # second occurrence: learn the exit indices from one more eager run
                st["pending"] = True
                return None
            x_s, t_s = noisy.clone(), timestep.clone()
            for c in kv_cache:
                c["global_end_index"], c["local_end_index"] = entry
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                head_out, _ = model.forward_tokens(x_s[0].permute(1, 0, 2, 3), t_s[0], prompt_embeds[0], kv_cache,
                                                   crossattn_cache, current_start)
                xt = x_s[0].to(head_out.dtype).contiguous()
                sigma = self._sigma_of(t_s[0].flatten(), head_out.device)
                flow, x0 = ops.unpatchify_x0(head_out, xt, sigma, model.out_dim, noisy.shape[1], noisy.shape[3],
                                             noisy.shape[4])
            st.update(graph=g, x=x_s, t=t_s, flow=flow, x0=x0)
        st["x"].copy_(noisy)
        st["t"].copy_(timestep)
        st["graph"].replay()
        for c in kv_cache:
            c["global_end_index"], c["local_end_index"] = st["exit"]
        return st["flow"][None].clone(), st["x0"][None].clone()

    def _note_exit_indices(self, noisy, timestep, kv_cache, crossattn_cache, current_start, entry):
        """After an eager pass: record the cache indices it left for the signature it started from."""
        mask = self.model.block_mask
        mkey = None if mask is None else (mask.num_frames, mask.frame_seqlen, mask.num_frame_per_block,
                                          mask.local_attn_size)
        for key, st in self._graphs.items():
            if st.get("pending") and key[0] == tuple(noisy.shape) and key[4] == current_start and key[5] == mkey \
                    and key[6] == entry:
                st["exit"] = (int(kv_cache[0]["global_end_index"]), int(kv_cache[0]["local_end_index"]))
                st["pending"] = False

    def get_scheduler(self):
        """(:303-315) binds the reference SchedulerInterface's conversion helpers onto the scheduler instance
        (training-side helpers; absent when the package runs without the reference checkout)."""
        s = self.scheduler
        if SchedulerInterface is not None:
            for name in ("convert_x0_to_noise", "convert_noise_to_x0", "convert_velocity_to_x0"):
                setattr(s, name, types.MethodType(getattr(SchedulerInterface, name), s))
        return s

    def post_init(self):
        self.get_scheduler()

    def enable_gradient_checkpointing(self) -> None:
        raise NotImplementedError("inference-only implementation")


class WanVAEWrapper(nn.Module):
    """utils/wan_wrapper.py:58-118 — classic-path VAE.  ``self.model`` carries the reference's WanVAE_
    state-dict keys (``encoder.*``, ``conv1.*``, ``conv2.*``, ``decoder.*``); decode and encode run on the
    sm_90a engines in the tensor's 16-bit dtype (bf16 on the classic path, wan_wrapper.py:102-104)."""

    def __init__(self, load_pretrained: bool = True):
        """``load_pretrained=False`` (not in the reference) builds the module tree without
        ``MODEL_FOLDER/Wan2.1-T2V-1.3B/Wan2.1_VAE.pth`` for synthetic / caller-loaded weights."""
        super().__init__()
        from realtime_video_b200.vae import MEAN, STD, CausalConv3d, Encoder3d, VAEDecoderWrapper

        class _WanVAEModel(VAEDecoderWrapper):
            """decoder + conv2 (VAEDecoderWrapper) plus encoder + conv1: the module tree of WanVAE_ (vae.py:491-516)."""

            def __init__(self):
                super().__init__()
                self.encoder = Encoder3d()
                self.conv1 = CausalConv3d(32, 32, 1)

        self.mean = torch.tensor(MEAN, dtype=torch.float32)
        self.std = torch.tensor(STD, dtype=torch.float32)
        self.model = _WanVAEModel()
        if load_pretrained:               # reference :73-77 (_video_vae(pretrained_path=...)): fails without the file
            vae_path = os.path.join(MODEL_FOLDER, "Wan2.1-T2V-1.3B", "Wan2.1_VAE.pth")
            if not os.path.isfile(vae_path):
                raise FileNotFoundError(f"{vae_path} not found; WanVAEWrapper(load_pretrained=False) builds the "
                                        f"module without a checkpoint")
            self.model.load_state_dict(torch.load(vae_path, map_location="cpu"), assign=True)
        self.model.eval().requires_grad_(False)
        self._cache = [None] * 55
        self._enc_engine = None

    def _apply(self, fn, *a, **k):     # .to() / .half() invalidate prepared weights
        self._enc_engine = None
        return super()._apply(fn, *a, **k)

    def decode_to_pixel(self, latent: torch.Tensor, use_cache: bool = False) -> torch.Tensor:
        """latent [B, F, 16, h, w] -> pixels [B, F', 3, H, W] fp32 in [-1, 1]
        (use_cache=False: fresh stream per call = WanVAE_.decode, vae.py:519-543;
         use_cache=True: WanVAE_.cached_decode, vae.py:545-567, batch 1)."""
        if use_cache:
            assert latent.shape[0] == 1, "Batch size must be 1 when using cache"
        outs = []
        for b in range(latent.shape[0]):
            cache = self._cache if use_cache else [None] * 55
            px, cache = self.model(latent[b:b + 1], *cache)
            if use_cache:
                self._cache = cache
            outs.append(px[0])
        return torch.stack(outs)

    def encode_to_latent(self, pixel: torch.Tensor) -> torch.Tensor:
        """pixel [B, 3, F, H, W] in [-1, 1], F = 1 + 4k -> latent [B, 1 + k, 16, H/8, W/8] fp32: per sample a fresh
        stream of WanVAE_.encode (vae.py:491-517: chunks of 1, 4, 4, ... frames), wan_wrapper.py:80-96."""
        from realtime_video_b200.vae import EncoderEngine
        if self._enc_engine is None:
            self._enc_engine = EncoderEngine(self.model.encoder, self.model.conv1, self.mean, self.std)
        eng = self._enc_engine
        dtype = pixel.dtype if pixel.dtype in (torch.float16, torch.bfloat16) else torch.float16
        eng._prepare(dtype, pixel.device, pixel.shape[-2], pixel.shape[-1])
        out = [eng.encode(u, [None] * 55, stream=False).float() for u in pixel]      # [16, T', h, w] each
        return torch.stack(out, dim=0).permute(0, 2, 1, 3, 4)
