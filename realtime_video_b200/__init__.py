"""realtime_video_b200 — H100-native (sm_90a) Self-Forcing causal-inference hot path of
krea-ai/realtime-video: causal Wan 2.1 DiT block stack with KV cache + causal 3D VAE decoder,
as hand-written CUDA behind a C ABI (include/krea_b200.h), driven through the reference's own
Python call surface (realtime_video_b200/dropin serves ``utils.wan_wrapper``, ``demo_utils.vae_block3``,
``demo_utils.vae`` and ``wan.modules.causal_model`` to the reference's unmodified callers)."""
__all__ = ["ops", "dit", "vae", "t5", "wan_wrapper", "factory", "dropin"]
