"""Causal 3D VAE decoder on the sm_90a kernels — host-side mirror of the reference's decoder.

Mirrors ``demo_utils/vae_block3.py`` (VAEDecoderWrapper :177-230, VAEDecoder3d :334-443) and the
layers of ``wan/modules/vae.py`` it is built from (CausalConv3d :17, RMS_norm :39, Resample :66,
ResidualBlock :175, AttentionBlock :212): same module tree / state-dict keys (``decoder.*``,
``conv2.*``), so the reference's ``load_state_dict`` of the Wan2.1 VAE checkpoint works.
The modules only HOLD parameters; ``DecoderEngine`` runs the arithmetic as a fixed schedule of
implicit-GEMM convolutions with fused epilogues (``ops.vae_conv``) on channels-last activations.

Cache semantics (reference vae.py:191-206, vae_block3.py:46-91):
  * every 3x3x3 conv keeps the last two frames of its INPUT; here each conv owns a persistent
    input buffer [2 + T, H, W, C] whose two leading frames are that cache (read in place);
  * a zero cache is exactly the reference's zero padding for the first chunk;
  * up3d ``Resample``: the very first latent frame skips ``time_conv`` and leaves a ZERO cache
    (sentinel, vae_block3.py:51-53); one-frame chunks then update the cache as
    [where(old_last == 0, 0, x), x] (vae_block3.py:56-60) — reproduced verbatim.
Latent frames of one call are processed together per layer (one launch per conv), which is
arithmetically identical to the reference's frame-by-frame loop because every conv is causal.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn

from . import ops

MEAN = [-0.7571, -0.7089, -0.9113, 0.1075, -0.1745, 0.9653, -0.1517, 1.5508,
        0.4134, -0.0715, 0.5517, -0.3632, -0.1922, -0.9497, 0.2503, -0.2921]
STD = [2.8184, 1.4541, 2.3275, 2.6558, 1.2196, 1.7708, 2.6052, 2.0743,
       3.2687, 2.1526, 2.8652, 1.5579, 1.6382, 1.1253, 2.8251, 1.9160]


# ---------------------------------------------------------------------------------------------
# parameter holders (same attribute names / state-dict keys as the reference modules)
# ---------------------------------------------------------------------------------------------
class CausalConv3d(nn.Conv3d):
    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._padding = (self.padding[2], self.padding[2], self.padding[1], self.padding[1],
                         2 * self.padding[0], 0)
        self.padding = (0, 0, 0)


class RMS_norm(nn.Module):
    def __init__(self, dim, channel_first=True, images=True, bias=False):
        super().__init__()
        bdims = (1, 1, 1) if not images else (1, 1)
        self.channel_first, self.scale = channel_first, dim ** 0.5
        self.gamma = nn.Parameter(torch.ones((dim, *bdims) if channel_first else (dim,)))
        self.bias = nn.Parameter(torch.zeros((dim, *bdims))) if bias else 0.


class Upsample(nn.Upsample):
    pass


class Resample(nn.Module):
    def __init__(self, dim, mode):
        assert mode in ("upsample2d", "upsample3d", "downsample2d", "downsample3d")
        super().__init__()
        self.dim, self.mode, self.cache_t = dim, mode, 2
        if mode.startswith("up"):
            self.resample = nn.Sequential(Upsample(scale_factor=(2., 2.), mode="nearest"),
                                          nn.Conv2d(dim, dim // 2, 3, padding=1))
            if mode == "upsample3d":
                self.time_conv = CausalConv3d(dim, dim * 2, (3, 1, 1), padding=(1, 0, 0))
        else:   # wan/modules/vae.py:84-92
            self.resample = nn.Sequential(nn.ZeroPad2d((0, 1, 0, 1)), nn.Conv2d(dim, dim, 3, stride=(2, 2)))
            if mode == "downsample3d":
                self.time_conv = CausalConv3d(dim, dim, (3, 1, 1), stride=(2, 1, 1), padding=(0, 0, 0))


class ResidualBlock(nn.Module):
    def __init__(self, in_dim, out_dim, dropout=0.0):
        super().__init__()
        self.in_dim, self.out_dim = in_dim, out_dim
        self.residual = nn.Sequential(
            RMS_norm(in_dim, images=False), nn.SiLU(), CausalConv3d(in_dim, out_dim, 3, padding=1),
            RMS_norm(out_dim, images=False), nn.SiLU(), nn.Dropout(dropout),
            CausalConv3d(out_dim, out_dim, 3, padding=1))
        self.shortcut = CausalConv3d(in_dim, out_dim, 1) if in_dim != out_dim else nn.Identity()


class AttentionBlock(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.dim = dim
        self.norm = RMS_norm(dim)
        self.to_qkv = nn.Conv2d(dim, dim * 3, 1)
        self.proj = nn.Conv2d(dim, dim, 1)
        nn.init.zeros_(self.proj.weight)


class VAEDecoder3d(nn.Module):
    """demo_utils/vae_block3.py:334-385 (module tree only)."""

    def __init__(self, dim=96, z_dim=16, dim_mult=[1, 2, 4, 4], num_res_blocks=2, attn_scales=[],
                 temperal_upsample=[True, True, False], dropout=0.0):
        super().__init__()
        if attn_scales:
            raise NotImplementedError("attn_scales is empty in every Wan 2.1 VAE")
        self.dim, self.z_dim, self.dim_mult, self.num_res_blocks = dim, z_dim, dim_mult, num_res_blocks
        self.temperal_upsample = temperal_upsample
        self.cache_t, self.decoder_conv_num = 2, 32
        dims = [dim * u for u in [dim_mult[-1]] + dim_mult[::-1]]
        self.conv1 = CausalConv3d(z_dim, dims[0], 3, padding=1)
        self.middle = nn.Sequential(ResidualBlock(dims[0], dims[0], dropout), AttentionBlock(dims[0]),
                                    ResidualBlock(dims[0], dims[0], dropout))
        ups = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            if i in (1, 2, 3):
                in_dim = in_dim // 2
            for _ in range(num_res_blocks + 1):
                ups.append(ResidualBlock(in_dim, out_dim, dropout))
                in_dim = out_dim
            if i != len(dim_mult) - 1:
                ups.append(Resample(out_dim, mode="upsample3d" if temperal_upsample[i] else "upsample2d"))
        self.upsamples = nn.Sequential(*ups)
        self.head = nn.Sequential(RMS_norm(out_dim, images=False), nn.SiLU(),
                                  CausalConv3d(out_dim, 3, 3, padding=1))


# ---------------------------------------------------------------------------------------------
# engine
# ---------------------------------------------------------------------------------------------
def _tile_for(H: int, W: int):
    """(tile_w, tile_h) with tile_w*tile_h == 128 minimising padded area."""
    best = None
    for tw in (4, 8, 16, 32, 64):
        th = 128 // tw
        area = math.ceil(W / tw) * tw * math.ceil(H / th) * th
        if best is None or area < best[0] or (area == best[0] and abs(tw - 16) < abs(best[1] - 16)):
            best = (area, tw, th)
    return best[1], best[2]


def _weights_tag(w: torch.Tensor):
    """Identity of a parameter's current contents for the prepared-weights cache: storage address + version counter
    (in-place updates such as ``load_state_dict`` bump it).  Inference tensors (a model built or cast under
    ``torch.inference_mode()``) track no version — they cannot be updated in place outside inference mode either —
    so the address alone identifies them."""
    try:
        ver = w._version
    except RuntimeError:
        ver = None
    return (w.data_ptr(), ver)


class _Conv:
    """Kernel-ready conv: weight [rows, taps*cin_pad], bias [n], taps, channel config, and (for
    temporal convs) the persistent input buffer whose two leading frames are the cache."""

    def __init__(self, weight, bias, cin_pad, n_pad, cout, taps):
        self.weight, self.bias = weight, bias
        self.cin, self.n, self.cout, self.taps = cin_pad, n_pad, cout, taps
        self.buf: Optional[torch.Tensor] = None     # [kt-1 + Tmax, H, W, cin]


def _prep_conv(w: torch.Tensor, b: torch.Tensor, dtype, device, cin_pad=None, n_pad=None) -> _Conv:
    if w.dim() == 4:                       # Conv2d [Cout, Cin, kh, kw] -> kt = 1
        w = w.unsqueeze(2)
    cout, cin, kt, kh, kw = w.shape
    cin_pad = cin_pad or cin
    n_pad = n_pad or cout
    wp = torch.zeros(n_pad, kt, kh, kw, cin_pad, dtype=dtype, device=device)
    wp[:cout, :, :, :, :cin] = w.to(device=device, dtype=dtype).permute(0, 2, 3, 4, 1)
    bp = torch.zeros(max(n_pad, 32), dtype=dtype, device=device)
    bp[:cout] = b.to(device=device, dtype=dtype)
    return _Conv(wp.reshape(n_pad, kt * kh * kw * cin_pad).contiguous(), bp, cin_pad, n_pad, cout, (kt, kh, kw))


def _vae_attention(b, x):
    """vae.py:229-251 — per frame single-head attention over H*W tokens, C channels."""
    T, H, W, C = x.shape
    L = H * W
    if L % 32 != 0:
        raise NotImplementedError(f"VAE attention: H*W={L} must be a multiple of 32")
    out = torch.empty_like(x)
    xn = ops.vae_rmsnorm_silu(x, b["g"], torch.empty_like(x), silu=False)
    for t in range(T):
        xt, xnt = x[t].view(L, C), xn[t].view(L, C)
        qkv = ops.gemm(xnt, b["wqkv"], b["bqkv"])
        q, k = qkv[:, :C], qkv[:, C:2 * C]
        s = ops.gemm(q, k, None, epilogue=ops.EPI_F32, alpha=1.0 / math.sqrt(C))      # [L, L] fp32
        p = ops.softmax_rows(s, torch.empty(L, L, dtype=x.dtype, device=x.device))
        vt = ops.gemm(b["wqkv"][2 * C:], xnt, None)                                       # V^T [C, L]
        o = ops.gemm(p, vt, b["bqkv"][2 * C:])       # softmax rows sum to 1: P(V + 1 b^T) = PV + b^T
        ops.gemm(o, b["wproj"], b["bproj"], epilogue=ops.EPI_BIAS_RES, residual=xt, out=out[t].view(L, C))
    return out


class _CacheList(list):
    """The feature-cache list handed to the caller: a plain ``list`` that can be weakly referenced."""
    __slots__ = ("__weakref__",)


class _StreamLedger:
    """VALUE semantics for the feature-cache lists at zero cost in the common case.

    The reference's cache entries are values: a caller may keep the list of one stream, run another stream through the
    same module and come back (the server shares its models between WebSocket sessions, release_server.py:760).  Here
    the entries handed out are VIEWS of the engine's own conv-input buffers (no copy, and passing them back is free).
    Copy-on-conflict keeps that honest: the engine remembers (weakly) the last list it handed out; the moment a
    DIFFERENT state arrives — a new stream (all None) or tensors that are not these buffers — the remembered list's
    entries are replaced, in place, by clones of the buffers before anything is overwritten.  So a list never goes stale,
    a single stream never pays a copy, and interleaved streams pay one snapshot + one restore per switch."""

    _outstanding = None          # weakref to the last _CacheList handed out

    def _views(self) -> List[Optional[torch.Tensor]]:        # engine: the buffers' cache frames, list positions fixed
        raise NotImplementedError

    def _hand_out(self) -> List[Optional[torch.Tensor]]:
        import weakref
        lst = _CacheList(self._views())
        self._outstanding = weakref.ref(lst)
        return lst

    def _detach_outstanding(self) -> None:
        """Another state is about to replace the buffers: give the list that still aliases them its own copy."""
        ref, self._outstanding = self._outstanding, None
        lst = ref() if ref is not None else None
        if lst is None:
            return
        for i, (t, mine) in enumerate(zip(lst, self._views())):
            if t is not None and mine is not None and t.data_ptr() == mine.data_ptr():
                lst[i] = t.clone()

    def _take_in(self, cache, what: str) -> bool:
        """Make the buffers hold the state ``cache`` describes.  Returns False for a fresh stream (all None)."""
        if cache is None or all(c is None for c in cache):
            self._detach_outstanding()
            return False
        mine = self._views()
        pairs = [(src, dst) for src, dst in zip(cache, mine) if dst is not None]
        if any(src is None for src, _ in pairs):
            raise ValueError(f"partial VAE feature cache: pass back the list this {what} returned")
        if any(src.data_ptr() != dst.data_ptr() for src, dst in pairs):
            self._detach_outstanding()       # foreign state (another stream's snapshot, a caller's clone): restore it
            for src, dst in pairs:
                if src.data_ptr() != dst.data_ptr():
                    dst.copy_(src.reshape(dst.shape))
        return True


class DecoderEngine(_StreamLedger):
    """Runs VAEDecoder3d (+ the wrapper's un-scale and conv2) on the sm_90a kernels."""

    MAX_CHUNK = 3          # latent frames per launch sequence

    def __init__(self, decoder: VAEDecoder3d, conv2: nn.Module, mean: torch.Tensor, std: torch.Tensor,
                 single_mode: bool = False):
        self.decoder, self.conv2, self.mean, self.std = decoder, conv2, mean, std
        # single_mode: semantics of demo_utils/vae.py (VAEDecoderWrapperSingle), see decode_single
        self.single_mode = single_mode
        self._key = None
        self.H = self.W = None

    # -- weight preparation ---------------------------------------------------------------
    def _prepare(self, dtype, device, H, W):
        key = (dtype, str(device), H, W, _weights_tag(self.decoder.conv1.weight))
        if self._key == key:
            return
        d = self.decoder
        pc = lambda m, **kw: _prep_conv(m.weight.data, m.bias.data, dtype, device, **kw)  # noqa: E731
        g = lambda n: n.gamma.data.reshape(-1).to(device=device, dtype=dtype).contiguous()  # noqa: E731
        self.dtype, self.device, self.H, self.W = dtype, device, H, W
        self.mean_d = self.mean.to(device=device, dtype=dtype)
        self.inv_std_d = (1.0 / self.std.to(device=device, dtype=dtype))
        self.w2 = self.conv2.weight.data.reshape(16, 16).to(device=device, dtype=dtype).contiguous()
        self.b2 = self.conv2.bias.data.to(device=device, dtype=dtype).contiguous()
        self.conv1 = pc(d.conv1, cin_pad=64)
        self.stages = []       # flat op list
        blocks = list(d.middle) + list(d.upsamples)
        self.blocks = []
        for m in blocks:
            if isinstance(m, ResidualBlock):
                r = m.residual
                self.blocks.append(dict(kind="res", g1=g(r[0]), c1=pc(r[2]), g2=g(r[3]), c2=pc(r[6]),
                                        sc=pc(m.shortcut) if isinstance(m.shortcut, nn.Conv3d) else None,
                                        cin=m.in_dim, cout=m.out_dim))
            elif isinstance(m, AttentionBlock):
                C = m.dim
                wqkv = m.to_qkv.weight.data.reshape(3 * C, C).to(device=device, dtype=dtype).contiguous()
                bqkv = m.to_qkv.bias.data.to(device=device, dtype=dtype).contiguous()
                self.blocks.append(dict(kind="attn", g=g(m.norm), wqkv=wqkv, bqkv=bqkv, C=C,
                                        wproj=m.proj.weight.data.reshape(C, C).to(device=device, dtype=dtype).contiguous(),
                                        bproj=m.proj.bias.data.to(device=device, dtype=dtype).contiguous()))
            elif isinstance(m, Resample):
                e = dict(kind="up", mode=m.mode, C=m.dim, conv=pc(m.resample[1]))
                if m.mode == "upsample3d":
                    e["tconv"] = pc(m.time_conv)
                    e["tcache"] = None
                self.blocks.append(e)
        self.g_head = g(d.head[0])
        self.head = pc(d.head[2], n_pad=16)
        self._key = key
        self._alloc(H, W)

    def _alloc(self, H, W):
        """Persistent conv-input buffers (cache frames in front) for a chunk of MAX_CHUNK latent
        frames; spatial size doubles at every Resample, frames double at every up3d."""
        dt, dev = self.dtype, self.device
        T = self.MAX_CHUNK

        def buf(conv: _Conv, t, h, w):
            conv.buf = torch.zeros(conv.taps[0] - 1 + t, h, w, conv.cin, dtype=dt, device=dev)

        buf(self.conv1, T, H, W)
        h, w, t = H, W, T
        for b in self.blocks:
            if b["kind"] == "res":
                buf(b["c1"], t, h, w)
                buf(b["c2"], t, h, w)
            elif b["kind"] == "up":
                if b["mode"] == "upsample3d":
                    b["tcache"] = torch.zeros(2, h, w, b["C"], dtype=dt, device=dev)
                    t *= 2
                h, w = 2 * h, 2 * w
        buf(self.head, t, h, w)
        self.initialised = False       # no frame decoded yet (first-frame sentinel state)

    def reset(self):
        """Forget the stream: zero caches, first-frame state."""
        self._detach_outstanding()
        self.conv1.buf.zero_()
        for b in self.blocks:
            if b["kind"] == "res":
                b["c1"].buf.zero_()
                b["c2"].buf.zero_()
            elif b["kind"] == "up" and b["mode"] == "upsample3d":
                b["tcache"].zero_()
        self.head.buf.zero_()
        self.initialised = False

    # -- cache export / import (opaque to the caller, tensors so that .to() works) -----------
    def export_cache(self) -> List[Optional[torch.Tensor]]:
        """The 55-slot list for the caller (views of the buffers; see _StreamLedger for the aliasing contract)."""
        return self._hand_out()

    def _views(self) -> List[Optional[torch.Tensor]]:
        out: List[Optional[torch.Tensor]] = [None] * 55
        out[0] = self.conv1.buf[:2]
        i = 1
        for b in self.blocks:
            if b["kind"] == "res":
                out[i], out[i + 1] = b["c1"].buf[:2], b["c2"].buf[:2]
                i += 2
            elif b["kind"] == "up" and b["mode"] == "upsample3d":
                out[i] = b["tcache"]
                i += 1
        out[i] = self.head.buf[:2]
        return out

    def import_cache(self, cache: List[Optional[torch.Tensor]]):
        if not self._take_in(cache, "decoder"):
            self.reset()
            return
        self.initialised = True

    # -- one conv with fused epilogue --------------------------------------------------------
    def _conv(self, c: _Conv, T, src: Optional[torch.Tensor] = None, **kw):
        x = c.buf if src is None else src
        H, W = x.shape[1], x.shape[2]
        ops.vae_conv(x, c.weight, c.bias, n=c.n, cout=c.cout, T=T, taps=c.taps, tile=_tile_for(H, W), **kw)
        if src is None and c.taps[0] == 3:
            # roll: the last two input frames become the cache (frames = rows of a [frames, H*W*C] view; the
            # in-place row shift is overlap-safe, so T = 1 needs no temporary)
            ops.kv_roll(c.buf.view(c.buf.shape[0], -1), 0, T, 2)

    def _new(self, t, h, w, c):
        return torch.empty(t, h, w, c, dtype=self.dtype, device=self.device)

    def _attention(self, b, x):
        return _vae_attention(b, x)

    # -- decode a chunk of latent frames -----------------------------------------------------
    def decode_chunk(self, z: torch.Tensor, first: bool) -> torch.Tensor:
        """z [T0, 16, h, w] (strided ok) -> pixels [T', 3, 8h, 8w] fp32 in [-1, 1];
        T' = 1 for the first-ever latent frame (first=True requires T0 == 1), else 4*T0."""
        T = z.shape[0]
        assert T <= self.MAX_CHUNK and (not first or T == 1)
        c1 = self.conv1
        ops.vae_scale_input(z, self.mean_d, self.inv_std_d, self.w2, self.b2, c1.buf[2:2 + T])
        blocks = self.blocks
        h, w = self.H, self.W

        def next_gamma(i):
            """gamma of the norm that consumes block i's output (next ResidualBlock / head)."""
            if i + 1 < len(blocks):
                nb = blocks[i + 1]
                return (nb["g1"], nb["c1"]) if nb["kind"] == "res" else (None, None)
            return self.g_head, self.head

        # conv1 -> raw x (residual stream) + normalised input of middle.0.conv1
        x = self._new(T, h, w, c1.cout)
        g, nxt = blocks[0]["g1"], blocks[0]["c1"]
        self._conv(c1, T, out_raw=x, out_norm=nxt.buf[2:2 + T], gamma=g)

        for i, b in enumerate(blocks):
            if b["kind"] == "res":
                ca, cb = b["c1"], b["c2"]
                res = x
                if b["sc"] is not None:
                    res = self._new(T, h, w, b["cout"])
                    self._conv(b["sc"], T, src=x, out_raw=res)
                self._conv(ca, T, out_norm=cb.buf[2:2 + T], gamma=b["g2"])
                g, nxt = next_gamma(i)
                need_raw = nxt is not self.head          # the head only needs the normalised tensor
                xo = self._new(T, h, w, b["cout"]) if need_raw else None
                self._conv(cb, T, residual=res, out_raw=xo,
                           out_norm=nxt.buf[2:2 + T] if g is not None else None, gamma=g)
                x = xo
            elif b["kind"] == "attn":
                x = self._attention(b, x)
                nb = blocks[i + 1]
                ops.vae_rmsnorm_silu(x, nb["g1"], nb["c1"].buf[2:2 + T])
            else:  # Resample
                C = b["C"]
                if b["mode"] == "upsample3d":
                    if first and self.single_mode:
                        # demo_utils/vae.py:112-123: [zeros, x] on the channel axis -> after the
                        # channel->time interleave a ZERO frame precedes every frame; cache untouched
                        y = torch.zeros(2 * T, h, w, C, dtype=self.dtype, device=self.device)
                        y[1::2] = x
                        x, T = y, 2 * T
                    elif first:
                        b["tcache"].zero_()                    # sentinel, time_conv skipped
                    else:
                        tc = b["tconv"]
                        y = self._new(2 * T, h, w, C)
                        frame = h * w * C
                        # chunk-wise cache update of vae_block3.py:55-62 per reference chunk
                        step = self._chunk_frames(i)
                        for s0 in range(0, T, step):
                            xin = torch.cat([b["tcache"], x[s0:s0 + step]], dim=0)
                            for half in range(2):
                                ops.vae_conv(xin, tc.weight[half * C:(half + 1) * C], tc.bias[half * C:],
                                             n=C, cout=C, T=step, taps=tc.taps, tile=_tile_for(h, w),
                                             out_raw=y[2 * s0 + half:], raw_frame_stride=2 * frame)
                            xs = x[s0:s0 + step]
                            if step >= 2:
                                b["tcache"].copy_(xs[-2:])
                            elif self.single_mode:         # demo_utils/vae.py:106-111: [0, x]
                                b["tcache"][0].zero_()
                                b["tcache"][1].copy_(xs[0])
                            else:
                                old_last = b["tcache"][1]
                                pad = torch.where(old_last == 0, torch.zeros_like(xs[0]), xs[0])
                                b["tcache"][0].copy_(pad)
                                b["tcache"][1].copy_(xs[0])
                        x, T = y, 2 * T
                up = ops.vae_upsample2x(x, self._new(T, 2 * h, 2 * w, C))
                h, w = 2 * h, 2 * w
                cv = b["conv"]
                x = self._new(T, h, w, cv.cout)
                g, nxt = next_gamma(i)
                self._conv(cv, T, src=up, out_raw=x, out_norm=nxt.buf[2:2 + T], gamma=g)
        # head conv -> clamped fp32 pixels [T, 3, H, W]
        pix = torch.empty(T, 3, h, w, dtype=torch.float32, device=self.device)
        self._conv(self.head, T, out_pix=pix)
        self.initialised = True
        return pix

    def _chunk_frames(self, block_index: int) -> int:
        """Frames per REFERENCE chunk (one latent frame) at the input of Resample `block_index`:
        1 before the first up3d, 2 before the second."""
        n = 1
        for b in self.blocks[:block_index]:
            if b["kind"] == "up" and b["mode"] == "upsample3d":
                n *= 2
        return n

    def decode(self, z: torch.Tensor, feat_cache: List[Optional[torch.Tensor]]):
        """z [1, T, 16, h, w] -> (pixels [1, T', 3, 8h, 8w] fp32, feat_cache list)."""
        assert z.shape[0] == 1, "batch size 1 (reference: release_server.py:404)"
        zt = z[0]
        dtype = zt.dtype if zt.dtype in (torch.float16, torch.bfloat16) else torch.float16
        self._prepare(dtype, zt.device, zt.shape[-2], zt.shape[-1])
        self.import_cache(feat_cache)
        zt = zt.to(dtype)
        outs = []
        i = 0
        if not self.initialised:
            outs.append(self.decode_chunk(zt[0:1], first=True))
            i = 1
        while i < zt.shape[0]:
            n = min(self.MAX_CHUNK, zt.shape[0] - i)
            outs.append(self.decode_chunk(zt[i:i + n], first=False))
            i += n
        pix = torch.cat(outs, dim=0) if len(outs) > 1 else outs[0]
        return pix[None], self.export_cache()


    def decode_single(self, z: torch.Tensor, is_first_frame, feat_cache: List[Optional[torch.Tensor]]):
        """demo_utils/vae.py:167-195: one latent frame, explicit first-frame flag, 32 positional
        caches -> (pixels [1, 4, 3, H, W] in z.dtype clamped to [-1, 1], list of 32 caches)."""
        assert z.shape[0] == 1 and z.shape[1] == 1
        zt = z[0]
        dtype = zt.dtype if zt.dtype in (torch.float16, torch.bfloat16) else torch.float16
        self._prepare(dtype, zt.device, zt.shape[-2], zt.shape[-1])
        mine = [c for c in self._views() if c is not None]
        if len(feat_cache) != len(mine):
            raise ValueError(f"expected {len(mine)} cache tensors, got {len(feat_cache)}")
        for src, dst in zip(feat_cache, mine):
            if src.data_ptr() != dst.data_ptr():
                # reference cache layout is [1, C, 2, H, W]; ours [2, H, W, C]
                if src.dim() == 5:
                    src = src[0].permute(1, 2, 3, 0)
                dst[..., :src.shape[-1]].copy_(src)
        first = bool(is_first_frame.item()) if torch.is_tensor(is_first_frame) else bool(is_first_frame)
        pix = self.decode_chunk(zt.to(dtype), first=first)
        return pix[None].to(z.dtype), [c for c in self._views() if c is not None]


# ---------------------------------------------------------------------------------------------
# torch.compile boundary: one opaque op per streaming decode (pattern: wan/modules/sage.py:12-19)
# ---------------------------------------------------------------------------------------------
_DECODERS: dict = {}


def _register_decoder(mod) -> int:
    import weakref
    h = len(_DECODERS) + 1
    _DECODERS[h] = weakref.ref(mod)
    return h


@torch.library.custom_op("krea_b200::vae_decode_stream", mutates_args=())
def _vae_decode_stream(z: torch.Tensor, first: bool, handle: int) -> List[torch.Tensor]:
    mod = _DECODERS[handle]()
    px, _ = mod._decode(z, [None] * 55 if first else mod.engine._views())
    mod._stream_calls = getattr(mod, "_stream_calls", 0) + 1
    return [px, torch.full((1,), mod._stream_calls, dtype=torch.int64, device=z.device)]


@_vae_decode_stream.register_fake
def _(z, first, handle):
    t = z.shape[1]
    frames = 4 * t - 3 if first else 4 * t
    return [z.new_empty((1, frames, 3, z.shape[-2] * 8, z.shape[-1] * 8), dtype=torch.float32),
            z.new_empty((1,), dtype=torch.int64)]


# ---------------------------------------------------------------------------------------------
# the reference-facing wrappers
# ---------------------------------------------------------------------------------------------
class VAEDecoderWrapper(nn.Module):
    """demo_utils/vae_block3.py:177-230: ``forward(z[1,T,16,h,w], *feat_cache) ->
    (pixels [1,T',3,H,W] fp32 in [-1,1], feat_cache)``.  The cache list entries are this
    implementation's channels-last buffers (opaque to the caller, which only passes them back)."""

    def __init__(self):
        super().__init__()
        self.decoder = VAEDecoder3d()
        self.register_buffer("mean", torch.tensor(MEAN, dtype=torch.float32))
        self.register_buffer("std", torch.tensor(STD, dtype=torch.float32))
        self.z_dim = 16
        self.conv2 = CausalConv3d(self.z_dim, self.z_dim, 1)
        self._engine: Optional[DecoderEngine] = None
        self._handle = _register_decoder(self)      # id of this module for the opaque torch.compile op

    def __setstate__(self, state):                  # deepcopy / unpickle (release_server.py:111-119): own handle, own engine
        super().__setstate__(state)
        self._engine = None
        self._handle = _register_decoder(self)

    @property
    def engine(self) -> DecoderEngine:
        if self._engine is None:
            self._engine = DecoderEngine(self.decoder, self.conv2, self.mean, self.std)
        return self._engine

    def _apply(self, fn, *a, **k):     # .to() / .half() invalidate prepared weights
        self._engine = None
        return super()._apply(fn, *a, **k)

    def _decode(self, z: torch.Tensor, feat_cache):
        eng = self.engine
        eng.mean, eng.std = self.mean, self.std
        return eng.decode(z, feat_cache)

    def forward(self, z: torch.Tensor, *feat_cache):
        if torch.compiler.is_compiling():
            # torch.compile(vae_decoder, fullgraph=True) (release_server.py:754): the whole streaming decode is ONE
            # opaque custom op; the feature cache stays inside the engine and the caller gets a 55-entry list whose
            # first entry is a stream token (all-None = new stream, exactly like the eager convention)
            first = all(c is None for c in feat_cache)
            px, token = torch.ops.krea_b200.vae_decode_stream(z, first, self._handle)
            return px, [token] + [None] * 54
        cache = list(feat_cache)
        if cache and cache[0] is not None and cache[0].dtype == torch.int64:      # token from a compiled call
            cache = self.engine._views()
        return self._decode(z, cache)


class VAEDecoderWrapperSingle(nn.Module):
    """demo_utils/vae.py:150-195: ``forward(z[1,1,16,h,w], is_first_frame, *32 caches) ->
    (pixels [1,4,3,H,W] (z.dtype), 32 caches)``.  NOT interchangeable with VAEDecoderWrapper: the
    first latent frame also yields 4 frames (a zero frame is interleaved in front of it) and
    one-frame time_conv chunks cache [0, x] (SURVEY.md appendix A)."""

    def __init__(self):
        super().__init__()
        self.decoder = VAEDecoder3d()
        self.mean = torch.tensor(MEAN, dtype=torch.float32)
        self.std = torch.tensor(STD, dtype=torch.float32)
        self.z_dim = 16
        self.conv2 = CausalConv3d(self.z_dim, self.z_dim, 1)
        self._engine: Optional[DecoderEngine] = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    @torch.compiler.disable
    def forward(self, z: torch.Tensor, is_first_frame: torch.Tensor, *feat_cache):
        if self._engine is None:
            self._engine = DecoderEngine(self.decoder, self.conv2, self.mean, self.std, single_mode=True)
        return self._engine.decode_single(z, is_first_frame, list(feat_cache))


# ---------------------------------------------------------------------------------------------
# encoder (first-chunk path): the first-frame re-encode of the server loop
# ---------------------------------------------------------------------------------------------
class Encoder3d(nn.Module):
    """wan/modules/vae.py:254-299 (module tree only; temperal_downsample=[False, True, True])."""

    def __init__(self, dim=96, z_dim=32, dim_mult=[1, 2, 4, 4], num_res_blocks=2,
                 temperal_downsample=[False, True, True], dropout=0.0):
        super().__init__()
        dims = [dim * u for u in [1] + dim_mult]
        self.conv1 = CausalConv3d(3, dims[0], 3, padding=1)
        downs = []
        for i, (in_dim, out_dim) in enumerate(zip(dims[:-1], dims[1:])):
            for _ in range(num_res_blocks):
                downs.append(ResidualBlock(in_dim, out_dim, dropout))
                in_dim = out_dim
            if i != len(dim_mult) - 1:
                downs.append(Resample(out_dim, mode="downsample3d" if temperal_downsample[i] else "downsample2d"))
        self.downsamples = nn.Sequential(*downs)
        self.middle = nn.Sequential(ResidualBlock(out_dim, out_dim, dropout), AttentionBlock(out_dim),
                                    ResidualBlock(out_dim, out_dim, dropout))
        self.head = nn.Sequential(RMS_norm(out_dim, images=False), nn.SiLU(),
                                  CausalConv3d(out_dim, z_dim, 3, padding=1))


class EncoderEngine(_StreamLedger):
    """Encoder3d + WanVAE_.conv1 + latent scaling on the sm_90a kernels, streaming like the reference
    (demo_utils/vae_block3.py:141-175 over wan/modules/vae.py:301-345): the first chunk is ONE pixel frame on
    an empty cache (every causal conv sees zero history, the downsample3d time_convs are skipped and only
    remember their input, vae.py:160-163), every later chunk is FOUR frames -> one latent frame (time_conv
    (3,1,1) stride (2,1,1) over [last cached frame, chunk], vae.py:164-171).  As in the decoder engine each
    causal conv owns a persistent input buffer whose two leading frames ARE its feature cache."""

    MAX_CHUNK = 4          # pixel frames per later chunk

    def __init__(self, encoder: Encoder3d, conv1: nn.Module, mean: torch.Tensor, std: torch.Tensor):
        self.encoder, self.conv1_mod, self.mean, self.std = encoder, conv1, mean, std
        self._key = None
        self.initialised = False

    def _prepare(self, dtype, device, H, W):
        e = self.encoder
        key = (dtype, str(device), H, W, _weights_tag(e.conv1.weight))
        if self._key == key:
            return
        pc = lambda m, **kw: _prep_conv(m.weight.data, m.bias.data, dtype, device, **kw)  # noqa: E731
        g = lambda n: n.gamma.data.reshape(-1).to(device=device, dtype=dtype).contiguous()  # noqa: E731
        self.dtype, self.device, self.H, self.W = dtype, device, H, W
        self.conv_in = pc(e.conv1, cin_pad=64)
        self.blocks = []
        for m in list(e.downsamples) + list(e.middle):
            if isinstance(m, ResidualBlock):
                r = m.residual
                self.blocks.append(dict(kind="res", g1=g(r[0]), c1=pc(r[2]), g2=g(r[3]), c2=pc(r[6]),
                                        sc=pc(m.shortcut) if isinstance(m.shortcut, nn.Conv3d) else None,
                                        cin=m.in_dim, cout=m.out_dim))
            elif isinstance(m, AttentionBlock):
                C = m.dim
                self.blocks.append(dict(
                    kind="attn", g=g(m.norm), C=C,
                    wqkv=m.to_qkv.weight.data.reshape(3 * C, C).to(device=device, dtype=dtype).contiguous(),
                    bqkv=m.to_qkv.bias.data.to(device=device, dtype=dtype).contiguous(),
                    wproj=m.proj.weight.data.reshape(C, C).to(device=device, dtype=dtype).contiguous(),
                    bproj=m.proj.bias.data.to(device=device, dtype=dtype).contiguous()))
            else:
                d = dict(kind="down", mode=m.mode, C=m.dim, conv=pc(m.resample[1]))
                if m.mode == "downsample3d":
                    d["tconv"] = pc(m.time_conv)
                self.blocks.append(d)
        self.g_head = g(e.head[0])
        self.head = pc(e.head[2])
        self.w_out = self.conv1_mod.weight.data.reshape(32, 32).to(device=device, dtype=dtype).contiguous()
        self.b_out = self.conv1_mod.bias.data.to(device=device, dtype=dtype).contiguous()
        self.mean_d = self.mean.to(device=device, dtype=dtype)
        self.inv_std_d = 1.0 / self.std.to(device=device, dtype=dtype)
        # conv-input buffers [2 history frames + up to t frames]; t halves at every downsample3d
        z = lambda t, h, w, c: torch.zeros(2 + t, h, w, c, dtype=dtype, device=device)  # noqa: E731
        t = self.MAX_CHUNK
        self.conv_in.buf = z(t, H, W, 64)
        h, w = H, W
        for b in self.blocks:
            if b["kind"] == "res":
                b["c1"].buf, b["c2"].buf = z(t, h, w, b["cin"]), z(t, h, w, b["cout"])
            elif b["kind"] == "down":
                h, w = h // 2, w // 2
                if b["mode"] == "downsample3d":
                    b["tcache"] = torch.zeros(1, h, w, b["C"], dtype=dtype, device=device)
                    t = max(1, t // 2)
        self.head.buf = z(t, h, w, self.head.cin)
        self._key = key
        self.initialised = False

    # -- stream state ------------------------------------------------------------------------------
    def _cache_tensors(self):
        out = [self.conv_in.buf[:2]]
        for b in self.blocks:
            if b["kind"] == "res":
                out += [b["c1"].buf[:2], b["c2"].buf[:2]]
            elif b["kind"] == "down" and b["mode"] == "downsample3d":
                out.append(b["tcache"])
        out.append(self.head.buf[:2])
        return out

    def reset(self):
        """Forget the stream: zero history frames (frames >= 2 of a buffer are rewritten before every use)."""
        self._detach_outstanding()
        for c in self._cache_tensors():
            c.zero_()
        self.initialised = False

    def _views(self) -> List[Optional[torch.Tensor]]:
        mine = self._cache_tensors()
        return mine + [None] * (55 - len(mine))

    def export_cache(self) -> List[Optional[torch.Tensor]]:
        """The reference's 55-slot list (24 used by the encoder); entries are views of this engine's own buffers
        (see _StreamLedger for the aliasing contract)."""
        return self._hand_out()

    def import_cache(self, cache):
        if not self._take_in(cache, "encoder"):
            self.reset()
            return
        self.initialised = True

    def _conv(self, c: _Conv, T, src=None, **kw):
        x = c.buf if src is None else src
        ops.vae_conv(x, c.weight, c.bias, n=c.n, cout=c.cout, T=T, taps=c.taps,
                     tile=_tile_for(x.shape[1], x.shape[2]), **kw)
        if src is None and c.taps[0] == 3:
            ops.kv_roll(c.buf.view(c.buf.shape[0], -1), 0, T, 2)     # roll the feature cache (see DecoderEngine._conv)

    # -- one chunk ---------------------------------------------------------------------------------
    def encode_chunk(self, frames: torch.Tensor, first: bool) -> torch.Tensor:
        """frames [T, 3, H, W] in [-1, 1] (T == 1 when ``first``, else 4) -> mu [16, T', H/8, W/8] with
        T' = 1: the scaled latent frame of this chunk."""
        dt, dev = self.dtype, self.device
        T = frames.shape[0]
        assert (T == 1) if first else (T == self.MAX_CHUNK), "chunks are 1 frame (first) or 4 frames"
        new = lambda t, h, w, c: torch.empty(t, h, w, c, dtype=dt, device=dev)  # noqa: E731
        cin = self.conv_in
        cin.buf[2:2 + T, :, :, :3] = frames.to(dt).permute(0, 2, 3, 1)
        blocks = self.blocks

        def next_norm(i):
            if i + 1 < len(blocks):
                nb = blocks[i + 1]
                return (nb["g1"], nb["c1"]) if nb["kind"] == "res" else (None, None)
            return self.g_head, self.head

        h, w = self.H, self.W
        x = new(T, h, w, cin.cout)
        self._conv(cin, T, out_raw=x, out_norm=blocks[0]["c1"].buf[2:2 + T], gamma=blocks[0]["g1"])
        for i, b in enumerate(blocks):
            if b["kind"] == "res":
                res = x
                if b["sc"] is not None:
                    res = new(T, h, w, b["cout"])
                    self._conv(b["sc"], T, src=x, out_raw=res)
                self._conv(b["c1"], T, out_norm=b["c2"].buf[2:2 + T], gamma=b["g2"])
                g, nxt = next_norm(i)
                need_raw = nxt is not self.head
                xo = new(T, h, w, b["cout"]) if need_raw else None
                self._conv(b["c2"], T, residual=res, out_raw=xo,
                           out_norm=nxt.buf[2:2 + T] if g is not None else None, gamma=g)
                x = xo
            elif b["kind"] == "attn":
                x = _vae_attention(b, x)
                nb = blocks[i + 1]
                ops.vae_rmsnorm_silu(x, nb["g1"], nb["c1"].buf[2:2 + T])
            else:   # Resample: stride-2 conv behind ZeroPad2d((0,1,0,1)) per frame (vae.py:84-92, :152-155)
                g, nxt = next_norm(i)
                C = b["C"]
                h, w = h // 2, w // 2
                if b["mode"] != "downsample3d" or first:
                    xo = new(T, h, w, C)
                    self._conv(b["conv"], T, src=x, out_raw=xo, out_norm=nxt.buf[2:2 + T], gamma=g, sub2=True)
                    if b["mode"] == "downsample3d":
                        b["tcache"].copy_(xo)                 # first chunk: remember, skip time_conv (:160-163)
                    x = xo
                else:
                    # [last cached frame, T frames] -> time_conv (3,1,1), stride 2 in time: T/2 frames (:164-171)
                    xin = new(T + 1, h, w, C)
                    xin[:1].copy_(b["tcache"])
                    self._conv(b["conv"], T, src=x, out_raw=xin[1:], sub2=True)
                    b["tcache"].copy_(xin[T:T + 1])
                    tc = b["tconv"]
                    T2 = T // 2
                    xo = new(T2, h, w, C)
                    for j in range(T2):
                        ops.vae_conv(xin[2 * j:2 * j + 3], tc.weight, tc.bias, n=tc.n, cout=tc.cout, T=1, taps=tc.taps,
                                     tile=_tile_for(h, w), out_raw=xo[j:j + 1], out_norm=nxt.buf[2 + j:3 + j], gamma=g)
                    x, T = xo, T2
        y = new(T, h, w, self.head.cout)
        self._conv(self.head, T, out_raw=y)
        out = ops.gemm(y.view(T * h * w, self.head.cout), self.w_out, self.b_out)       # WanVAE_.conv1 (1x1x1)
        mu = out[:, :16]
        mu = (mu - self.mean_d.view(1, 16)) * self.inv_std_d.view(1, 16)               # vae_block3.py:168-172
        self.initialised = True
        return mu.reshape(T, h, w, 16).permute(3, 0, 1, 2)

    def encode_first(self, frame: torch.Tensor) -> torch.Tensor:
        """frame [3, H, W] -> mu [16, H/8, W/8] on a fresh stream (the server's first-frame re-encode)."""
        self.reset()
        return self.encode_chunk(frame[None], first=True)[:, 0]

    def encode(self, z: torch.Tensor, feat_cache, stream: bool = False):
        """The wrapper loop of vae_block3.py:141-165: z [3, T, H, W] -> mu [16, T', H/8, W/8]."""
        self.import_cache(feat_cache)
        t = z.shape[1]
        outs = []
        offset = 1
        for i in range(1 + (t - 1) // 4):
            if i == 0 and not self.initialised:
                outs.append(self.encode_chunk(z[:, :1].transpose(0, 1), first=True))
            else:
                start = i - 1
                if stream:
                    offset, start = 0, i
                chunk = z[:, offset + 4 * start:offset + 4 * (start + 1)]
                if chunk.shape[1] != self.MAX_CHUNK:
                    raise ValueError(f"VAE encoder: chunk {i} has {chunk.shape[1]} frames (needs 4); pass 1 + 4k "
                                     f"frames on a fresh cache or 4k frames with stream=True on a warm one")
                o = self.encode_chunk(chunk.transpose(0, 1), first=False)
                if i == 0 and stream:
                    outs = [o]
                else:
                    outs.append(o)
        return torch.cat(outs, dim=1) if len(outs) > 1 else outs[0]


class VAEEncoderWrapper(nn.Module):
    """demo_utils/vae_block3.py:116-175: ``forward(z [1, 3, T, H, W], feat_cache, stream=False) ->
    (mu [1, 16, T', H/8, W/8], feat_cache)``.  Fresh cache (all None): T = 1 + 4k pixel frames -> 1 + k latent
    frames (the server's first-frame re-encode, start frame and v2v uploads, release_server.py:531-538, :574,
    :585); warm cache with ``stream=True``: T = 4k frames -> k latent frames (webcam blocks, :518-525).  The
    returned cache entries are this implementation's channels-last buffers (opaque; pass them back)."""

    def __init__(self, vae=None):
        super().__init__()
        self.encoder = Encoder3d()
        self.conv1 = CausalConv3d(32, 32, 1)
        if vae is not None:       # reference signature: take the weights of a loaded WanVAE
            self.encoder.load_state_dict(vae.model.encoder.state_dict())
            self.conv1.load_state_dict(vae.model.conv1.state_dict())
        self.register_buffer("mean", torch.tensor(MEAN, dtype=torch.float32))
        self.register_buffer("std", torch.tensor(STD, dtype=torch.float32))
        self.z_dim = 16
        self._engine: Optional[EncoderEngine] = None

    def _apply(self, fn, *a, **k):
        self._engine = None
        return super()._apply(fn, *a, **k)

    @torch.compiler.disable
    def forward(self, z: torch.Tensor, feat_cache, stream: bool = False):
        if z.shape[0] != 1:
            raise NotImplementedError("VAE encoder: batch size 1 (as every call site of the reference)")
        if self._engine is None:
            self._engine = EncoderEngine(self.encoder, self.conv1, self.mean, self.std)
        eng = self._engine
        dtype = z.dtype if z.dtype in (torch.float16, torch.bfloat16) else torch.float16
        eng._prepare(dtype, z.device, z.shape[-2], z.shape[-1])
        mu = eng.encode(z[0], list(feat_cache), stream=stream)
        return mu[None], eng.export_cache()


def __getattr__(name: str):
    """``demo_utils.vae`` re-exports ``ZERO_VAE_CACHE`` / ``ALL_INPUTS_NAMES`` (demo_utils/vae.py:6, used by
    demo_utils/vae_torch2trt.py:2-5).  When this module is served under that name (realtime_video_b200.dropin) the
    two constants come from the reference's own ``demo_utils/constant.py`` — ``VAEDecoderWrapperSingle`` accepts its
    ``[1, C, 2, H, W]`` cache tensors."""
    if name in ("ZERO_VAE_CACHE", "ALL_INPUTS_NAMES"):
        try:
            import demo_utils.constant as c      # the reference checkout
        except ImportError as e:
            raise AttributeError(f"{name} lives in the reference's demo_utils/constant.py, which is not importable "
                                 f"here ({e})") from None
        return getattr(c, name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
