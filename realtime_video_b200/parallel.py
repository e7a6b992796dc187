"""Single-stream multi-GPU mode: Ulysses-style sequence parallelism for the DiT block stack (SURVEY.md §8e opt. 3).

The hot path is ONE strictly sequential stream (B=1; every pass needs the previous one), so it does not shard
into independent units.  Here all N GPUs of a box work on the same block:

  * token rows are sharded contiguously (L/N rows per rank) for everything token-wise: LayerNorm/modulation,
    QKV / o / cross-attention / FFN GEMMs (stream-K kernel: an L/N-row GEMM has too few tiles for 132 SMs),
    RMSNorm+RoPE — weights replicated (28 GB of 180 GB);
  * self-attention is sharded by HEAD (heads/N per rank, full sequence).

Two exchange back ends:

``p2p`` (GPUs, default): the exchange is done BY THE KERNELS over NVLink peer memory.  Every rank owns one
    symmetric allocation (torch.distributed._symmetric_memory: rendezvous hands out the peers' addresses; torch is
    plumbing) holding its head-sharded q buffer, its head-sharded KV caches and its row-sharded attention-output
    buffer.  ``kr_qkv_norm_rope_p2p`` (RMSNorm + RoPE of my rows) stores each head's columns straight into the
    owning rank's q buffer / K-cache slot / V-cache slot; after the attention ``kr_comm_scatter_rows`` stores my
    heads' output rows into the owners' row buffers.  Per layer: two device-side barriers (symmetric-memory signal
    pads) instead of four NCCL all-to-alls and their pack / unpack copies.
    Buffer reuse is safe with exactly these two barriers: a rank passes barrier A(l+1) only after its own o-proj(l)
    read its row buffer, and passes barrier B(l) only after every rank's attention(l) has read its q buffer.
``nccl`` (and gloo in the CPU tests): torch.distributed all_to_all_single with pack / unpack copies — the
    baseline the p2p path is measured against, and the host-logic reference for tests/test_parallel.py.

Every kernel computes each output row / head exactly as on one GPU; only the placement changes.  (The stream-K
GEMM sums split-K partials in a different order than the data-parallel kernel: results agree to fp32 rounding of
the accumulator, not bit for bit.)
"""
from __future__ import annotations

import ctypes
from typing import Optional

import torch
import torch.distributed as dist


class SequenceParallel:
    def __init__(self, group: Optional[dist.ProcessGroup] = None, exchange: Optional[str] = None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised before SequenceParallel()")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        if exchange is None:
            exchange = "p2p" if dist.get_backend(group) == "nccl" else "nccl"
        if exchange not in ("p2p", "nccl"):
            raise ValueError(exchange)
        self.exchange = exchange
        self._arena = None           # symmetric allocation (uint8)
        self._hdl = None
        self._peer_base = None
        self._used = 0
        self._ptr_cache = {}
        self._kv = self._kv_key = self._q_buf = self._o_rows_buf = self._o_heads_buf = None
        self.fallback_reason = None  # set when the p2p setup failed and the collective exchange took over

    # -- sharding arithmetic -------------------------------------------------------------------
    def rows(self, L: int):
        """(first global row, number of local rows) of this rank for a sequence of L tokens."""
        if L % self.world != 0:
            raise ValueError(f"sequence length {L} is not divisible by {self.world} ranks")
        n = L // self.world
        return self.rank * n, n

    def local_heads(self, heads: int) -> int:
        if heads % self.world != 0:
            raise ValueError(f"{heads} heads are not divisible by {self.world} ranks")
        return heads // self.world

    # -- p2p back end: symmetric arena ---------------------------------------------------------
    @property
    def p2p(self) -> bool:
        return self.exchange == "p2p"

    def reserve(self, nbytes: int, device) -> None:
        """Create the symmetric arena (once; collective).  Sized by the caller for: KV caches + q / o buffers."""
        if self._arena is not None:
            if self._arena.numel() < nbytes:
                raise RuntimeError("symmetric arena already created with a smaller size")
            return
        g = self.group if self.group is not None else dist.group.WORLD
        err = None
        try:
            import torch.distributed._symmetric_memory as symm_mem
            arena = symm_mem.empty(nbytes, dtype=torch.uint8, device=device)
            hdl = symm_mem.rendezvous(arena, g.group_name)
            peer_base = [int(p) for p in hdl.buffer_ptrs]
            if peer_base[self.rank] != arena.data_ptr():
                raise RuntimeError("symmetric-memory rendezvous returned a foreign base address for this rank")
        except Exception as ex:  # noqa: BLE001 - any failure (no P2P access, allocator limits, ...) takes the fallback
            err = ex
        # the decision must be the same on every rank: one rank on the p2p path and another on collectives would hang
        ok = torch.tensor([0 if err is not None else 1], dtype=torch.int32, device=device)
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.group)
        if int(ok.item()) == 0:
            self.exchange = "nccl"
            self.fallback_reason = f"{type(err).__name__}: {err}" if err is not None else "a peer rank failed"
            import warnings
            warnings.warn("SequenceParallel: symmetric-memory setup failed on at least one rank "
                          f"({self.fallback_reason}); using the torch.distributed all-to-all exchange instead")
            return
        self._arena, self._hdl, self._peer_base = arena, hdl, peer_base
        self._used = 0

    def carve(self, shape, dtype) -> torch.Tensor:
        """A tensor inside the arena; every rank must carve the same sequence of shapes (same offsets)."""
        n = 1
        for d in shape:
            n *= int(d)
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        off = (self._used + 255) // 256 * 256
        if off + nbytes > self._arena.numel():
            raise RuntimeError(f"symmetric arena exhausted: need {off + nbytes} of {self._arena.numel()} bytes")
        self._used = off + nbytes
        return self._arena[off:off + nbytes].view(dtype).view(*shape)

    def peer_ptrs(self, t: torch.Tensor, byte_offset_of=None):
        """ctypes array of world pointers: the address of ``t``'s first element in every rank's arena."""
        key = t.data_ptr()
        arr = self._ptr_cache.get(key)
        if arr is None:
            off = key - self._arena.data_ptr()
            if off < 0 or off >= self._arena.numel():
                raise RuntimeError("tensor is not inside the symmetric arena")
            arr = (ctypes.c_void_p * self.world)(*[b + off for b in self._peer_base])
            if len(self._ptr_cache) > 4096:
                self._ptr_cache.clear()
            self._ptr_cache[key] = arr
        return arr

    def barrier(self) -> None:
        """Device-side barrier on the current stream (symmetric-memory signal pads): all ranks' earlier kernels —
        including their remote stores into this rank's arena — are complete and visible afterwards."""
        self._hdl.barrier(channel=0)

    def alloc_kv_cache(self, num_layers: int, shape, dtype, device):
        """KV caches [1, rows, heads_local, head_dim] x 2 x layers plus the exchange buffers, all inside ONE symmetric
        allocation created here (collective, once per object).  Returns [(k, v)] per layer, zero-filled — or None
        when the symmetric-memory setup failed on any rank: the object has then switched (on every rank) to the
        collective exchange and the caller allocates ordinary caches."""
        key = (num_layers, tuple(int(d) for d in shape), dtype)
        if self._arena is None:
            rows, hl, hd = key[1][1], key[1][2], key[1][3]
            es = torch.empty((), dtype=dtype).element_size()
            dh, D = hl * hd, hl * hd * self.world

            def al(n):
                return (n + 255) // 256 * 256
            n_loc = rows // self.world + 8
            self.reserve(2 * num_layers * al(rows * dh * es) + al(rows * dh * es) + al(n_loc * D * es) + 4096, device)
            if self._arena is None:          # setup failed on some rank: every rank is on the collective exchange now
                return None
            self._kv = [(self.carve(key[1], dtype), self.carve(key[1], dtype)) for _ in range(num_layers)]
            self._q_buf = self.carve((rows, dh), dtype)                 # all rows, my heads (peers write)
            self._o_rows_buf = self.carve((n_loc, D), dtype)            # my rows, all heads (peers write)
            self._o_heads_buf = torch.empty(rows, dh, dtype=dtype, device=device)     # local attention output
            self._kv_key = key
        elif self._kv_key != key:
            raise RuntimeError(f"SequenceParallel holds a KV cache of geometry {self._kv_key}; asked for {key}")
        for k, v in self._kv:
            k.zero_()
            v.zero_()
        return self._kv

    def exchange_buffers(self, L: int):
        """q_full [L, D/N] (all rows, my heads), o_heads [L, D/N] (local), o_rows [L/N, D] (my rows, all heads)."""
        if self._arena is None or L > self._q_buf.shape[0]:
            raise RuntimeError("exchange buffers are sized with the KV cache: allocate it through alloc_kv_cache "
                               "(harness PipelineState does) before the first forward")
        return self._q_buf[:L], self._o_heads_buf[:L], self._o_rows_buf[:L // self.world]

    # -- nccl / gloo back end ------------------------------------------------------------------
    def rows_to_heads(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """x [L/N, H*128] (my rows, all heads) -> [L, H/N*128] (all rows in global order, my heads).
        ``out`` may be a row-contiguous view (e.g. a KV-cache slot) that receives the result."""
        n, width = x.shape
        W = self.world
        blk = width // W
        send = x.view(n, W, blk).transpose(0, 1).contiguous()          # [W, n, blk]: chunk d -> rank d
        if out is None:
            out = torch.empty(W * n, blk, dtype=x.dtype, device=x.device)
        if not out.is_contiguous():
            raise ValueError("rows_to_heads: output must be contiguous")
        dist.all_to_all_single(out.view(W, n, blk), send, group=self.group)   # chunk s <- rank s's rows
        return out

    def heads_to_rows(self, x: torch.Tensor) -> torch.Tensor:
        """x [L, H/N*128] (all rows, my heads) -> [L/N, H*128] (my rows, all heads)."""
        L, blk = x.shape
        W = self.world
        n = L // W
        recv = torch.empty(W, n, blk, dtype=x.dtype, device=x.device)
        dist.all_to_all_single(recv, x.contiguous().view(W, n, blk), group=self.group)
        return recv.transpose(0, 1).reshape(n, W * blk)                # heads of rank s at columns s*blk

    def gather_rows(self, x: torch.Tensor) -> torch.Tensor:
        """x [L/N, C] -> [L, C] on every rank."""
        out = torch.empty(self.world * x.shape[0], *x.shape[1:], dtype=x.dtype, device=x.device)
        dist.all_gather_into_tensor(out, x.contiguous(), group=self.group)
        return out


class LayerPipeline:
    """BASELINE configs[2] as written: the DiT blocks sharded BY LAYER over the GPUs of one box (40 layers -> 5 per GPU
    on 8 GPUs), the residual stream handed from GPU i to GPU i+1 with one point-to-point transfer per pass
    (``torch.distributed`` send / recv: NCCL over NVLink on GPUs, gloo in the CPU tests).  Every rank keeps the KV and
    prompt caches of its own layers only; the time / text embeddings are recomputed on every rank (two small GEMMs)
    instead of being shipped; the last rank runs the head and broadcasts the [L, 64] result so that every rank can
    carry the denoising loop on.

    This is the capacity configuration (weights and caches of 1/N of the layers per GPU), NOT a latency one: the
    stages of one stream run one after another, so a single stream gains nothing (SURVEY.md 8e option 1 says so);
    the sequence-parallel mode above is the one that scales a stream.  Hand-off per pass: (N - 1) x 47.9 MB."""

    def __init__(self, group: Optional[dist.ProcessGroup] = None):
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed must be initialised before LayerPipeline()")
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)

    def layers(self, num_layers: int):
        """[lo, hi) of the layers this rank owns (contiguous, as even as possible, earlier ranks take the remainder)."""
        base, extra = divmod(num_layers, self.world)
        lo = self.rank * base + min(self.rank, extra)
        return lo, lo + base + (1 if self.rank < extra else 0)

    def _global(self, r: int) -> int:
        return r if self.group is None else dist.get_global_rank(self.group, r)

    @property
    def first(self) -> bool:
        return self.rank == 0

    @property
    def last(self) -> bool:
        return self.rank == self.world - 1

    def recv_from_previous(self, x: torch.Tensor) -> torch.Tensor:
        """Overwrite ``x`` (contiguous) with the residual stream the previous stage produced."""
        dist.recv(x, src=self._global(self.rank - 1), group=self.group)
        return x

    def send_to_next(self, x: torch.Tensor) -> None:
        dist.send(x.contiguous(), dst=self._global(self.rank + 1), group=self.group)

    def broadcast_from_last(self, x: torch.Tensor) -> torch.Tensor:
        dist.broadcast(x, src=self._global(self.world - 1), group=self.group)
        return x
