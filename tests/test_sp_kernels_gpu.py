"""The sequence-parallel (SP) kernel paths on one GPU.  SP splits the token rows of one stream across W ranks; the
kernels then take a ``row_offset`` (the global index of the local row 0) and, in the p2p mode, store through a table
of W device pointers.  Here W separate buffers on the one device stand in for the W ranks, so every path runs without
a second GPU:

  * row sharding is invisible: ``ln_modulate`` / ``qkv_norm_rope`` on each shard with ``row_offset = r * n_loc`` give
    exactly (``torch.equal``) the rows of one call over all rows -- what the multi-GPU check expects bit for bit;
  * ``qkv_norm_rope_p2p`` fills every rank's head-sharded q / K slot / V slot exactly as slicing the one-GPU output by
    heads, and ``comm_scatter_rows`` is exactly the row split; bytes outside each destination slot are untouched;
  * the gate / residual epilogue of the bf16 and FP8 GEMMs picks the gate row of the GLOBAL row,
    ``(i + row_offset) // rows_per_gate``.  The kernel choice depends on M, so each shard is compared per row with a
    float64 restatement (rounding points of kr_ops.h: cast(res + cast(cast(acc + bias) * gate))): the relative L2
    error of each row's gated term is <= 1e-2 (measured on an H100: <= 1.7e-3); a wrong gate row misses by O(1)."""
import ctypes

import pytest
import torch

from tests import kernel_refs as R

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FS = 1560
L = 3 * FS
SENT = -777.0


def _ops():
    from realtime_video_b200 import ops
    return ops


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _qkv(D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(L, 3 * D, device="cuda", generator=g) * 1.5).to(BF)
    wq = (1 + 0.3 * torch.randn(D, device="cuda", generator=g)).to(BF)
    wk = (1 + 0.3 * torch.randn(D, device="cuda", generator=g)).to(BF)
    return qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:], wq, wk


@pytest.mark.parametrize("W", [2, 4, 8])
def test_row_shards_equal_one_call(W):
    """4680 rows (3 frames of 1560) in W shards: with W = 8 the shards are 585 rows, and shards 2, 5 cross the frame
    boundaries 1560 / 3120, so the per-frame modulation and the RoPE frame index must come from the global row."""
    ops = _ops()
    D, gh, gw = 5120, 30, 52
    n_loc = L // W
    x = (torch.randn(L, D, device="cuda") * 2).to(BF)
    mod = (0.5 * torch.randn(3, 6, D, device="cuda")).to(BF)
    full = ops.ln_modulate(x, eps=1e-6, mod=mod, shift_idx=0, scale_idx=1, rows_per_frame=FS)
    parts = [ops.ln_modulate(x[r * n_loc:(r + 1) * n_loc], eps=1e-6, mod=mod, shift_idx=0, scale_idx=1,
                             rows_per_frame=FS, row_offset=r * n_loc) for r in range(W)]
    assert torch.equal(torch.cat(parts), full)

    q, k, v, wq, wk = _qkv(D, W)
    rope = R.rope_table_f32(128, "cuda")
    rq, rk = torch.empty(L, D, dtype=BF, device="cuda"), torch.empty(L, D, dtype=BF, device="cuda")
    ops.qkv_norm_rope(q, k, None, wq, wk, rq, rk, None, rope, head_dim=128, grid_h=gh, grid_w=gw, start_frame=4,
                      eps=1e-6)
    sq, sk = torch.empty_like(rq), torch.empty_like(rk)
    for r in range(W):
        s = slice(r * n_loc, (r + 1) * n_loc)
        ops.qkv_norm_rope(q[s], k[s], None, wq, wk, sq[s], sk[s], None, rope, head_dim=128, grid_h=gh, grid_w=gw,
                          start_frame=4, eps=1e-6, row_offset=r * n_loc)
    assert torch.equal(sq, rq) and torch.equal(sk, rk)


@pytest.mark.parametrize("W", [2, 4, 8])
def test_qkv_norm_rope_p2p_is_the_head_split(W):
    """Rank r normalises / rotates its own n_loc rows (all heads) and stores head group d's columns into rank d's
    q buffer (row pitch Dh + 16), K slot and V slot (rows [ls, ls + L) of a cache with pitch Dh), at row r * n_loc.
    After all W calls, every rank's buffers equal the one-GPU output sliced by heads, bit for bit, and every byte
    outside the written rows / columns keeps its sentinel.  W = 8 at D 5120 gives peer_cols 640 (5 heads)."""
    ops = _ops()
    D, gh, gw = 5120, 30, 52
    Dh, n_loc, ls = D // W, L // W, 96
    q, k, v, wq, wk = _qkv(D, 100 + W)
    rope = R.rope_table_f32(128, "cuda")
    rq, rk = torch.empty(L, D, dtype=BF, device="cuda"), torch.empty(L, D, dtype=BF, device="cuda")
    ops.qkv_norm_rope(q, k, None, wq, wk, rq, rk, None, rope, head_dim=128, grid_h=gh, grid_w=gw, start_frame=1,
                      eps=1e-6)
    qb = [torch.full((L + 4, Dh + 16), SENT, dtype=BF, device="cuda") for _ in range(W)]
    kb = [torch.full((ls + L + 64, Dh), SENT, dtype=BF, device="cuda") for _ in range(W)]
    vb = [torch.full((ls + L + 64, Dh), SENT, dtype=BF, device="cuda") for _ in range(W)]
    for r in range(W):
        r0 = r * n_loc
        s = slice(r0, r0 + n_loc)
        ops.qkv_norm_rope_p2p(q[s], k[s], v[s], wq, wk, _ptrs([b[2 + r0] for b in qb]), Dh + 16,
                              _ptrs([b[ls + r0] for b in kb]), Dh, _ptrs([b[ls + r0] for b in vb]), Dh, W, Dh, rope,
                              head_dim=128, grid_h=gh, grid_w=gw, start_frame=1, eps=1e-6, row_offset=r0)
    for d in range(W):
        cs = slice(d * Dh, (d + 1) * Dh)
        assert torch.equal(qb[d][2:2 + L, :Dh], rq[:, cs]), d
        assert torch.equal(kb[d][ls:ls + L], rk[:, cs]), d
        assert torch.equal(vb[d][ls:ls + L], v[:, cs]), d
        assert bool((qb[d][:2] == SENT).all() and (qb[d][2 + L:] == SENT).all() and (qb[d][:, Dh:] == SENT).all())
        for b in (kb[d], vb[d]):
            assert bool((b[:ls] == SENT).all() and (b[ls + L:] == SENT).all())


@pytest.mark.parametrize("W", [2, 4, 8])
def test_comm_scatter_rows_is_the_row_split(W):
    """Rank s holds the attention output of ITS heads for ALL rows ([L, Dh]); comm_scatter_rows sends rows
    [d * n_loc, (d + 1) * n_loc) to rank d's row-sharded output at columns [s * Dh, (s + 1) * Dh) (pitch D).  After
    all W calls rank d's rows are exactly the row split of the concatenated head outputs; guards are untouched."""
    ops = _ops()
    D = 5120
    Dh, n_loc = D // W, L // W
    src = [torch.randn(L, Dh, device="cuda").to(BF) for _ in range(W)]
    ob = [torch.full((n_loc + 2, D + 8), SENT, dtype=BF, device="cuda") for _ in range(W)]
    dst = [b[1:1 + n_loc, :D] for b in ob]
    for s in range(W):
        ops.comm_scatter_rows(src[s], _ptrs([o[:, s * Dh:] for o in dst]), D + 8, n_loc, W)
    whole = torch.cat(src, dim=1)
    for d in range(W):
        assert torch.equal(dst[d], whole[d * n_loc:(d + 1) * n_loc]), d
        assert bool((ob[d][0] == SENT).all() and (ob[d][-1] == SENT).all() and (ob[d][:, D:] == SENT).all())


def _gate_ref(a_deq, w_deq, bias, res, gate, r0):
    y = R.r16(a_deq @ w_deq.t() + bias.double())
    g = gate.double()[(torch.arange(a_deq.shape[0], device=a_deq.device) + r0) // FS]
    gated = R.r16(y * g)
    return R.r16(res.double() + gated), gated


def _row_err(out, ref, gated):
    return (out.double() - ref).norm(dim=1) / gated.norm(dim=1).clamp_min(1e-30)


@pytest.mark.parametrize("M,r0", [(585, 1170), (1170, 1170), (2340, 2340), (585, 2925)])
@pytest.mark.parametrize("path", ["bf16", "fp8"])
def test_gemm_gate_epilogue_row_offset(M, r0, path):
    """out = cast(res + cast(cast(a w^T + bias) * gate[(i + r0) // 1560])) on an SP shard of M rows starting at global
    row r0; every shard's global rows cross a gate boundary.  Gate rows differ per frame, so a gate taken from the
    local row index misses whole rows."""
    ops = _ops()
    from realtime_video_b200 import fp8
    N, K = 5120, 1536
    g = torch.Generator(device="cuda").manual_seed(M + r0)
    a = torch.randn(M, K, device="cuda", generator=g).to(BF)
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.03).to(BF)
    bias = (0.1 * torch.randn(N, device="cuda", generator=g)).to(BF)
    res = torch.randn(M, N, device="cuda", generator=g).to(BF)
    gate = (1 + torch.randn(3, N, device="cuda", generator=g)).to(BF)
    kw = dict(epilogue=ops.EPI_BIAS_GATE_RES, residual=res, gate=gate, rows_per_gate=FS, row_offset=r0)
    if path == "bf16":
        out = ops.gemm(a, w, bias, **kw)
        a_deq, w_deq = a.double(), w.double()
    else:
        wq, sw = fp8.quantize_weight(w)
        out = ops.linear_fp8(a, wq, sw, bias, **kw)
        aq, st = ops.fp8_quantize(a)
        a_deq = aq.view(torch.float8_e4m3fn).double() * float(st[1])
        w_deq = wq.view(torch.float8_e4m3fn).double() * sw
    ref, gated = _gate_ref(a_deq, w_deq, bias, res, gate, r0)
    err = _row_err(out, ref, gated)
    worst = float(err.max())
    assert worst <= 1e-2, (worst, int(err.argmax()))
    print(f"gate epilogue {path} M={M} r0={r0}: worst row {worst:.2e}")
