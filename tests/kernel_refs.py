"""Float64 restatements of single kernels, shared by the per-kernel GPU parity tests and checked on the CPU by
``tests/test_kernel_refs_cpu.py`` against ``oracle/dit_oracle.py``, ``oracle/vae_oracle.py`` and torch.

Every function computes in float64 on the device of its inputs and rounds to the 16-bit storage type exactly at
the points the kernel's header comment names (``r16``), so a correct kernel differs from it only where its fp32
arithmetic lands on the other side of a 16-bit rounding boundary: at most one unit in the last place (``ulp``).
Each function also returns the unrounded float64 value where a test bounds the whole rounding chain.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import dit_oracle as O
from oracle import vae_oracle as V

F64 = torch.float64
_MANT = {torch.bfloat16: 7, torch.float16: 10, torch.float32: 23}


def r16(x: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """Round a float64 tensor to ``dtype`` (round-to-nearest-even) and return it as float64."""
    return x.to(dtype).to(F64)


def ulp(x: torch.Tensor, dtype=torch.bfloat16) -> torch.Tensor:
    """Spacing of ``dtype`` values at |x| (float64; the smallest normal spacing at 0)."""
    tiny = torch.finfo(dtype).tiny
    e = torch.floor(torch.log2(x.double().abs().clamp_min(tiny)))
    return torch.exp2(e - _MANT[dtype])


def ulp_excess(got: torch.Tensor, ref: torch.Tensor, dtype=torch.bfloat16):
    """(max |got - ref| / ulp(ref), fraction of elements that are not bit-identical)."""
    g, r = got.double(), ref.double()
    d = (g - r).abs()
    return float((d / ulp(r, dtype)).max()), float((d != 0).double().mean())


# ---------------------------------------------------------------------------------------------
# kr_dit_elem.cu
# ---------------------------------------------------------------------------------------------
def ln_modulate(x, eps, weight=None, bias=None, mod=None, shift_idx=0, scale_idx=1, rows_per_frame=0,
                row_offset=0):
    """y = r16(LN(x) [* w + b]);  out = r16(r16(y * r16(1 + scale[f])) + shift[f]),  f = (row + row_offset) // rpf.
    Returns (out, exact, prod): ``exact`` without any rounding, ``prod`` = y * (1 + scale) (float64 magnitudes of the
    product rounding point, for the rounding-chain bound)."""
    xd = x.double()
    w = None if weight is None else weight.double()
    b = None if bias is None else bias.double()
    exact = O.layer_norm(xd, eps, w, b)
    y = r16(exact)
    if mod is None:
        return y, exact, exact
    f = (torch.arange(x.shape[0], device=x.device) + row_offset) // rows_per_frame
    sc, sh = mod[f, scale_idx].double(), mod[f, shift_idx].double()
    prod = y * r16(1 + sc)
    return r16(r16(prod) + sh), exact * (1 + sc) + sh, prod


def rope_table_f32(head_dim: int, device) -> torch.Tensor:
    """The kernel's (cos, sin) float32 table [1024, head_dim/2, 2] built from the oracle's angles."""
    a = O.rope_table(head_dim)
    return torch.stack([a.cos(), a.sin()], dim=-1).float().contiguous().to(device)


def qk_norm_rope(x, weight, eps, head_dim, grid_h, grid_w, start_frame=0):
    """One of q / k: r16(rope(r16(r16(x * rsqrt(mean x^2 + eps)) * w))) over rows [0, L), L a multiple of
    grid_h * grid_w (row r is frame r // (h*w) + start_frame, row (r % (h*w)) // w, column r % w).
    Returns (rounded, exact)."""
    L, D = x.shape
    hw = grid_h * grid_w
    assert L % hw == 0
    grid = (L // hw, grid_h, grid_w)
    ang = O.rope_table(head_dim).to(x.device)
    xd = x.double()
    n = O.rms_norm(xd, torch.ones(D, dtype=F64, device=x.device), eps)
    a = r16(r16(n) * weight.double())
    out = O.rope_apply(a.view(L, D // head_dim, head_dim), grid, ang, start_frame).reshape(L, D)
    exact = O.rope_apply((n * weight.double()).view(L, D // head_dim, head_dim), grid, ang,
                         start_frame).reshape(L, D)
    return r16(out), exact


def rmsnorm(x, weight, eps):
    """r16(r16(x * rsqrt(mean x^2 + eps)) * w) (model.py:69-85 in bf16)."""
    xd = x.double()
    n = O.rms_norm(xd, torch.ones(x.shape[-1], dtype=F64, device=x.device), eps)
    return r16(r16(n) * weight.double())


def silu(x):
    return F.silu(x.double())


def gelu_tanh(x):
    return F.gelu(x.double(), approximate="tanh")


def patchify(x):
    """x [C, F, H, W] -> [F*(H/2)*(W/2), 4C] in the Conv3d(1,2,2) weight order (c, ph, pw)
    (causal_model.py:614-615: the conv is a matmul of these rows with weight.flatten(1))."""
    C, Fr, H, W = x.shape
    t = x.reshape(C, Fr, H // 2, 2, W // 2, 2).permute(1, 2, 4, 0, 3, 5)    # f, hh, ww, c, ph, pw
    return t.reshape(Fr * (H // 2) * (W // 2), C * 4)


def unpatchify(head_out, C, Fr, H, W):
    """head_out [F*h2*w2, 4C] with column order (ph, pw, c) -> [F, C, H, W] (causal_model.py:1145-1147)."""
    u = head_out.reshape(Fr, H // 2, W // 2, 2, 2, C)                       # f, hh, ww, ph, pw, c
    return u.permute(0, 5, 1, 3, 2, 4).reshape(Fr, C, H, W)


def flow_to_x0(flow, xt, sigma):
    """bf16(double(xt) - sigma[f] * double(flow)) (utils/wan_wrapper.py:181-205), sigma [F] float64."""
    return (xt.double() - sigma.double().view(-1, 1, 1, 1) * flow.double()).to(flow.dtype)


# ---------------------------------------------------------------------------------------------
# kr_attn.cu
# ---------------------------------------------------------------------------------------------
def attention(q, k, v, heads, block_len=0, window=0, pad_keys=0, softmax_scale=None):
    """softmax(scale * q k^T) v per head in float64 -> [Lq, heads*128] float64.

    With ``block_len`` the keys are right-padded with ``pad_keys`` zero rows (score 0, value 0) and the block-causal
    rule of the oracle (``kv < ends[q]``, optional ``kv >= ends[q] - window``) is applied over the padded length, as
    causal_model.py:316-348 pads before FlexAttention."""
    Lq, Lkv = q.shape[0], k.shape[0]
    d = 128
    scale = 1.0 / math.sqrt(d) if softmax_scale is None else softmax_scale
    qd = q.double().view(Lq, heads, d).transpose(0, 1)
    kd = k.double().view(Lkv, heads, d).transpose(0, 1)
    vd = v.double().view(Lkv, heads, d).transpose(0, 1)
    if block_len and pad_keys:
        kd = torch.cat([kd, kd.new_zeros(heads, pad_keys, d)], dim=1)
        vd = torch.cat([vd, vd.new_zeros(heads, pad_keys, d)], dim=1)
    s = (qd @ kd.transpose(1, 2)) * scale
    if block_len:
        m = O.block_causal_mask(Lq, kd.shape[1], block_len, window, q.device)
        s = s.masked_fill(~m, float("-inf"))
    return (torch.softmax(s, dim=-1) @ vd).transpose(0, 1).reshape(Lq, heads * d)


def rel_rows_heads(got, ref, heads):
    """Relative L2 error of every (row, head) 128-vector; returns the [L, heads] float64 tensor."""
    g = got.double().view(got.shape[0], heads, -1)
    r = ref.double().view(ref.shape[0], heads, -1)
    return (g - r).norm(dim=-1) / r.norm(dim=-1).clamp_min(1e-300)


# ---------------------------------------------------------------------------------------------
# kr_attn.cu attn_fwd_kernel and kr_t5attn.cu t5_attn_kernel: their online-softmax schedules as float64 intervals
# ---------------------------------------------------------------------------------------------
# |s - q.k| <= C_S |q|.|k| for the fp32 wgmma scores, |O - sum P v| <= C_PV sum P |v| for the fp32 P V accumulator
# (carried across tiles and rescales), and the relative error of ex2.approx.ftz.f32 (assumed, not measured: no case
# needs any).  The smallest values both kernels still pass on an H100 SXM (700 W) are 2^-23 for both C_S and C_PV
# (tests/test_attn_parity_gpu.py); each constant is 8x that.
C_S = 2.0 ** -20
C_PV = 2.0 ** -20
EXP2_REL = 2.0 ** -21
U32 = 2.0 ** -24                     # fp32 unit roundoff
TINY32 = 2.0 ** -126                 # smallest normal fp32: ex2.approx.ftz flushes results below it to 0
LOG2E_F32 = float(torch.tensor(1.4426950408889634, dtype=torch.float32))   # log2 e as the kernels hold it
T5_MIN = float(torch.finfo(torch.bfloat16).min)
ATTN_TILE = 128


def f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def attn_scale_log2(softmax_scale=None) -> float:
    """kr_attn_fwd's scale_log2 = fp32(scale) * fp32(log2 e), rounded to fp32 (kr_api.cu)."""
    scale = 1.0 / math.sqrt(128) if softmax_scale is None else softmax_scale
    return f32(f32(scale) * LOG2E_F32)


def attn_rows(Lq, Lkv, block_len=0, window=0, pad_keys=0, device="cpu"):
    """(row_lo, row_hi, n_phantom) int64 [Lq]: the keys [row_lo, row_hi) each query row sees and the number of padded
    (phantom) keys it adds in the epilogue, exactly as attn_fwd_kernel derives them."""
    rows = torch.arange(Lq, device=device)
    if not block_len:
        z = torch.zeros_like(rows)
        return z, z + Lkv, z
    hi = (rows // block_len + 1) * block_len
    lo = (hi - window).clamp_min(0) if window > 0 else torch.zeros_like(rows)
    n_ph = (hi - Lkv).clamp_min(0).clamp_max(pad_keys)
    return lo, hi.clamp_max(Lkv), n_ph


def _exp2_bounds(a_lo, a_hi, c_exp):
    """[lo, hi] of ex2.approx.ftz(x) for x in [a_lo, a_hi] (float64; results below 2^-126 may be flushed to 0)."""
    lo = torch.exp2(a_lo) * (1 - c_exp)
    return torch.where(lo < TINY32, torch.zeros_like(lo), lo), torch.exp2(a_hi) * (1 + c_exp)


def _scale_interval(x_lo, x_hi, a_lo, a_hi):
    """[x_lo, x_hi] * [a_lo, a_hi] for a_lo >= 0, widened by one fp32 rounding of the product."""
    lo = torch.minimum(x_lo * a_lo, x_lo * a_hi)
    hi = torch.maximum(x_hi * a_lo, x_hi * a_hi)
    return lo - U32 * lo.abs(), hi + U32 * hi.abs()


def _pv_interval(P_lo, P_hi, v):
    """[lo, hi] of P v over P in [P_lo, P_hi] (P >= 0) elementwise, and P_hi |v|."""
    vp, vn = v.clamp_min(0), v.clamp_max(0)
    return P_lo @ vp + P_hi @ vn, P_hi @ vp + P_lo @ vn, P_hi @ v.abs()


def _l_chain(n_tiles, n_rescale):
    """Relative bound of the fp32 row sum l: each thread adds the pairs a0 + a1 of its 2 columns of every 8 (32 adds
    per tile), is multiplied by alpha on every rescale, then 2 shuffle adds; every term is >= 0."""
    return (32 * n_tiles + n_rescale + 4) * U32 * 1.01


def _flash_walk(qh, kh, vh, sl2, row_lo, row_hi, dtype, c_s, c_pv, c_exp, rescale_if_ambiguous):
    """One head of attn_fwd_kernel's tile walk.  Returns the interval state (O_lo, O_hi, A, l_lo, l_hi, mu_lo, mu_hi,
    n_ambiguous [Lq]): O and l are bounded in the frame of the kernel's own (unknown) m_used, mu = m_used * sl2 in
    log2 units (-inf while the row has seen no key), A = the P_hi |v| sum behind the C_PV bound."""
    Lq, dev = qh.shape[0], qh.device
    inf = torch.tensor(float("inf"), dtype=F64, device=dev)
    mu_lo = torch.full((Lq,), -float("inf"), dtype=F64, device=dev)
    mu_hi = mu_lo.clone()
    O_lo = torch.zeros(Lq, vh.shape[1], dtype=F64, device=dev)
    O_hi, A = O_lo.clone(), O_lo.clone()
    l_lo = torch.zeros(Lq, dtype=F64, device=dev)
    l_hi = l_lo.clone()
    amb = torch.zeros(Lq, dtype=torch.int64, device=dev)
    n_resc = torch.zeros(Lq, dtype=torch.int64, device=dev)
    qa = qh.abs()
    for k0 in range(0, int(row_hi.max()), ATTN_TILE):
        k1 = min(k0 + ATTN_TILE, kh.shape[0])
        cols = torch.arange(k0, k1, device=dev)
        vis = (cols[None] >= row_lo[:, None]) & (cols[None] < row_hi[:, None])
        has = vis.any(1)
        if not bool(has.any()):
            continue
        t = (qh @ kh[k0:k1].t()) * sl2
        dl = (qa @ kh[k0:k1].abs().t()) * (c_s * sl2)
        t_lo = torch.where(vis, t - dl, -inf)
        t_hi = torch.where(vis, t + dl, -inf)
        tmax_lo, tmax_hi = t_lo.amax(1), t_hi.amax(1)
        # need = fl(fl(m_new - m_run) * sl2) > 8, m_new = max(m_run, tile max); certain on a row's first keys
        first = has & torch.isinf(mu_lo)
        D_lo, D_hi = tmax_lo - mu_hi, tmax_hi - mu_lo
        sure = first | (has & (D_lo * (1 - 4 * U32) > 8))
        maybe = has & ~sure & (D_hi * (1 + 4 * U32) > 8)
        amb += maybe.long()
        resc = sure | (maybe & rescale_if_ambiguous)
        old = resc & ~first
        if bool(old.any()):
            # alpha = ex2(fl(fl(m_run - m_new) * sl2)) on O and l, in the old frame
            a_lo, a_hi = mu_lo - tmax_hi, mu_hi - tmax_lo
            al_lo, al_hi = _exp2_bounds(a_lo - 2 * U32 * a_lo.abs(), a_hi + 2 * U32 * a_hi.abs(), c_exp)
            ol, oh = _scale_interval(O_lo, O_hi, al_lo[:, None], al_hi[:, None])
            o2 = old[:, None]
            O_lo, O_hi = torch.where(o2, ol, O_lo), torch.where(o2, oh, O_hi)
            A = torch.where(o2, A * al_hi[:, None] * (1 + U32), A)
            l_lo = torch.where(old, l_lo * al_lo, l_lo)
            l_hi = torch.where(old, l_hi * al_hi, l_hi)
            n_resc += old.long()
        mu_lo = torch.where(resc, tmax_lo, mu_lo)
        mu_hi = torch.where(resc, tmax_hi, mu_hi)
        # p = ex2.approx(fl(s * sl2 + fl(-m_used * sl2))): both roundings, the key's and the max's own +-delta
        mabs = torch.maximum(mu_lo.abs(), mu_hi.abs()).nan_to_num(0.0, posinf=0.0)
        d_lo = t_lo - (mu_hi + U32 * mabs)[:, None]
        d_hi = t_hi - (mu_lo - U32 * mabs)[:, None]
        d_lo = torch.where(vis, d_lo - U32 * d_lo.abs(), -inf)
        d_hi = torch.where(vis, d_hi + U32 * d_hi.abs(), -inf)
        p_lo, p_hi = _exp2_bounds(d_lo, d_hi, c_exp)
        P_lo, P_hi = r16(p_lo, dtype), r16(p_hi, dtype)
        l_lo, l_hi = l_lo + p_lo.sum(1), l_hi + p_hi.sum(1)
        a, b, c = _pv_interval(P_lo, P_hi, vh[k0:k1])
        O_lo, O_hi, A = O_lo + a, O_hi + b, A + c
    n_tiles = (row_hi + ATTN_TILE - 1) // ATTN_TILE
    g = _l_chain(n_tiles, n_resc).double()
    return O_lo, O_hi, A, l_lo * (1 - g), l_hi * (1 + g), mu_lo, mu_hi, amb


def _flash_epilogue(O_lo, O_hi, A, l_lo, l_hi, mu_lo, mu_hi, n_ph, c_pv, c_exp):
    """Unrounded [lo, hi] of fl(O * inv_l) with the phantom keys: m_fin = max(m, 0), o_scale = ex2((m - m_fin) sl2),
    l' = l o_scale + n_ph ex2(-m_fin sl2), inv_l = o_scale / l'  ==  1 / (l + n_ph 2^-mu) for either sign of mu."""
    E = c_pv * A + 2.0 ** -120
    O_lo, O_hi = O_lo - E, O_hi + E
    seen = ~torch.isinf(mu_lo)
    mabs = torch.where(seen, torch.maximum(mu_lo.abs(), mu_hi.abs()), torch.zeros_like(mu_lo))
    nph = n_ph.double()
    ph_lo = torch.where(seen, nph * torch.exp2(-(mu_hi + U32 * mabs)) * (1 - c_exp), nph)
    ph_hi = torch.where(seen, nph * torch.exp2(-(mu_lo - U32 * mabs)) * (1 + c_exp), nph)
    den_lo, den_hi = l_lo + ph_lo, l_hi + ph_hi
    if bool((den_lo <= 0).any()):
        raise ValueError("attn_interval: a row sees neither a key nor a padded key (its softmax is undefined)")
    rel = 2 * c_exp + 6 * U32
    inv_lo, inv_hi = (1 - rel) / den_hi, (1 + rel) / den_lo
    # ex2 of (m - m_fin) sl2 below -126 flushes o_scale, and with it the row, to 0
    inv_lo = torch.where((n_ph > 0) & (mu_lo < -125), torch.zeros_like(inv_lo), inv_lo)
    inv_lo = torch.where(seen, inv_lo, torch.zeros_like(inv_lo))     # no real key: o_scale = 0
    inv_hi = torch.where(seen, inv_hi, torch.zeros_like(inv_hi))
    return _scale_interval(O_lo, O_hi, inv_lo[:, None], inv_hi[:, None])


def attn_interval(q, k, v, heads, block_len=0, window=0, pad_keys=0, softmax_scale=None, dtype=torch.bfloat16,
                  head_list=None, *, c_s=C_S, c_pv=C_PV, c_exp=EXP2_REL):
    """Per-element [lo, hi] (float64 holding ``dtype`` values) of attn_fwd_kernel's 16-bit output, restating its
    schedule rather than softmax: 128-key tiles in order; scores t = sl2 (q.k) in log2 units with the bound
    delta = C_S sl2 |q|.|k|; the visible keys [row_lo, row_hi) of :func:`attn_rows`; the lazy running max (rescale only
    when the tile's max exceeds m_used by more than 8, else P is taken against the stale m_used and may reach 2^8;
    m_used = -inf until the row's first visible key); p = 2^(t - m_used) with both +-delta, EXP2_REL, the fp32
    rounding of the fma argument and ftz; P = [r16(p_lo), r16(p_hi)]; l sums the unrounded p (fp32 chain bound of
    :func:`_l_chain`), O sums P v (C_PV sum P |v|); alpha on a rescale carries its own EXP2_REL; the epilogue of
    :func:`_flash_epilogue`.  A lazy decision within the error margin of the threshold is ambiguous: the walk runs
    again deciding every ambiguous tile the other way, and the union is returned (rows with two or more ambiguous tiles
    are not enumerated over mixed decisions; the count lets a test report them).

    Returns (lo, hi, info) with lo / hi [Lq, len(head_list) * 128] and info: ``u_lo`` / ``u_hi`` (the unrounded
    bounds), ``ambiguous`` (number of ambiguous tiles), ``heads`` (the restated heads, all by default)."""
    Lq, Lkv = q.shape[0], k.shape[0]
    head_list = list(range(heads)) if head_list is None else list(head_list)
    sl2 = attn_scale_log2(softmax_scale)
    row_lo, row_hi, n_ph = attn_rows(Lq, Lkv, block_len, window, pad_keys, q.device)
    us_lo, us_hi, n_amb = [], [], 0
    for h in head_list:
        cs = slice(h * 128, (h + 1) * 128)
        qh, kh, vh = q[:, cs].double(), k[:, cs].double(), v[:, cs].double()
        lo = hi = None
        for policy in (False, True):
            st = _flash_walk(qh, kh, vh, sl2, row_lo, row_hi, dtype, c_s, c_pv, c_exp, policy)
            a, b = _flash_epilogue(*st[:7], n_ph, c_pv, c_exp)
            lo = a if lo is None else torch.minimum(lo, a)
            hi = b if hi is None else torch.maximum(hi, b)
            n = int(st[7].sum())
            if not policy:
                n_amb += n
            if n == 0:
                break
        us_lo.append(lo)
        us_hi.append(hi)
    u_lo, u_hi = torch.cat(us_lo, 1), torch.cat(us_hi, 1)
    return r16(u_lo, dtype), r16(u_hi, dtype), {"u_lo": u_lo, "u_hi": u_hi, "ambiguous": n_amb, "heads": head_list}


def t5_attn_interval(q, k, v, bias_delta, key_mask, heads, *, c_s=C_S, c_pv=C_PV, c_exp=EXP2_REL):
    """Per-element [lo, hi] of t5_attn_kernel's bf16 output [L, heads*64] (head_dim 64, no scaling): per key
    r16(s) as an interval ([r16(s - C_S |q|.|k|), r16(s + ...)], nearly always one value), then
    r16(r16(s) + bias[h, k - q + L - 1]); masked keys are finfo.min, keys past L are excluded.  The running max is
    exact (not lazy) over these bf16 values; p = ex2(fl(fl(v - m) log2e)) (the difference of two bf16 values is exact in
    fp32) with EXP2_REL and ftz, P = r16(p) un-normalised, l and O in fp32 with the rescale by
    alpha = ex2(fl(fl(m_run - m_new) log2e)), and out = r16(O / l).  A row whose first tile is masked whole runs that
    tile's softmax over equal finfo.min values (p = 1) until a real key's alpha = 0 drops it; an all-masked row ends as
    the mean of V.  Returns (lo, hi, info) as :func:`attn_interval`."""
    L, dev = q.shape[0], q.device
    d = q.shape[1] // heads
    bf = torch.bfloat16
    idx = torch.arange(L, device=dev)
    off = idx[None, :] - idx[:, None] + (L - 1)
    km = torch.ones(L, dtype=torch.bool, device=dev) if key_mask is None else key_mask.to(dev) != 0
    us_lo, us_hi = [], []
    for h in range(heads):
        cs = slice(h * d, (h + 1) * d)
        qh, kh, vh = q[:, cs].double(), k[:, cs].double(), v[:, cs].double()
        S = qh @ kh.t()
        E = c_s * (qh.abs() @ kh.abs().t())
        b = bias_delta[h].double()[off]
        val_lo = torch.where(km[None], r16(r16(S - E, bf) + b, bf), torch.full_like(S, T5_MIN))
        val_hi = torch.where(km[None], r16(r16(S + E, bf) + b, bf), torch.full_like(S, T5_MIN))
        m_lo = torch.full((L,), -float("inf"), dtype=F64, device=dev)
        m_hi = m_lo.clone()
        O_lo = torch.zeros(L, d, dtype=F64, device=dev)
        O_hi, A = O_lo.clone(), O_lo.clone()
        l_lo = torch.zeros(L, dtype=F64, device=dev)
        l_hi = l_lo.clone()
        n_tiles = (L + ATTN_TILE - 1) // ATTN_TILE
        for k0 in range(0, L, ATTN_TILE):
            k1 = min(k0 + ATTN_TILE, L)
            vl, vu = val_lo[:, k0:k1], val_hi[:, k0:k1]
            n_lo, n_hi = torch.maximum(m_lo, vl.amax(1)), torch.maximum(m_hi, vu.amax(1))
            if k0 > 0:
                a_lo, a_hi = (m_lo - n_hi) * LOG2E_F32, (m_hi - n_lo) * LOG2E_F32
                al_lo, al_hi = _exp2_bounds(a_lo - 2 * U32 * a_lo.abs(), a_hi + 2 * U32 * a_hi.abs(), c_exp)
                O_lo, O_hi = _scale_interval(O_lo, O_hi, al_lo[:, None], al_hi[:, None])
                A = A * al_hi[:, None] * (1 + U32)
                l_lo, l_hi = l_lo * al_lo, l_hi * al_hi
            m_lo, m_hi = n_lo, n_hi
            x_lo = (vl - m_hi[:, None]) * LOG2E_F32
            x_hi = (vu - m_lo[:, None]) * LOG2E_F32
            x_lo, x_hi = x_lo - 2 * U32 * x_lo.abs(), x_hi + 2 * U32 * x_hi.abs()
            p_lo, p_hi = _exp2_bounds(x_lo, x_hi, c_exp)
            P_lo, P_hi = r16(p_lo, bf), r16(p_hi, bf)
            l_lo, l_hi = l_lo + p_lo.sum(1), l_hi + p_hi.sum(1)
            a, b2, c = _pv_interval(P_lo, P_hi, vh[k0:k1])
            O_lo, O_hi, A = O_lo + a, O_hi + b2, A + c
        g = _l_chain(n_tiles, n_tiles)
        l_lo, l_hi = l_lo * (1 - g), l_hi * (1 + g)
        Eo = c_pv * A + 2.0 ** -120
        inv_lo, inv_hi = (1 - U32) / l_hi, (1 + U32) / l_lo
        lo, hi = _scale_interval(O_lo - Eo, O_hi + Eo, inv_lo[:, None], inv_hi[:, None])
        us_lo.append(lo)
        us_hi.append(hi)
    u_lo, u_hi = torch.cat(us_lo, 1), torch.cat(us_hi, 1)
    return r16(u_lo, bf), r16(u_hi, bf), {"u_lo": u_lo, "u_hi": u_hi, "ambiguous": 0, "heads": list(range(heads))}


def check_attn(got, lo, hi, dtype, info=None):
    """Hold an attention output to its restated interval with zero slack.  Returns (violations, stats): ``span``
    (fraction of elements whose interval holds more than one 16-bit value), ``frac`` (fraction not equal to r16 of the
    unrounded midpoint), ``ratio`` (the largest share of the interval's unrounded half-width an element needed: the
    distance from the midpoint to the rounding boundary on the element's side, as :func:`acc_ratio`; <= 1 inside),
    ``ambiguous`` (lazy decisions within the threshold's error margin)."""
    viol = []
    g = got.double()
    if not bool(torch.isfinite(g).all()):
        viol.append(f"{int((~torch.isfinite(g)).sum())} non-finite elements")
        g = torch.nan_to_num(g, nan=1e300)
    out = (g < lo) | (g > hi)
    if bool(out.any()):
        i = int(out.flatten().nonzero()[0])
        r, c = divmod(i, g.shape[1])
        viol.append(f"{int(out.sum())} elements outside the restated interval, first ({r}, {c}): "
                    f"{float(g[r, c]):.8g} not in [{float(lo[r, c]):.8g}, {float(hi[r, c]):.8g}]")
    stats = {"span": float((lo != hi).double().mean()), "ambiguous": 0, "ratio": 0.0, "frac": 0.0}
    if info is not None:
        mid = 0.5 * (info["u_lo"] + info["u_hi"])
        half = 0.5 * (info["u_hi"] - info["u_lo"])
        off = g != r16(mid, dtype)
        stats["frac"] = float(off.double().mean())
        stats["ambiguous"] = info["ambiguous"]
        if bool(off.any()):
            y, mm, hh = g[off], mid[off], half[off]
            bnd = 0.5 * (y + _bits_neighbour(y, y < mm, dtype))
            stats["ratio"] = float(((bnd - mm).abs() / hh.clamp_min(1e-300)).max())
    return viol, stats


# ---------------------------------------------------------------------------------------------
# kr_vae.cu
# ---------------------------------------------------------------------------------------------
def vae_rmsnorm(x, gamma, dtype):
    """RMS_norm of vae.py:39-54 on channels-last x [..., C] with the 16-bit eager rounding points:
    n = r16(||x||), y = r16(x / n), y = r16(r16(y * sqrt(C)) * gamma).  Returns (rounded, exact)."""
    xd = x.double()
    C = x.shape[-1]
    n = r16(xd.norm(dim=-1, keepdim=True), dtype)
    y = r16(xd / n.clamp_min(1e-12), dtype)
    y = r16(r16(y * math.sqrt(C), dtype) * gamma.double(), dtype)
    exact = V.rms_norm(xd.movedim(-1, 1), gamma.double().view(-1, *([1] * (x.dim() - 2)))).movedim(1, -1) \
        if x.dim() >= 2 else None
    return y, exact


def vae_rmsnorm_silu(x, gamma, dtype):
    """The kernel's output r16(SiLU(y)) of :func:`vae_rmsnorm` (SiLU evaluated on the rounded y), and SiLU(exact)."""
    y, exact = vae_rmsnorm(x, gamma, dtype)
    return r16(F.silu(y), dtype), F.silu(exact)


def softmax_rows(s):
    return torch.softmax(s.double(), dim=-1)


# ---------------------------------------------------------------------------------------------
# kr_gemm.cu, kr_gemm2.cu, kr_gemm_sk.cu, kr_gemm_fp8.cu (gemm_epilogue_row's rounding points)
# ---------------------------------------------------------------------------------------------
EPI_BIAS, EPI_BIAS_GELU, EPI_BIAS_GATE_RES, EPI_BIAS_RES, EPI_F32, EPI_MUL = 0, 1, 2, 3, 4, 5
EPI_NAMES = {EPI_BIAS: "bias", EPI_BIAS_GELU: "gelu", EPI_BIAS_GATE_RES: "gate_res", EPI_BIAS_RES: "res",
             EPI_F32: "f32", EPI_MUL: "mul"}
# The accumulation bound E = c_acc * (|a| |w|^T) of one kernel family, float64 operands decoded exactly.  Largest
# ratio observed on an H100 SXM (700 W) by tests/test_gemm_parity_gpu.py: 3.7e-6 = 2^-18.0 for 16-bit operands (the
# VAE's P V at K = 14400; <= 8.6e-7 at K <= 5120), 6.4e-5 = 2^-13.9 for e4m3 with per-k-block promotion.  Each
# constant is >= 4x that; a dropped k-block of unit-variance operands at K = 5120 exceeds E_16 > 100-fold (median) and
# E_e4m3 on most elements.
C_ACC_16 = 2.0 ** -16
C_ACC_E4M3 = 2.0 ** -11
# the fp32 operations between the accumulator and the first 16-bit rounding (scales, bias add), relative
F32_EPI = 2.0 ** -22
# the fp32 tanhf GELU of the kernel: absolute error bound (a few ulps of 1 + tanh, times x / 2) and the largest
# fraction of elements allowed to round to a neighbour of the float64 GELU
_GELU_ABS = 2.0 ** -21
GELU_MAX_FRAC = 5e-3
GELU_ARGMIN, GELU_MIN = -0.7524614212122512, -0.170040750571254
# guard buffers: bits no kernel writes (a NaN in bf16, fp16 and fp32)
SENTINEL16, SENTINEL32 = 0x7E5A, 0x7FC0DEAD
GUARD_ROWS, GUARD_COLS = 3, 8


def gemm_interval(a, w, bias=None, row_scale=None, col_scale=None, c_acc=C_ACC_16):
    """(z, m, E) in float64 on the device of the operands: z = (a w^T) [* row_scale[m]] [* col_scale[n]] + bias,
    m = |a| |w|^T with the same scales, and the bound E = c_acc * m + 2^-22 (|z| + |bias|) that the kernel's fp32
    result before its first 16-bit rounding must lie within.  ``a`` / ``w`` are already decoded to a float type
    (e4m3 operands decode exactly); ``col_scale`` may be a Python float (the per-tensor FP8 scale)."""
    a64, w64 = a.double(), w.double()
    z = a64 @ w64.t()
    m = a64.abs() @ w64.abs().t()
    if row_scale is not None:
        rs = row_scale.double().view(-1, 1)
        z, m = z * rs, m * rs.abs()
    if col_scale is not None:
        cs = col_scale.double().view(1, -1) if torch.is_tensor(col_scale) else float(col_scale)
        z = z * cs
        m = m * (cs.abs() if torch.is_tensor(cs) else abs(cs))
    babs = 0.0
    if bias is not None:
        z = z + bias.double()
        babs = bias.double().abs()
    return z, m, c_acc * m + F32_EPI * (z.abs() + babs)


def _bits_neighbour(y: torch.Tensor, up: torch.Tensor, dtype) -> torch.Tensor:
    """The 16-bit value adjacent to y (float64 holding dtype values) above it where ``up``, below it elsewhere."""
    b = y.to(dtype).view(torch.int16).to(torch.int32)
    o = torch.where(b < 0, -(b & 0x7FFF), b)                      # sign-magnitude -> ordered integers
    o = o + torch.where(up, 1, -1)
    b = torch.where(o < 0, (-o) | 0x8000, o).to(torch.int16)    # -0 and +0 are one step apart here: harmless
    return b.view(dtype).to(F64)


def acc_ratio(y16, z, m, dtype) -> float:
    """Largest c for which y16 = r16(acc + b) needs |acc + b - z| >= c * m: the distance from z to the rounding
    boundary nearest to it on y16's side, over m, for the elements where y16 != r16(z) (0 elsewhere)."""
    y = y16.double()
    off = y != r16(z, dtype)
    if not bool(off.any()):
        return 0.0
    y, zz, mm = y[off], z[off], m[off]
    mid = 0.5 * (y + _bits_neighbour(y, y < zz, dtype))
    return float(((mid - zz).abs() / mm.clamp_min(1e-300)).max())


def gelu_interval(lo, hi):
    """[min, max] of GELU-tanh over [lo, hi] (float64): monotone except for its minimum at GELU_ARGMIN."""
    g_lo, g_hi = gelu_tanh(lo), gelu_tanh(hi)
    mn = torch.minimum(g_lo, g_hi)
    mn = torch.where((lo < GELU_ARGMIN) & (hi > GELU_ARGMIN), torch.full_like(mn, GELU_MIN), mn)
    return mn, torch.maximum(g_lo, g_hi)


def gate_rows(M, gate, rows_per_gate, row_offset, device):
    """gate[(row + row_offset) // rows_per_gate] for rows [0, M), float64."""
    g = (torch.arange(M, device=device) + row_offset) // rows_per_gate
    return gate.double()[g]


def epi_chain(epi, y16, dtype, residual=None, gate_r=None):
    """gemm_epilogue_row on the rounded first value y16 = r16(acc + b) (float64), with the kernel's rounding points:
    r16(gelu(y16)), r16(res + r16(y16 * g)), r16(res + y16), r16(y16 * res).  Exact for every epilogue but GELU
    (the products and sums of two 16-bit values are exact in fp32); for GELU the unrounded float64 value."""
    if epi == EPI_BIAS:
        return y16
    if epi == EPI_BIAS_GELU:
        return gelu_tanh(y16)
    res = residual.double()
    if epi == EPI_BIAS_GATE_RES:
        return r16(res + r16(y16 * gate_r, dtype), dtype)
    if epi == EPI_BIAS_RES:
        return r16(res + y16, dtype)
    if epi == EPI_MUL:
        return r16(y16 * res, dtype)
    raise ValueError(epi)


def _mul_interval(lo, hi, f):
    a, b = lo * f, hi * f
    return torch.minimum(a, b), torch.maximum(a, b)


def chain_interval(epi, lo, hi, dtype, residual=None, gate_r=None):
    """The epilogue chain applied to both ends of y16's interval [lo, hi] (every step monotone on it, or bounded by
    its extremum), so that any correct kernel's output lies inside the returned [lo, hi]."""
    if epi == EPI_BIAS:
        return lo, hi
    if epi == EPI_BIAS_GELU:
        g_lo, g_hi = gelu_interval(lo, hi)
        return (r16(g_lo - _GELU_ABS * lo.abs().maximum(hi.abs()), dtype),
                r16(g_hi + _GELU_ABS * lo.abs().maximum(hi.abs()), dtype))
    res = residual.double()
    if epi == EPI_BIAS_GATE_RES:
        p_lo, p_hi = _mul_interval(lo, hi, gate_r)
        return r16(res + r16(p_lo, dtype), dtype), r16(res + r16(p_hi, dtype), dtype)
    if epi == EPI_BIAS_RES:
        return r16(res + lo, dtype), r16(res + hi, dtype)
    if epi == EPI_MUL:
        p_lo, p_hi = _mul_interval(lo, hi, res)
        return r16(p_lo, dtype), r16(p_hi, dtype)
    raise ValueError(epi)


def _outside(got, lo, hi, scale):
    """Largest distance of got outside [lo, hi], in units of ``scale`` (0 when every element is inside)."""
    d = (lo - got).clamp_min(0) + (got - hi).clamp_min(0)
    return float((d / scale).max()) if d.numel() else 0.0


def check_gemm(epi, got, z, m, E, dtype, *, residual=None, gate_r=None, alpha=1.0, y16=None):
    """Hold one GEMM output to the float64 reference.  Returns (violations, stats).

    got: the kernel's output (16-bit, or fp32 for EPI_F32).  z, m, E: :func:`gemm_interval`.  y16: the EPI_BIAS
    output of the SAME kernel on the same operands (same accumulation order), when the planner sent both there; the
    rest of the chain is then checked exactly (GELU: within the fp32 tanhf error on all elements, and not
    bit-identical on at most GELU_MAX_FRAC of them).  Every epilogue is also checked against the accumulation
    interval carried through the chain.  stats: ``excess`` (ulps outside the interval), ``frac`` (elements not equal
    to the chain applied to r16(z)), ``ratio`` (:func:`acc_ratio`, first-rounding epilogues only)."""
    viol = []
    g = got.double()
    if not bool(torch.isfinite(g).all()):
        viol.append("non-finite output")
        g = torch.nan_to_num(g, nan=1e300)
    if epi == EPI_F32:
        lo, hi = (z - E) * alpha, (z + E) * alpha
        u = ulp(torch.maximum(lo.abs(), hi.abs()), torch.float32)
        ex = _outside(g, lo - 2 * u, hi + 2 * u, u)
        if ex > 0:
            viol.append(f"f32: {ex:.3g} fp32 ulps outside [(z-E)a, (z+E)a] widened by 2 ulps")
        d = (g / alpha - z).abs() if alpha != 0 else (g - z).abs()
        ratio = float(((d - 2 * u / abs(alpha)).clamp_min(0) / m.clamp_min(1e-300)).max())
        return viol, {"excess": ex, "frac": float((g != (z * alpha).float().double()).double().mean()),
                      "ratio": ratio}
    lo, hi = r16(z - E, dtype), r16(z + E, dtype)
    c_lo, c_hi = chain_interval(epi, lo, hi, dtype, residual, gate_r)
    ex = _outside(g, c_lo, c_hi, ulp(g, dtype))
    if ex > 0:
        viol.append(f"{EPI_NAMES[epi]}: {ex:.3g} ulps outside the accumulation interval")
    nearest = epi_chain(epi, r16(z, dtype), dtype, residual, gate_r)
    stats = {"excess": ex, "frac": float((g != r16(nearest, dtype)).double().mean())}
    if epi == EPI_BIAS:
        stats["ratio"] = acc_ratio(g, z, m, dtype)
    if y16 is not None:
        want = epi_chain(epi, y16.double(), dtype, residual, gate_r)
        if epi == EPI_BIAS_GELU:
            s = _GELU_ABS * y16.double().abs()
            ex2 = _outside(g, r16(want - s, dtype), r16(want + s, dtype), ulp(g, dtype))
            fr = float((g != r16(want, dtype)).double().mean())
            stats["chain_frac"] = fr
            if ex2 > 0 or fr > GELU_MAX_FRAC:
                viol.append(f"gelu chain: {ex2:.3g} ulps outside the fp32 GELU error, {fr:.3g} not bit-identical")
        else:
            bad = int((g != want).sum())
            stats["chain_frac"] = bad / max(1, g.numel())
            if bad:
                viol.append(f"{EPI_NAMES[epi]} chain: {bad} elements differ from the exact restatement")
    return viol, stats


def guarded(rows: int, cols: int, dtype, device, fill=None):
    """A [rows, cols] view inside a sentinel-filled buffer with GUARD_ROWS rows above and below and GUARD_COLS + 16
    columns beside it (row pitch cols + 24 > cols, 16-byte aligned).  ``fill``, if given, is copied into the view."""
    buf = torch.empty(rows + 2 * GUARD_ROWS, cols + 3 * GUARD_COLS, dtype=dtype, device=device)
    if dtype == torch.float32:
        buf.view(torch.int32).fill_(SENTINEL32)
    else:
        buf.view(torch.int16).fill_(SENTINEL16)
    view = buf[GUARD_ROWS:GUARD_ROWS + rows, GUARD_COLS:GUARD_COLS + cols]
    if fill is not None:
        view.copy_(fill)
    return buf, view


def guard_intact(buf: torch.Tensor, rows: int, cols: int) -> bool:
    """True when every element of ``buf`` outside the view of :func:`guarded` still holds the sentinel."""
    if buf.dtype == torch.float32:
        bits, s = buf.view(torch.int32), SENTINEL32
    else:
        bits, s = buf.view(torch.int16), SENTINEL16
    keep = torch.ones(bits.shape, dtype=torch.bool, device=buf.device)
    keep[GUARD_ROWS:GUARD_ROWS + rows, GUARD_COLS:GUARD_COLS + cols] = False
    return bool((bits[keep] == s).all())


# ---------------------------------------------------------------------------------------------
# kr_vae.cu conv_igemm_kernel / conv_halo_kernel (conv_epilogue_frag's rounding points)
# ---------------------------------------------------------------------------------------------
# the fused RMS_norm -> SiLU of the epilogue against vae_rmsnorm_silu on the kernel's own raw values: not bit-identical
# (fp32 sum of squares, a multiply by the fp32 reciprocal of the norm instead of a division, __expf) on at most
# NORM_MAX_FRAC of the elements.  A 1-ulp difference at one of the three 16-bit roundings before the SiLU grows to a few
# ulps of the output where SiLU is small against its argument (x < 0), so at most NORM_FAR_FRAC of the elements may be
# more than 1 ulp away, and none more than NORM_FAR_ULPS.  An emulation of the kernel's fp32 arithmetic on 3.8e7
# random elements shows 6 ulps on 9e-6 of them; on an H100 SXM (700 W) the worst was 5 ulps, with 4.3e-4 of the
# elements not bit-identical.
NORM_MAX_FRAC, NORM_FAR_FRAC, NORM_FAR_ULPS = 2e-2, 1e-4, 8
CONV_FORMS = ("raw", "res", "norm", "head")


def conv_interval(x, w5, bias, taps, sub2=False, T=None, c_acc=C_ACC_16, frames_per_chunk=4):
    """(z, m, E) float64 [T, Ho, Wo, rows] of the causal conv on the device of its operands.

    x [t_in, H, W, cin] holds the kt - 1 history frames in front of the T new ones (T defaults to t_in - kt + 1; frames
    past T + kt - 1 are not read); w5 [rows, kt, kh, kw, cin] (the kernel's weight [rows, taps*cin] viewed); H / W are
    zero padded by kh // 2, kw // 2.  ``sub2``: ZeroPad2d((0,1,0,1)) then the stride-2 conv (vae.py:84-92), output
    H // 2 x W // 2.  m is the same conv of |x| and |w|, and E = c_acc m + 2^-22 (|z| + |b|)."""
    kt, kh, kw = taps
    rows = w5.shape[0]
    T = x.shape[0] - kt + 1 if T is None else T
    wd = w5.double().reshape(rows, kt, kh, kw, -1).permute(0, 4, 1, 2, 3)
    zs, ms = [], []
    for t0 in range(0, T, frames_per_chunk):
        t1 = min(T, t0 + frames_per_chunk)
        xd = x[t0:t1 + kt - 1].double().permute(3, 0, 1, 2)[None]
        if sub2:
            assert (kh, kw) == (3, 3)
            pad, stride = (0, 1, 0, 1, 0, 0), (1, 2, 2)
        else:
            pad, stride = (kw // 2, kw // 2, kh // 2, kh // 2, 0, 0), 1
        zs.append(F.conv3d(F.pad(xd, pad), wd, stride=stride)[0].permute(1, 2, 3, 0))
        ms.append(F.conv3d(F.pad(xd.abs(), pad), wd.abs(), stride=stride)[0].permute(1, 2, 3, 0))
        del xd
    z, m = torch.cat(zs), torch.cat(ms)
    babs = 0.0
    if bias is not None:
        z = z + bias[:rows].double()
        babs = bias[:rows].double().abs()
    return z, m, c_acc * m + F32_EPI * (z.abs() + babs)


def check_conv(form, got, z, m, E, dtype, *, y16=None, residual=None, gamma=None, cout=None):
    """Hold one conv output to the float64 reference.  Returns (violations, stats) as :func:`check_gemm`.

    raw:  r16(acc + b) inside [r16(z - E), r16(z + E)] (stats["ratio"]: :func:`acc_ratio`).
    res:  r16(res + r16(acc + b)): inside the interval carried through the add, and equal to r16(res + y16) exactly,
          y16 the raw-only output of the same kernel on the same operands.
    norm: SiLU(RMS_norm(raw) * sqrt(cout) * gamma) on the kernel's own raw values ``y16`` (the raw, or raw + residual,
          output of the same launch form): channels < cout within 1 ulp of :func:`vae_rmsnorm_silu` but for
          NORM_FAR_FRAC of them (<= NORM_FAR_ULPS), not bit-identical on at most NORM_MAX_FRAC; channels >= cout (zero
          weight rows) exactly 0.
    head: clamp(r16(acc + b), -1, 1) as fp32, ``got`` [T, Ho, Wo, cout] (the NCHW output permuted), z of the first
          cout channels."""
    viol = []
    if form == "raw":
        return check_gemm(EPI_BIAS, got, z, m, E, dtype)
    if form == "res":
        return check_gemm(EPI_BIAS_RES, got, z, m, E, dtype, residual=residual, y16=y16)
    g = got.double()
    if not bool(torch.isfinite(g).all()):
        viol.append("non-finite output")
        g = torch.nan_to_num(g, nan=1e300)
    if form == "head":
        c = g.shape[-1]
        lo = r16(z[..., :c] - E[..., :c], dtype).clamp(-1, 1)
        hi = r16(z[..., :c] + E[..., :c], dtype).clamp(-1, 1)
        ex = _outside(g, lo, hi, ulp(g, dtype))
        if ex > 0:
            viol.append(f"head: {ex:.3g} ulps outside the clamped accumulation interval")
        nearest = r16(z[..., :c], dtype).clamp(-1, 1)
        inner = (g > -1) & (g < 1)
        ratio = acc_ratio(torch.where(inner, g, r16(z[..., :c], dtype)), z[..., :c], m[..., :c], dtype)
        return viol, {"excess": ex, "frac": float((g != nearest).double().mean()), "ratio": ratio}
    if form == "norm":
        cout = g.shape[-1] if cout is None else cout
        want, _ = vae_rmsnorm_silu(y16[..., :cout], gamma[:cout], dtype)
        du = (g[..., :cout] - want).abs() / ulp(want, dtype)
        worst = float(du.max())
        frac, far = float((du != 0).double().mean()), float((du > 1).double().mean())
        if worst > NORM_FAR_ULPS or far > NORM_FAR_FRAC or frac > NORM_MAX_FRAC:
            viol.append(f"norm: {worst:.3g} ulps from the restatement on the kernel's raw values, "
                        f"{far:.3g} more than 1 ulp away, {frac:.3g} not bit-identical")
        if g.shape[-1] > cout and bool((g[..., cout:] != 0).any()):
            viol.append("norm: a channel >= cout is not 0")
        return viol, {"excess": max(0.0, worst - NORM_FAR_ULPS), "frac": frac, "far": far, "worst_ulps": worst}
    raise ValueError(form)


def guarded_frames(T, H, W, C, dtype, device, fill=None, before=1, after=1):
    """A [T, H, W, C] channels-last view (pixel pitch C + GUARD_COLS, dense rows) inside a sentinel-filled
    [before + T + after, H, W, C + GUARD_COLS] buffer.  fp32 buffers are [before + T + after, C, H, W] NCHW pixel
    stacks (``out_pix``): no pitch, a guard frame before and after."""
    if dtype == torch.float32:
        buf = torch.empty(before + T + after, C, H, W, dtype=dtype, device=device)
        buf.view(torch.int32).fill_(SENTINEL32)
        view = buf[before:before + T]
    else:
        buf = torch.empty(before + T + after, H, W, C + GUARD_COLS, dtype=dtype, device=device)
        buf.view(torch.int16).fill_(SENTINEL16)
        view = buf[before:before + T, :, :, :C]
    if fill is not None:
        view.copy_(fill)
    return buf, view


def frames_intact(buf, T, C, before=1, untouched=()) -> bool:
    """True when every element of a :func:`guarded_frames` buffer outside its view still holds the sentinel, and so does
    every frame of the view listed in ``untouched`` (the other half of an interleaved output)."""
    if buf.dtype == torch.float32:
        bits, s = buf.view(torch.int32), SENTINEL32
    else:
        bits, s = buf.view(torch.int16), SENTINEL16
    keep = torch.ones(bits.shape, dtype=torch.bool, device=buf.device)
    if buf.dtype == torch.float32:
        keep[before:before + T] = False
    else:
        keep[before:before + T, :, :, :C] = False
    for f in untouched:
        keep[before + f] = True
    return bool((bits[keep] == s).all())
