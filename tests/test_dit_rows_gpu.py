"""Per-kernel GPU parity of the DiT row kernels of ``kr_dit_elem.cu`` against the float64 restatements of
``tests/kernel_refs.py`` (built from ``oracle/dit_oracle.py``, computed on the device).

Two checks per kernel, both per element:

(a) against the restatement rounded to bf16 at the kernel's documented rounding points.  The kernel does the same
    arithmetic in fp32, so it can only land on the other side of a bf16 rounding boundary: per element the difference
    is <= 1 ulp of the result, plus 2^-7 |t| for each earlier rounding point t whose one-ulp flip is carried to the
    output, plus 2^-16 of the normalised row's scale (the fp32 evaluation error, which shows where a result cancels
    to nearly 0).  The fraction of elements that are not bit-identical is bounded by FRAC = 1e-4 (measured on an
    H100: <= 3.1e-5 for ln_modulate, <= 2.9e-5 for qkv_norm_rope, <= 1.3e-6 for rmsnorm).
(b) against the float64 value with no rounding at all: each of the k rounding points adds at most half an ulp,
    2^-8 |value|, of its own value, which bounds the whole chain (stated per kernel below).

Pure data movement (V append, patchify, unpatchify, the modulation add of two bf16 values whose fp32 sum is exact)
is compared with ``torch.equal``.  Guard rows and columns around every strided output must keep their sentinel."""
import pytest
import torch

from tests import kernel_refs as R

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
H8 = 2.0 ** -8                 # half a bf16 ulp, relative
FRAC = 1e-4                    # bound on the fraction of elements that are not bit-identical
SENT = -12345.0                # sentinel of guard regions (exactly representable in bf16)


def _ops():
    from realtime_video_b200 import ops
    return ops


def _guarded(rows, cols, pad_r=2, pad_c=16):
    """A sentinel-filled buffer and the [rows, cols] window inside it (row pitch cols + 2*pad_c)."""
    buf = torch.full((rows + 2 * pad_r, cols + 2 * pad_c), SENT, dtype=BF, device="cuda")
    return buf, buf[pad_r:pad_r + rows, pad_c:pad_c + cols]


def _outside_untouched(buf, view_rows, view_cols):
    m = torch.ones_like(buf, dtype=torch.bool)
    m[view_rows, view_cols] = False
    return bool((buf[m] == SENT).all())


def _check_a(got, ref, t=None, scale=1.0, frac_max=FRAC):
    """(a): |got - ref| <= ulp(ref) + 2^-7 |t| + 2^-16 scale, and at most frac_max of the elements differ at all.
    ``t`` is the magnitude, carried to the output, of an earlier rounding point (a one-ulp flip there moves the result
    by up to 2^-7 |t|); ``scale`` the size of the normalised row, whose fp32 evaluation error (far below 2^-16 of it)
    dominates where the result cancels to nearly 0."""
    g, r = got.double(), ref.double()
    d = (g - r).abs()
    tol = R.ulp(r) + 2.0 ** -16 * scale
    if t is not None:
        tol = tol + 2.0 ** -7 * t.abs()
    worst = float((d / tol).max())
    frac = float((d != 0).double().mean())
    assert worst <= 1.0 and frac <= frac_max, (worst, frac)
    return worst, frac


# ---------------------------------------------------------------------------------------------
# ln_modulate
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [256, 1000, 1536, 5120, 6144, 8192])
@pytest.mark.parametrize("variant", ["plain", "affine", "mod"])
def test_ln_modulate(D, variant):
    """LayerNorm (+affine) (+ per-frame modulation) at every kVec instantiation: D 256 / 1000 (idle threads) take
    kVec 1, 1536 kVec 2, 5120 kVec 5, 6144 and 8192 the kVec-8 branch (6 and 8 of its slots).  x and out have row
    pitches larger than D.  Rounding chain (b): y = r16(LN), then r16(1 + scale), r16(y * .), r16(. + shift), so
    |out - exact| <= 2^-8 (3 |y (1 + scale)| + |out|) (plain / affine: 2^-8 |y|), plus the fp32 LN error (< 2^-16
    of the bound here).  Measured on an H100: (b) <= 0.994 of the bound."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D + len(variant))
    fs, Fr = 1560, 3
    L = fs * Fr
    xb, x = _guarded(L, D)
    x.copy_((torch.randn(L, D, device="cuda", generator=g) * 2 + 0.5).to(BF))
    ob, out = _guarded(L, D, pad_c=24)
    kw, args = {}, {}
    if variant == "affine":
        kw = dict(weight=(1 + 0.3 * torch.randn(D, device="cuda", generator=g)).to(BF),
                  bias=(0.2 * torch.randn(D, device="cuda", generator=g)).to(BF))
        args = dict(weight=kw["weight"], bias=kw["bias"])
    elif variant == "mod":
        mod = (0.5 * torch.randn(Fr, 6, D, device="cuda", generator=g)).to(BF)
        kw = dict(mod=mod, shift_idx=3, scale_idx=4, rows_per_frame=fs)
        args = kw
    ops.ln_modulate(x, eps=1e-6, out=out, **kw)
    ref, exact, prod = R.ln_modulate(x, 1e-6, **args)
    worst, frac = _check_a(out, ref, 2 * prod if variant == "mod" else None, 1 + exact.abs())
    bound = H8 * (3 * prod.abs() + ref.abs()) if variant == "mod" else \
        H8 * torch.maximum(ref.abs(), exact.abs()) * (1 + 2 ** -10)
    ratio = float(((out.double() - exact).abs() / (bound + 2.0 ** -16)).max())
    assert ratio <= 1.0, ratio
    assert _outside_untouched(ob, slice(2, 2 + L), slice(24, 24 + D))
    assert bool((xb[:2] == SENT).all())
    print(f"ln_modulate D={D} {variant}: (a) {worst:.2f} of the bound, {frac:.2e} not identical, chain {ratio:.3f}")


def test_ln_modulate_per_frame_rows():
    """Every row takes the modulation of its own frame: with a modulation that is constant within a frame and differs
    between frames, the rows on both sides of each frame boundary (1559 | 1560, 3119 | 3120) match the reference."""
    ops = _ops()
    D, fs = 512, 1560
    x = torch.randn(3 * fs, D, device="cuda").to(BF)
    mod = torch.zeros(3, 6, D, device="cuda")
    mod[:, 1] = torch.tensor([0.0, 1.0, -0.5], device="cuda")[:, None]
    mod[:, 0] = torch.tensor([0.0, 3.0, -2.0], device="cuda")[:, None]
    mod = mod.to(BF)
    out = ops.ln_modulate(x, eps=1e-6, mod=mod, shift_idx=0, scale_idx=1, rows_per_frame=fs)
    ref, _, prod = R.ln_modulate(x, 1e-6, mod=mod, shift_idx=0, scale_idx=1, rows_per_frame=fs)
    for r in (fs - 1, fs, 2 * fs - 1, 2 * fs):
        _check_a(out[r], ref[r], 2 * prod[r], frac_max=0.05)


@pytest.mark.parametrize("D", [8200, 1004])
def test_ln_modulate_rejects_unsupported_widths(D):
    from realtime_video_b200._lib import KreaB200Error
    ops = _ops()
    x = torch.zeros(4, D, device="cuda", dtype=BF)
    with pytest.raises(KreaB200Error):
        ops.ln_modulate(x, eps=1e-6)


# ---------------------------------------------------------------------------------------------
# qkv_norm_rope
# ---------------------------------------------------------------------------------------------
def _qkv_inputs(L, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = (torch.randn(L, 3 * D, device="cuda", generator=g) * 1.5).to(BF)       # the fused to_qkv output
    wq = (1 + 0.3 * torch.randn(D, device="cuda", generator=g)).to(BF)
    wk = (1 + 0.3 * torch.randn(D, device="cuda", generator=g)).to(BF)
    return qkv, wq, wk


def _pair(x):
    """|(x_2i, x_2i+1)| of the rotated pair each element belongs to."""
    e = x.view(x.shape[0], -1, 2)
    return e.norm(dim=-1, keepdim=True).expand_as(e).reshape(x.shape)


def _rope_chain_ratio(got, exact, head_dim):
    """(b) for q / k: the two rounding points before the rotation move a pair by <= 2 * 2^-8 * sqrt(2) |pair| and
    the final rounding by 2^-8 |out|: |got - exact| <= 2^-8 (3 |pair| + |out|)."""
    e = exact.view(exact.shape[0], -1, 2)
    pair = e.norm(dim=-1, keepdim=True).expand_as(e).reshape(exact.shape)
    bound = H8 * (3 * pair + exact.abs()) + 2.0 ** -16 * pair
    return float(((got.double() - exact).abs() / (bound + 1e-30)).max())


@pytest.mark.parametrize("D,gh,gw,frames,start_frame", [
    (1024, 60, 104, 2, 0), (1024, 60, 104, 2, 3), (1024, 60, 104, 2, 7),
    (1536, 24, 40, 3, 0),                     # the 1.3B width (kVec 2)
    (5120, 30, 52, 3, 0),                     # the 14B width at the bench token grid (kVec 5)
    (6144, 12, 20, 2, 1),                     # the kVec-8 branch
])
def test_qkv_norm_rope(D, gh, gw, frames, start_frame):
    """RMSNorm + 3-axis RoPE of q and k, K written into rows [ls, le) of a wider cache view, V copied into its slot.
    q / K: (a) <= 1 ulp, (b) <= the rope rounding chain; V bit-exact; every cache row and column outside the slot
    keeps its sentinel.  The reference built on the exchanged grid (grid_w x grid_h) is far from the kernel's
    output, so the check tells the h and w sub-bands apart.  Measured on an H100: (a) <= 0.93, (b) <= 0.73 of
    their bounds."""
    ops = _ops()
    hd = 128
    L = frames * gh * gw
    qkv, wq, wk = _qkv_inputs(L, D, D + start_frame)
    q, k, v = qkv[:, :D], qkv[:, D:2 * D], qkv[:, 2 * D:]
    rope = R.rope_table_f32(hd, "cuda")
    ls = 333
    kb, _ = _guarded(L + 2 * ls, D, pad_r=0)
    vb, _ = _guarded(L + 2 * ls, D, pad_r=0)
    k_slot, v_slot = kb[ls:ls + L, 16:16 + D], vb[ls:ls + L, 16:16 + D]
    rq = torch.empty(L, D, dtype=BF, device="cuda")
    ops.qkv_norm_rope(q, k, v, wq, wk, rq, k_slot, v_slot, rope, head_dim=hd, grid_h=gh, grid_w=gw,
                      start_frame=start_frame, eps=1e-6)
    for got, x, w in ((rq, q, wq), (k_slot, k, wk)):
        ref, exact = R.qk_norm_rope(x, w, 1e-6, hd, gh, gw, start_frame)
        worst, frac = _check_a(got, ref, _pair(exact), _pair(exact))
        ratio = _rope_chain_ratio(got, exact, hd)
        assert ratio <= 1.0, ratio
        print(f"qkv_norm_rope D={D} grid {gh}x{gw} sf={start_frame}: (a) {worst:.2f} of the bound, "
              f"{frac:.2e} not identical, "
              f"chain {ratio:.3f}")
    assert torch.equal(v_slot, v)
    for buf in (kb, vb):
        assert _outside_untouched(buf, slice(ls, ls + L), slice(16, 16 + D))
    # the h / w sub-bands are distinguishable: the exchanged grid's reference misses by many ulps
    swapped, _ = R.qk_norm_rope(q, wq, 1e-6, hd, gw, gh, start_frame)
    assert float(((rq.double() - swapped).abs() / R.ulp(swapped)).max()) > 8


def test_qkv_norm_rope_without_v():
    """v = None (the fused QKV GEMM already wrote V into the cache): q and K as usual, the V slot is not written."""
    ops = _ops()
    D, gh, gw = 1536, 24, 40
    L = gh * gw
    qkv, wq, wk = _qkv_inputs(L, D, 11)
    rope = R.rope_table_f32(128, "cuda")
    rq = torch.empty(L, D, dtype=BF, device="cuda")
    rk = torch.full((L, D), SENT, dtype=BF, device="cuda")
    ops.qkv_norm_rope(qkv[:, :D], qkv[:, D:2 * D], None, wq, wk, rq, rk, None, rope, head_dim=128, grid_h=gh,
                      grid_w=gw, start_frame=2, eps=1e-6)
    for got, x, w in ((rq, qkv[:, :D], wq), (rk, qkv[:, D:2 * D], wk)):
        ref, exact = R.qk_norm_rope(x, w, 1e-6, 128, gh, gw, 2)
        _check_a(got, ref, _pair(exact), _pair(exact))


# ---------------------------------------------------------------------------------------------
# rmsnorm / add_modulation / activation
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [512, 4680])
@pytest.mark.parametrize("inplace", [False, True])
def test_rmsnorm(rows, inplace):
    """out = r16(r16(x * rsqrt(mean x^2 + eps)) * w) at D 5120, out of place and in place (``out=x``, as the
    cross-attention normalises q and k).  (b): two rounding points, |out - exact| <= 2^-8 (|x r w| + |out|).
    Measured on an H100: (a) <= 0.88, (b) <= 0.99 of their bounds."""
    ops = _ops()
    D = 5120
    g = torch.Generator(device="cuda").manual_seed(rows)
    x = (torch.randn(rows, D, device="cuda", generator=g) * 3).to(BF)
    w = (1 + 0.3 * torch.randn(D, device="cuda", generator=g)).to(BF)
    x0 = x.clone()
    out = ops.rmsnorm(x, w, 1e-6, out=x if inplace else None)
    if inplace:
        assert out.data_ptr() == x.data_ptr()
    ref = R.rmsnorm(x0, w, 1e-6)
    xd = x0.double()
    exact = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + 1e-6) * w.double()
    worst, frac = _check_a(out, ref, exact, exact.abs())
    ratio = float(((out.double() - exact).abs() / (H8 * (exact.abs() + out.double().abs()) + 1e-30)).max())
    assert ratio <= 1.0, ratio
    print(f"rmsnorm rows={rows} inplace={inplace}: (a) {worst:.2f} of the bound, {frac:.2e} not identical, "
          f"chain {ratio:.3f}")


@pytest.mark.parametrize("F", [1, 3, 7])
def test_add_modulation(F):
    """e[f] = bf16(modulation + e0[f]) with an e0 frame stride of 6*D + 64 elements: bit-exact (the fp32 sum of two
    bf16 values rounds to bf16 exactly as their float64 sum does)."""
    ops = _ops()
    D = 5120
    mod = torch.randn(1, 6, D, device="cuda").to(BF)
    e0b = torch.full((F, 6 * D + 64), SENT, dtype=BF, device="cuda")
    e0 = e0b[:, :6 * D].view(F, 6, D)
    e0.copy_((torch.randn(F, 6, D, device="cuda") * 4).to(BF))
    assert F == 1 or e0.stride(0) == 6 * D + 64
    out = ops.add_modulation(mod, e0)
    assert torch.equal(out.double(), R.r16(mod.double() + e0.double()))


@pytest.mark.parametrize("kind", ["silu", "gelu"])
def test_activation(kind):
    """SiLU and tanh-GELU over [-100, 100], random values and +-0.  SiLU: <= 1 ulp of the float64 value.  GELU is
    0.5 x (1 + tanh(.)) in fp32 like torch's own bf16 kernel; for x << 0, 1 + tanh cancels and carries the fp32
    error of tanh (<= 2^-23), so the bound is 1 ulp + 2^-23 |x|.  Below x = -88.7 exp(-x) overflows fp32 and both
    formulas return -0 (as torch's kernels do) where the true value is below 1e-36: an absolute 1e-36 is allowed."""
    from realtime_video_b200._lib import KreaB200Error
    ops = _ops()
    x = torch.cat([torch.linspace(-100, 100, 200001, device="cuda"), torch.randn(65535, device="cuda") * 4,
                   torch.tensor([0.0, -0.0], device="cuda")]).to(BF)
    x = x[:x.numel() // 8 * 8]
    x[-2:] = torch.tensor([0.0, -0.0])
    y = ops.activation(x, kind)
    ref = R.r16(R.silu(x) if kind == "silu" else R.gelu_tanh(x))
    d = (y.double() - ref).abs()
    tol = R.ulp(ref) + 1e-36 + (0.0 if kind == "silu" else 2.0 ** -23 * x.double().abs())
    assert bool((d <= tol).all()), float((d / tol).max())
    assert float(y[-2]) == 0.0 and float(y[-1]) == 0.0
    with pytest.raises(KreaB200Error):
        ops.activation(torch.zeros(12, device="cuda", dtype=BF), kind)


# ---------------------------------------------------------------------------------------------
# patchify / unpatchify_x0
# ---------------------------------------------------------------------------------------------
def test_patchify_strided_input():
    """x [C, F, H, W] given as a permuted, non-contiguous view: bit-exact against the Conv3d(1,2,2) im2col."""
    ops = _ops()
    C, Fr, H, W = 16, 3, 60, 104
    base = torch.randn(Fr, H, C, W, device="cuda").to(BF)
    x = base.permute(2, 0, 1, 3)
    assert not x.is_contiguous()
    assert torch.equal(ops.patchify(x), R.patchify(x))


def test_unpatchify_x0_per_frame_sigma():
    """head_out with a row pitch of 4C + 16, three frames with three different sigmas: flow bit-exact against the
    reshape/permute of causal_model.py:1145-1147, x0 bit-exact against bf16(double(xt) - sigma[f] double(flow))."""
    ops = _ops()
    C, Fr, H, W = 16, 3, 60, 104
    L = Fr * (H // 2) * (W // 2)
    hb = torch.randn(L, 4 * C + 16, device="cuda").to(BF)
    head = hb[:, :4 * C]
    xt = torch.randn(Fr, C, H, W, device="cuda").to(BF)
    sigma = torch.tensor([0.9375, 0.5, 0.0625], dtype=torch.float64, device="cuda")
    flow, x0 = ops.unpatchify_x0(head, xt, sigma, C, Fr, H, W)
    want = R.unpatchify(head, C, Fr, H, W)
    assert torch.equal(flow, want)
    assert torch.equal(x0, R.flow_to_x0(want, xt, sigma))
