"""The attention restatements of ``tests/kernel_refs.py`` (``attn_interval`` / ``t5_attn_interval`` / ``check_attn``)
proven on the CPU with the GPU file's own per-case checks (``tests/test_attn_parity_gpu.flash_check`` / ``t5_check``):
an fp32 emulation of each kernel's schedule (128-key tiles, attn_fwd_kernel's lazy rescale, the per-thread partial l
over the kernel's column pattern, P rounded to nearest, the epilogue with the padded keys) passes on a CPU-sized subset
of the case table in both 16-bit types, and each of twelve plausible kernel bugs is rejected by the case named beside
it.

Every bug of the list is caught, in both dtypes.  The subtlest is deciding the lazy rescale in raw-score units instead
of log2 units: the softmax it computes is the same, only the points where O is rescaled move, and with it the m_used
that P is rounded against; the restatement's intervals are narrow enough that this moves elements out of them."""
import math

import pytest
import torch

from tests import kernel_refs as R
from tests import test_attn_parity_gpu as G

BF, FP = torch.bfloat16, torch.float16
DTYPES = [BF, FP]
NEG_INF = float("-inf")


def _f32(x):
    return torch.as_tensor(x, dtype=torch.float32)


def _mm32(a, b):
    """An fp32 product as a tensor-core tile computes it: to within a few fp32 roundings of the exact sum (here the
    exact sum rounded once; torch's CPU sgemm is several times less accurate than the H100's wgmma)."""
    return (a.double() @ b.double()).float()


def _ex2(x):
    """ex2.approx.ftz.f32 (to within EXP2_REL): results below 2^-126 flushed to 0."""
    p = torch.exp2(x)
    return torch.where(p < R.TINY32, torch.zeros_like(p), p)


def _round16(x, dtype, truncate=False):
    if not truncate:
        return x.to(dtype).float()
    y = x.to(dtype).float()
    return torch.where(y.abs() > x.abs(), R._bits_neighbour(y.double(), y < 0, dtype).float(), y)


def _l_partials(l_run, p):
    """Add a tile's p [rows, 128] into the per-thread partial sums l_run [rows, 4] as the kernel does: thread t of a
    quad owns columns 8 nb + 2 t + e and adds a0 + a1 per nb in order."""
    pr = p.view(p.shape[0], 16, 4, 2)
    for nb in range(16):
        l_run = l_run + (pr[:, nb, :, 0] + pr[:, nb, :, 1])
    return l_run


def _l_total(l_run):
    return (l_run[:, 0] + l_run[:, 1]) + (l_run[:, 2] + l_run[:, 3])


def emulate_flash(case, q, k, v, dtype, mutate=None):
    """What attn_fwd_kernel computes, in fp32 on the CPU; ``mutate`` names a deliberate bug."""
    Lq, Lkv, heads = case["Lq"], case["Lkv"], case["heads"]
    sl2 = _f32(R.attn_scale_log2(case["scale"]))
    row_lo, row_hi, n_ph = R.attn_rows(Lq, Lkv, case["block_len"], case["window"], case["pad"])
    if mutate == "drop_last_key":
        row_hi = row_hi - 1
    if mutate == "window_one_too_many":
        row_lo = torch.where(row_lo > 0, row_lo - 1, row_lo)
    if mutate == "phantom_off_by_one":
        n_ph = torch.where(n_ph > 0, n_ph + 1, n_ph)
    if mutate == "keys_past_lkv_scored_0" and not case["block_len"]:
        row_hi = torch.full_like(row_hi, (Lkv + 127) // 128 * 128)
    out = torch.empty(Lq, heads * 128, dtype=dtype)
    for h in range(heads):
        cs = slice(h * 128, (h + 1) * 128)
        qh = q[:, cs].float()
        if mutate == "wg1_reads_wg0_rows":
            r = torch.arange(Lq)
            src = torch.where(r % 128 >= 64, r - 64, r)
            qh = qh[src]
        kh, vh = k[:, cs].float(), v[:, cs].float()
        n_keys = (Lkv + 127) // 128 * 128
        kh = torch.cat([kh, kh.new_zeros(n_keys - Lkv, 128)])     # TMA zero fill past Lkv
        vh = torch.cat([vh, vh.new_zeros(n_keys - Lkv, 128)])
        m_run = torch.full((Lq,), NEG_INF)
        l_run = torch.zeros(Lq, 4)
        O = torch.zeros(Lq, 128)
        for j in range(n_keys // 128):
            c = torch.arange(j * 128, j * 128 + 128)
            s = _mm32(qh, kh[c].t())
            s = torch.where((c[None] >= row_hi[:, None]) | (c[None] < row_lo[:, None]), NEG_INF, s)
            m_new = torch.maximum(m_run, s.amax(1))
            diff = (m_new - m_run) if mutate == "threshold_raw_units" else (m_new - m_run) * sl2
            need = diff > 8.0
            m_used = torch.where(need, m_new, m_run)
            alpha = torch.where(need, _ex2((m_run - m_new) * sl2), torch.ones(()))
            if j > 0:
                O = torch.where(need[:, None], O * alpha[:, None], O)
            if mutate != "l_not_rescaled":
                l_run = l_run * alpha[:, None]
            m_run = m_used
            nms = torch.where(m_used == NEG_INF, torch.zeros(()), -m_used * sl2)
            arg = (s.double() * sl2.double() + nms.double()[:, None]).float()      # fmaf: one rounding
            p = _ex2(arg)
            l_run = _l_partials(l_run, p)
            P = _round16(p, dtype, truncate=mutate == "p_truncated")
            O = O + _mm32(P, vh[c])
        l = _l_total(l_run)
        o_scale = torch.ones(Lq)
        m_fin = torch.maximum(m_run, torch.zeros(()))
        ph = n_ph > 0
        o_scale = torch.where(ph, _ex2((m_run - m_fin) * sl2), o_scale)
        l = torch.where(ph, l * o_scale + n_ph.float() * _ex2(-m_fin * sl2), l)
        out[:, cs] = (O * (o_scale / l)[:, None]).to(dtype)
    return out


def emulate_t5(case, q, k, v, bias, km, mutate=None):
    """What t5_attn_kernel computes (p = ex2(fl(v - m) log2e)), in fp32 on the CPU."""
    L, heads = case["L"], case["heads"]
    l2e = _f32(R.LOG2E_F32)
    kmin = _f32(R.T5_MIN)
    idx = torch.arange(L)
    off = idx[None, :] - idx[:, None] + (L - 1)
    if mutate == "bias_offset_off_by_one":
        off = (off + 1).clamp_max(2 * L - 2)
    mask = torch.ones(L, dtype=torch.bool) if km is None else km != 0
    out = torch.empty(L, heads * 64, dtype=BF)
    for h in range(heads):
        cs = slice(h * 64, (h + 1) * 64)
        s = _mm32(q[:, cs], k[:, cs].t())
        b = bias[h].float()[off]
        val = (s + b).bfloat16().float() if mutate == "bias_before_round" else (s.bfloat16().float() + b).bfloat16().float()
        val = torch.where(mask[None], val, kmin)
        vh = v[:, cs].float()
        m_run = torch.full((L,), NEG_INF)
        l_run = torch.zeros(L, 4)
        O = torch.zeros(L, 64)
        for k0 in range(0, L, 128):
            x = val[:, k0:k0 + 128]
            n = x.shape[1]
            m_new = torch.maximum(m_run, x.amax(1))
            alpha = _ex2((m_run - m_new) * l2e)
            O, l_run, m_run = O * alpha[:, None], l_run * alpha[:, None], m_new
            p = _ex2((x - m_new[:, None]) * l2e)
            p = torch.cat([p, p.new_zeros(L, 128 - n)], 1)
            l_run = _l_partials(l_run, p)
            P = p.bfloat16().float()
            O = O + _mm32(P[:, :n], vh[k0:k0 + n])
        l = _l_total(l_run)
        if mutate == "p_normalised":    # the reference's order: softmax normalised in fp32, then rounded, then P V
            pn = torch.softmax(val, dim=-1).bfloat16().float()
            out[:, cs] = _mm32(pn, vh).bfloat16()
        else:
            out[:, cs] = (O * (1.0 / l)[:, None]).bfloat16()
    return out


# ---------------------------------------------------------------------------------------------
# the CPU-sized subset of the GPU case table
# ---------------------------------------------------------------------------------------------
CPU_FLASH = ["1x1", "63x129", "64x512", "65x1300", "127x127", "128x128", "129x1300", "block end in a tile",
             "block end on a tile boundary", "window edge in a tile", "phantom negative", "phantom only rows",
             "jump at tile edge", "jump inside tile", "jump under 8", "jump masked", "spread +-100", "spread masked",
             "scale 0.25", "scale dit"]
CPU_T5 = [dict(L=1, heads=1, mask="none"), dict(L=2, heads=4, mask="prefix1"), dict(L=129, heads=1, mask="first128"),
          dict(L=200, heads=4, mask="random"), dict(L=200, heads=1, mask="all"), dict(L=200, heads=1, mask="prefix37"),
          dict(L=512, heads=4, mask="prefix129"), dict(L=777, heads=1, mask="first128")]


def _flash_case(name):
    return next(c for c in G.FLASH_CASES if c["name"] == name)


def run_flash(name, dtype, mutate=None):
    case = _flash_case(name)
    q, k, v = G.flash_inputs(case, dtype, "cpu")
    got = emulate_flash(case, q, k, v, dtype, mutate)
    if mutate == "one_ulp":
        lo, hi, _ = R.attn_interval(q, k, v, case["heads"], case["block_len"], case["window"], case["pad"],
                                    case["scale"], dtype)
        got[5 % case["Lq"], 7] = R._bits_neighbour(hi[5 % case["Lq"], 7].view(1), torch.tensor([True]), dtype)[0]
    return G.flash_check(case, dtype, got, q, k, v)


def run_t5(case, mutate=None):
    q, k, v, bias, km = G.t5_inputs(case, "cpu")
    got = emulate_t5(case, q, k, v, bias, km, mutate)
    if mutate == "one_ulp":
        lo, hi, _ = R.t5_attn_interval(q, k, v, bias, km, case["heads"])
        got[3 % case["L"], 5] = R._bits_neighbour(lo[3 % case["L"], 5].view(1), torch.tensor([False]), BF)[0]
    return G.t5_check(case, got, q, k, v, bias, km)


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("name", CPU_FLASH)
def test_flash_restatement_accepts_the_emulated_kernel(name, dtype):
    viol, stats = run_flash(name, dtype)
    assert not viol, (name, viol, stats)
    assert stats["ratio"] <= 1


@pytest.mark.parametrize("case", CPU_T5, ids=G._cid)
def test_t5_restatement_accepts_the_emulated_kernel(case):
    viol, stats = run_t5(case)
    assert not viol, (viol, stats)


# each bug and the case that catches it
FLASH_BUGS = [(m, n, dt) for m, n in [
    ("drop_last_key", "129x1300"),
    ("drop_last_key", "block end in a tile"),
    ("window_one_too_many", "window edge in a tile"),
    ("phantom_off_by_one", "phantom negative"),
    ("keys_past_lkv_scored_0", "65x1300"),
    ("p_truncated", "128x128"),
    ("l_not_rescaled", "jump at tile edge"),
    ("threshold_raw_units", "jump under 8"),
    ("wg1_reads_wg0_rows", "129x1300"),
    ("one_ulp", "64x512"),
] for dt in ("bf16", "fp16")]


@pytest.mark.parametrize("mutate,name,dtype", FLASH_BUGS)
def test_flash_checks_reject_each_kernel_bug(mutate, name, dtype):
    viol, stats = run_flash(name, {"bf16": BF, "fp16": FP}[dtype], mutate)
    assert viol, (mutate, name, stats)


T5_BUGS = [
    ("bias_offset_off_by_one", dict(L=200, heads=4, mask="random")),
    ("bias_before_round", dict(L=200, heads=1, mask="prefix37")),
    ("p_normalised", dict(L=200, heads=4, mask="random")),
    ("one_ulp", dict(L=129, heads=1, mask="first128")),
]


@pytest.mark.parametrize("mutate,case", T5_BUGS, ids=[m for m, _ in T5_BUGS])
def test_t5_checks_reject_each_kernel_bug(mutate, case):
    viol, stats = run_t5(case, mutate)
    assert viol, (mutate, stats)


def test_interval_helpers():
    lo, hi, n = R.attn_rows(250, 250, 84, 2, 6)
    assert (hi[168:] - lo[168:]).max() <= 0 and n[168:].tolist() == [2] * 82      # only phantom keys
    assert lo[:84].tolist() == [82] * 84 and hi[:84].tolist() == [84] * 84
    lo, hi, n = R.attn_rows(1200, 1200, 240, 480, 80)
    assert sorted(set(lo.tolist())) == [0, 240, 480, 720] and int(n.max()) == 0
    assert R.attn_scale_log2() == R.f32(R.f32(1 / math.sqrt(128)) * R.LOG2E_F32)
    p_lo, p_hi = R._exp2_bounds(torch.tensor([-127.0, 0.0]).double(), torch.tensor([-127.0, 0.0]).double(), 0.0)
    assert p_lo.tolist() == [0.0, 1.0] and p_hi.tolist() == [2.0 ** -127, 1.0]
