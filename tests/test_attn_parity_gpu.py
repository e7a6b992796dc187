"""Element-wise float64 parity of both 16-bit attention kernels against restatements of their online-softmax schedules
(``tests/kernel_refs.attn_interval`` for kr_attn_fwd, ``t5_attn_interval`` for kr_t5_attn): every output element must
lie inside its restated interval, with zero slack.

kr_attn_fwd, bf16 and fp16: Lq 1..129 around the 64-row warpgroup halves and the 128-row tile, 4680 (19 q-tiles, a
tail inside the second consumer warpgroup); Lkv 1..129 around the 128-key tile, 512 (text length), 1300 and 9360
(the 4-stage K / V ring wraps more than once); heads 1-3 and the production 40 heads at 4680 x 9360 (heads 0, 13, 26
and 39 restated); block-causal masks with block ends inside a tile and on a tile boundary, window lower edges inside a
tile and skipping whole tiles (the m = -inf path), padded ("phantom") keys carrying a large share of negative-score rows
and rows that see only phantom keys; score jumps of more than 8 (log2 units) at a tile boundary and inside a tile and
just under 8 (P near 2^8); scores spread over +-100 (ftz zeros, fp16-subnormal P); softmax_scale at its default,
0.25 and the fp32-rounded 1 / sqrt(128) of kr_dit_block.cu; Q with a row pitch, K / V as cache views at a row offset.
kr_t5_attn: L 1..1024, heads 1, 4 and 64, a bias distinct per offset up to +-30, no mask, prefix masks of 1, 37, 127,
128, 129 and L - 1 keys, a random mask, the first 128 keys masked and every key masked; L 1025 is refused.

Every output sits inside a sentinel-filled buffer (pitch > heads * D, rows above and below) that must be unchanged,
and a second launch must give the same bits.  Each kernel and dtype prints one summary line: cases, the largest
share of an interval's half-width an element needed (``ratio``), the fraction of elements whose interval holds two
16-bit values (``span``), the fraction not equal to r16 of the interval midpoint (``frac``) and the number of
ambiguous lazy-rescale decisions.

The constants of the restatement are C_S (scores), C_PV (P V) and EXP2_REL (ex2.approx); ``test_constants_margin``
shrinks each in turn, with the others at their values, on the widest cases and requires a margin of at least 4x.
On an H100 SXM (80 GB HBM3, 700 W power limit) the smallest values both kernels still pass were C_S 2^-23 and C_PV
2^-23, and EXP2_REL 0 (no case needs any, so its 2^-21 is an assumption); C_S = C_PV = 2^-20 keep an 8x margin.
Summary lines of that run (``span`` and ``frac`` are the largest over the cases):
  kr_attn_fwd bf16: 61 cases, ratio 0.999, span <= 0.548, frac <= 0.121, ambiguous lazy decisions 1
  kr_attn_fwd fp16: 61 cases, ratio 0.996, span <= 1,     frac <= 0.294, ambiguous lazy decisions 0
  kr_t5_attn  bf16: 70 cases, ratio 1,     span <= 0.227, frac <= 0.0073
The widest spans are the fp16 cases with thousands of keys: fp16 P has 3 more mantissa bits than bf16, so the score
bound spans two fp16 values of P on many keys, and the P V bound sums those widths over every key.
"""
import math

import pytest
import torch

from tests import kernel_refs as R

pytestmark = pytest.mark.gpu

BF, FP = torch.bfloat16, torch.float16
DTN = {BF: "bf16", FP: "fp16"}
KR_ERR_UNSUPPORTED_SHAPE = -2
SCALE_DIT = R.f32(1.0 / math.sqrt(128.0))     # kr_dit_block.cu: static_cast<float>(1 / sqrt(128))


# ---------------------------------------------------------------------------------------------
# kr_attn_fwd cases
# ---------------------------------------------------------------------------------------------
def _fc(name, Lq, Lkv, heads, block_len=0, window=0, pad=0, kind="randn", scale=None, layout="dense", restate=None):
    return dict(name=name, Lq=Lq, Lkv=Lkv, heads=heads, block_len=block_len, window=window, pad=pad, kind=kind,
                scale=scale, layout=layout, restate=restate)


def _flash_cases():
    cases = []
    i = 0
    for Lq in (1, 63, 64, 65, 127, 128, 129):
        for Lkv in (1, 127, 128, 129, 512, 1300):
            cases.append(_fc(f"{Lq}x{Lkv}", Lq, Lkv, 1 + i % 3, layout="strided" if i % 2 else "dense"))
            i += 1
    for Lkv in (1, 129, 1300):
        cases.append(_fc(f"4680x{Lkv}", 4680, Lkv, 2, layout="strided"))
    cases += [
        _fc("block end in a tile", 700, 700, 2, 84, 0, 68),
        _fc("block end on a tile boundary", 1024, 1024, 1, 256, 0, 0),
        _fc("window edge in a tile", 1200, 1200, 2, 240, 480, 80),
        _fc("window skips tiles", 1560, 1560, 2, 480, 480, 104),
        _fc("phantom negative", 250, 250, 2, 84, 0, 6, kind="negative"),
        _fc("phantom only rows", 250, 250, 2, 84, 2, 6, kind="negative"),
        _fc("bench mask negative", 4680, 4680, 2, 3120, 3120, 56, kind="negative"),
        _fc("jump at tile edge", 300, 1300, 2, kind="jump_edge"),
        _fc("jump inside tile", 300, 1300, 2, kind="jump_inside"),
        _fc("jump under 8", 300, 1300, 2, kind="jump_under8"),
        _fc("jump masked", 700, 700, 2, 84, 168, 68, kind="jump_edge"),
        _fc("spread +-100", 256, 1300, 2, kind="spread"),
        _fc("spread masked", 700, 700, 1, 240, 480, 68, kind="spread"),
        _fc("scale 0.25", 300, 700, 2, scale=0.25, layout="strided"),
        _fc("scale dit", 300, 700, 2, scale=SCALE_DIT),
        _fc("production 40 heads", 4680, 9360, 40, scale=SCALE_DIT, layout="strided", restate=[0, 13, 26, 39]),
    ]
    return cases


FLASH_CASES = _flash_cases()


def flash_inputs(case, dtype, device, seed=0):
    """(q, k, v) of one case: ``strided`` gives Q a row pitch wider than heads * 128 and K / V as row-offset views of
    larger cache tensors."""
    g = torch.Generator(device=device).manual_seed(seed + case["Lq"] * 7 + case["Lkv"] * 3 + case["heads"])
    Lq, Lkv, D = case["Lq"], case["Lkv"], case["heads"] * 128
    q = torch.randn(Lq, D, device=device, generator=g)
    k = torch.randn(Lkv, D, device=device, generator=g)
    v = torch.randn(Lkv, D, device=device, generator=g)
    kind = case["kind"]
    if kind == "negative":          # every real score ~ -4: the padded keys (score 0) carry a large share
        q, k = q.abs() * 0.75, -k.abs() * 0.75
    elif kind.startswith("jump"):   # q, k >= 0: scores ~ 10.4 f per key in log2 units, f stepping up
        f = torch.ones(Lkv, device=device)
        edge, step = {"jump_edge": (128, 2.2), "jump_inside": (200, 2.2), "jump_under8": (128, 1.7)}[kind]
        f[edge:] = step
        f[edge + 384:] = step + (step - 1)
        q, k = q.abs(), k.abs() * f[:, None]
    elif kind == "spread":          # scores ~ N(0, 43^2) in log2 units
        k = k * 30
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    if case["layout"] == "strided":
        qb = torch.zeros(Lq, D + 64, device=device, dtype=dtype)
        kb = torch.zeros(77 + Lkv + 50, D, device=device, dtype=dtype)
        vb = torch.zeros(77 + Lkv + 50, D, device=device, dtype=dtype)
        qb[:, 32:32 + D] = q
        kb[77:77 + Lkv] = k
        vb[77:77 + Lkv] = v
        q, k, v = qb[:, 32:32 + D], kb[77:77 + Lkv], vb[77:77 + Lkv]
    return q, k, v


def flash_check(case, dtype, got, q, k, v, **consts):
    """Hold one kr_attn_fwd output to :func:`kernel_refs.attn_interval`; returns (violations, stats)."""
    heads = case["heads"]
    lo, hi, info = R.attn_interval(q, k, v, heads, case["block_len"], case["window"], case["pad"], case["scale"],
                                   dtype, head_list=case["restate"], **consts)
    cols = torch.cat([torch.arange(h * 128, (h + 1) * 128, device=got.device) for h in info["heads"]])
    return R.check_attn(got[:, cols], lo, hi, dtype, info)


def run_flash(case, q, k, v, out):
    from realtime_video_b200 import ops
    ops.attention(q, k, v, heads=case["heads"], out=out, softmax_scale=case["scale"], block_len=case["block_len"],
                  window=case["window"], pad_keys=case["pad"])


# ---------------------------------------------------------------------------------------------
# kr_t5_attn cases
# ---------------------------------------------------------------------------------------------
T5_L = (1, 2, 127, 128, 129, 200, 512, 777, 1024)


def _t5_cases():
    cases = []
    for i, L in enumerate(T5_L):
        masks = ["none", "random", "all"] + [f"prefix{n}" for n in sorted({1, 37, 127, 128, 129, L - 1}) if 0 < n < L]
        if L > 128:
            masks.append("first128")
        for j, m in enumerate(masks):
            cases.append(dict(L=L, heads=4 if (i + j) % 2 else 1, mask=m))
    cases += [dict(L=512, heads=64, mask="none"), dict(L=512, heads=64, mask="prefix37"),
              dict(L=512, heads=64, mask="first128")]
    return cases


T5_CASES = _t5_cases()


def t5_inputs(case, device, seed=0):
    """(q, k, v, bias_delta, key_mask): bias uniform in +-30 per (head, offset), so an off-by-one in the offset moves
    many elements."""
    L, heads = case["L"], case["heads"]
    g = torch.Generator(device=device).manual_seed(seed + 11 * L + heads)
    D = heads * 64
    q = (torch.randn(L, D, device=device, generator=g) * 0.6).bfloat16()
    k = (torch.randn(L, D, device=device, generator=g) * 0.6).bfloat16()
    v = torch.randn(L, D, device=device, generator=g).bfloat16()
    bias = ((torch.rand(heads, 2 * L - 1, device=device, generator=g) * 2 - 1) * 30).bfloat16()
    m = case["mask"]
    km = None
    if m != "none":
        km = torch.ones(L, dtype=torch.uint8, device=device)
        if m == "all":
            km.zero_()
        elif m == "random":
            km = (torch.rand(L, device=device, generator=g) < 0.6).to(torch.uint8)
        elif m == "first128":
            km[:128] = 0
        else:
            km[int(m[len("prefix"):]):] = 0
    return q, k, v, bias, km


def t5_check(case, got, q, k, v, bias, km, **consts):
    lo, hi, info = R.t5_attn_interval(q, k, v, bias, km, case["heads"], **consts)
    return R.check_attn(got, lo, hi, BF, info)


def _cid(c):
    return c["name"].replace(" ", "_") if "name" in c else f"L{c['L']}_h{c['heads']}_{c['mask']}"


# ---------------------------------------------------------------------------------------------
# the tests
# ---------------------------------------------------------------------------------------------
_SUMMARY = {}


def _note(key, stats):
    s = _SUMMARY.setdefault(key, {"cases": 0, "ratio": 0.0, "span": 0.0, "frac": 0.0, "ambiguous": 0})
    s["cases"] += 1
    s["ratio"] = max(s["ratio"], stats["ratio"])
    s["span"] = max(s["span"], stats["span"])
    s["frac"] = max(s["frac"], stats["frac"])
    s["ambiguous"] += stats["ambiguous"]


@pytest.fixture(scope="module", autouse=True)
def _summary_lines():
    yield
    for key, s in sorted(_SUMMARY.items()):
        print(f"\n{key}: {s['cases']} cases, ratio {s['ratio']:.3g}, span <= {s['span']:.3g}, "
              f"frac <= {s['frac']:.3g}, ambiguous lazy decisions {s['ambiguous']}")


def _launch_twice(rows, cols, dtype, run):
    buf, out = R.guarded(rows, cols, dtype, "cuda")
    buf2, out2 = R.guarded(rows, cols, dtype, "cuda")
    run(out)
    run(out2)
    torch.cuda.synchronize()
    assert R.guard_intact(buf, rows, cols) and R.guard_intact(buf2, rows, cols), "guard overwritten"
    assert torch.equal(out.view(torch.int16), out2.view(torch.int16)), "two launches differ"
    return out


@pytest.mark.parametrize("dtype", [BF, FP], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", FLASH_CASES, ids=_cid)
def test_flash_attention_inside_restated_schedule(case, dtype):
    q, k, v = flash_inputs(case, dtype, "cuda")
    out = _launch_twice(case["Lq"], case["heads"] * 128, dtype, lambda o: run_flash(case, q, k, v, o))
    viol, stats = flash_check(case, dtype, out, q, k, v)
    _note(f"kr_attn_fwd {DTN[dtype]}", stats)
    assert not viol, (case["name"], viol, stats)


@pytest.mark.parametrize("case", T5_CASES, ids=_cid)
def test_t5_attention_inside_restated_schedule(case):
    from realtime_video_b200 import ops
    q, k, v, bias, km = t5_inputs(case, "cuda")
    out = _launch_twice(case["L"], case["heads"] * 64, BF,
                        lambda o: ops.t5_attention(q, k, v, bias, km, heads=case["heads"], out=o))
    viol, stats = t5_check(case, out, q, k, v, bias, km)
    _note("kr_t5_attn bf16", stats)
    assert not viol, (_cid(case), viol, stats)


def test_t5_all_masked_row_is_the_mean_of_v():
    """torch.softmax over L equal finfo.min scores is uniform: every row of an all-masked call is the mean of V."""
    from realtime_video_b200 import ops
    case = dict(L=300, heads=2, mask="all")
    q, k, v, bias, km = t5_inputs(case, "cuda")
    out = ops.t5_attention(q, k, v, bias, km, heads=2)
    mean = v.double().mean(0, keepdim=True).expand_as(out)
    assert torch.isfinite(out).all()
    assert float((out.double() - mean).abs().max()) <= float(R.ulp(mean, BF).max())


def test_t5_length_past_1024_is_refused():
    from realtime_video_b200 import _lib
    L, heads = 1025, 1
    q = torch.zeros(L, 64, dtype=BF, device="cuda")
    bias = torch.zeros(heads, 2 * L - 1, dtype=BF, device="cuda")
    out = torch.zeros_like(q)
    rc = _lib.load().kr_t5_attn(q.data_ptr(), 64, q.data_ptr(), 64, q.data_ptr(), 64, out.data_ptr(), 64, L, heads,
                                bias.data_ptr(), None, None)
    assert rc == KR_ERR_UNSUPPORTED_SHAPE


MARGIN_FLASH = ["4680x1300", "jump under 8", "spread +-100", "bench mask negative", "production 40 heads"]
MARGIN_T5 = [dict(L=1024, heads=4, mask="random"), dict(L=512, heads=64, mask="prefix37")]


def _smallest_passing(check, name, full):
    """The smallest of full * 2^-j (j = 0..16) and 0 for which ``check({name: c})`` has no violation."""
    best = full
    for c in [full * 2.0 ** -j for j in range(1, 17)] + [0.0]:
        if check({name: c})[0]:
            break
        best = c
    return best


def test_constants_margin():
    """Shrink C_S, C_PV and EXP2_REL one at a time on the widest cases: every constant keeps at least a 4x margin
    over the smallest value with which both kernels still pass, and the smallest values are printed."""
    from realtime_video_b200 import ops
    runs = []
    for name in MARGIN_FLASH:
        case = next(c for c in FLASH_CASES if c["name"] == name)
        for dtype in (BF, FP):
            q, k, v = flash_inputs(case, dtype, "cuda")
            out = torch.empty(case["Lq"], case["heads"] * 128, dtype=dtype, device="cuda")
            run_flash(case, q, k, v, out)
            runs.append((f"attn {DTN[dtype]} {name}",
                         lambda c, case=case, dtype=dtype, out=out, q=q, k=k, v=v: flash_check(case, dtype, out, q, k,
                                                                                              v, **c)))
    for case in MARGIN_T5:
        q, k, v, bias, km = t5_inputs(case, "cuda")
        out = ops.t5_attention(q, k, v, bias, km, heads=case["heads"])
        runs.append((f"t5 {_cid(case)}", lambda c, case=case, a=(out, q, k, v, bias, km): t5_check(case, *a, **c)))
    full = {"c_s": R.C_S, "c_pv": R.C_PV, "c_exp": R.EXP2_REL}
    need = {n: 0.0 for n in full}
    for what, check in runs:
        assert not check({})[0], what
        for n, c in full.items():
            need[n] = max(need[n], _smallest_passing(check, n, c))
    print("\nsmallest passing constants: " + ", ".join(
        f"{n} {v:.3g} (2^{math.log2(v):.1f})" if v else f"{n} 0" for n, v in need.items()))
    for n, c in full.items():
        assert need[n] <= c / 4, (n, need[n], c)
