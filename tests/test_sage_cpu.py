"""Quantised attention tier (kr_sage_quantize / kr_sage_attn) without a GPU: the oracle's scale groups, key order and
K smoothing; the DiT host schedule with ``attn_quant="sage"`` on stand-in kernels; argument validation of the C ABI;
the SASS and register budget of sage_attn_kernel."""
import ctypes
import math
import re
import shutil
import subprocess
import types

import pytest
import torch

from oracle import sage_oracle as so
from tests import cpu_ops_emulation as emu
from tests.golden_io import load_npz, rel_l2, weights


# ---------------------------------------------------------------------------------------------------------------
# oracle
# ---------------------------------------------------------------------------------------------------------------
def test_scale_groups_are_the_wgmma_fragment_rows_and_columns():
    """A thread of a consumer warp holds S rows lane/4 and lane/4 + 8 of its 16-row block and S columns
    8j + 2(lane%4) + {0,1} of a 128-key tile: one Q group per (block, lane/4), one K group per (tile, lane%4)."""
    for lane in range(32):
        assert so.q_group_rows(3, lane // 4) == [48 + lane // 4, 56 + lane // 4]
        assert so.k_group_keys(2, lane % 4) == sorted(256 + 8 * j + 2 * (lane % 4) + e for j in range(16) for e in range(2))
    assert sorted(sum((so.q_group_rows(0, t) for t in range(8)), [])) == list(range(16))
    assert sorted(sum((so.k_group_keys(0, t) for t in range(4)), [])) == list(range(128))


def test_oracle_scales_follow_the_groups():
    torch.manual_seed(0)
    H, Lq, Lkv = 2, 40, 300
    q, k, v = (torch.randn(n, H * 128).bfloat16() for n in (Lq, Lkv, Lkv))
    b = so.quantize(q, k, v, H)
    ks = (k - b["k_mean"]).float()
    for h in range(H):
        cols = slice(128 * h, 128 * h + 128)
        for blk in range((Lq + 15) // 16):
            for t in range(8):
                rows = [r for r in so.q_group_rows(blk, t) if r < Lq]      # rows >= Lq do not count
                amax = q[rows, cols].float().abs().max() if rows else torch.tensor(0.0)
                assert float(b["q_scale"][h, blk, t]) == float(amax / 127 + 1e-7)
        for c in range((Lkv + 127) // 128):
            for t in range(4):
                keys = [j for j in so.k_group_keys(c, t) if j < Lkv]
                amax = ks[keys, cols].abs().max() if keys else torch.tensor(0.0)
                assert float(b["k_scale"][h, c, t]) == float(amax / 127 + 1e-7)
    deq = b["q_i8"].float().view(Lq, H, 128) * b["q_scale"][:, torch.arange(Lq) // 16, torch.arange(Lq) % 8].t()[..., None]
    assert rel_l2(deq.view(Lq, -1), q.float()) < 1e-2
    assert int(b["q_i8"].abs().max()) == 127 and int(b["k_i8"].abs().max()) == 127
    assert b["v_t8"].shape == (H * 128, 384) and int(so.unpermute_keys(b["v_t8"])[:, Lkv:].sum()) == 0


def test_key_permutation_round_trips_and_is_the_k32_register_layout():
    x = torch.arange(64)
    assert torch.equal(so.unpermute_keys(so.permute_keys(x)), x)
    assert torch.equal(so.permute_keys(so.unpermute_keys(x)), x)
    for t in range(4):       # A bytes 4t..4t+3 of the e4m3 k32 fragment = the thread's S columns 2t, 2t+1, 8+2t, 9+2t
        assert so.PERM[4 * t:4 * t + 4] == [2 * t, 2 * t + 1, 8 + 2 * t, 9 + 2 * t]


def test_oracle_error_against_exact_attention():
    """The tier's size on Gaussian data (one head): V and P in e4m3 dominate."""
    torch.manual_seed(1)
    q, k, v = (torch.randn(n, 128).bfloat16() for n in (256, 2000, 2000))
    got = so.sage_attention(q, k, v, 1)
    want = so.exact_attention(q, k, v, 1)
    r = rel_l2(got.float(), want)
    cos = torch.nn.functional.cosine_similarity(got.double().flatten(), want.double().flatten(), 0)
    assert 2e-2 < r < 5e-2 and cos > 0.998, (r, float(cos))


def test_k_smoothing_removes_a_per_channel_offset():
    """A per-channel offset added to every key leaves softmax unchanged.  With smoothing the quantised pipeline sees
    the same k - mean and its output barely moves; without it the offset inflates every INT8 K scale.  K lies on a
    1/16 grid with zero column means and the offsets are integers, so k + offset is exact in bf16."""
    torch.manual_seed(2)
    q = torch.randn(128, 128).bfloat16()
    v = torch.randn(1024, 128).bfloat16()
    half = (torch.randn(512, 128) * 16).round() / 16
    k = torch.cat([half, -half]).bfloat16()
    off = torch.randint(-3, 4, (128,)).float()
    k2 = (k.float() + off).bfloat16()
    assert torch.equal(k2.float() - off, k.float())
    moved = rel_l2(so.sage_attention(q, k2, v, 1).float(), so.sage_attention(q, k, v, 1).float())
    moved_raw = rel_l2(so.sage_attention(q, k2, v, 1, smooth=False).float(),
                       so.sage_attention(q, k, v, 1, smooth=False).float())
    assert moved < 1e-3 and moved_raw > 1e-2, (moved, moved_raw)


# ---------------------------------------------------------------------------------------------------------------
# DiT host schedule on stand-in kernels
# ---------------------------------------------------------------------------------------------------------------
def _stand_ins(calls):
    ns = types.SimpleNamespace(**{n: getattr(emu, n) for n in dir(emu) if not n.startswith("__")})

    def attention(q, k, v, *, heads, out=None, block_len=0, **kw):
        calls.append(("attention", block_len > 0))
        return emu.attention(q, k, v, heads=heads, out=out, block_len=block_len, **kw)

    def sage_attention(q, k, v, *, heads, out=None, softmax_scale=None):
        calls.append(("sage", q.shape[0], k.shape[0]))
        o = so.sage_attention(q.bfloat16(), k.bfloat16(), v.bfloat16(), heads, softmax_scale).to(q.dtype)
        return emu._store(out, o)
    ns.attention, ns.sage_attention = attention, sage_attention
    return ns


def _small_model():
    import realtime_video_b200.dit as dit
    g = load_npz("dit_small.npz")
    m = dit.CausalWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=2, text_dim=128)
    m.load_state_dict(weights(g, torch.float32), strict=False)
    m = m.float().eval()
    for blk in m.blocks:
        blk.self_attn.fuse_projections()
    return m, g


def _run(m, g, mask=None):
    kv = [dict(k=torch.zeros(1, 6 * 96, 2, 128), v=torch.zeros(1, 6 * 96, 2, 128), global_end_index=0,
               local_end_index=0) for _ in range(2)]
    ca = [dict(k=torch.zeros(1, 512, 2, 128), v=torch.zeros(1, 512, 2, 128), is_init=False) for _ in range(2)]
    m.block_mask = mask
    with torch.no_grad():
        return m(g["in/x0"].float()[None], t=torch.full((1, 3), 750.0), context=g["in/ctx"].float()[None],
                 seq_len=32760, kv_cache=kv, crossattn_cache=ca, current_start=0)[0]


@pytest.mark.parametrize("branch", ["cache", "recompute"])
def test_schedule_sends_the_unmasked_attention_to_the_quantised_tier(monkeypatch, branch):
    """attn_quant="sage": the cache-branch self-attention and the cross-attention call sage_attention, the block-causal
    recompute branch stays on attention; the result tracks the bf16 schedule within the tier's tolerance."""
    import realtime_video_b200.dit as dit
    calls = []
    monkeypatch.setattr(dit, "ops", _stand_ins(calls))
    m, g = _small_model()
    mask = None if branch == "cache" else m._prepare_blockwise_causal_attn_mask("cpu", num_frames=3, frame_seqlen=96)
    ref = _run(m, g, mask)
    assert all(c[0] == "attention" for c in calls) and len(calls) == 4
    calls.clear()
    m.attn_quant = "sage"
    got = _run(m, g, mask)
    L = 3 * 96
    if branch == "cache":
        assert calls == [("sage", L, L), ("sage", L, 512)] * 2
    else:
        assert calls == [("attention", True), ("sage", L, 512)] * 2
    r = rel_l2(got, ref)
    assert torch.isfinite(got).all() and r < 0.1, r


def test_one_call_blocks_are_ineligible_with_the_quantised_tier():
    m, _ = _small_model()
    m = m.to(torch.bfloat16)
    x = torch.zeros(8, 256, dtype=torch.bfloat16)
    blk = m.blocks[0]
    assert m._block_fwd_eligible(blk, x, {"is_init": True})
    m.attn_quant = "sage"
    assert not m._block_fwd_eligible(blk, x, {"is_init": True})


def test_environment_switch_sets_the_attribute(monkeypatch):
    from realtime_video_b200.dit import CausalWanModel

    def make():
        return CausalWanModel(dim=256, ffn_dim=512, num_heads=2, num_layers=1, text_dim=128)
    monkeypatch.delenv("KR_SAGE_ATTN", raising=False)
    assert make().attn_quant is None
    monkeypatch.setenv("KR_SAGE_ATTN", "0")
    assert make().attn_quant is None
    monkeypatch.setenv("KR_SAGE_ATTN", "1")
    assert make().attn_quant == "sage"


def test_unknown_tier_is_an_error(monkeypatch):
    import realtime_video_b200.dit as dit
    monkeypatch.setattr(dit, "ops", _stand_ins([]))
    m, g = _small_model()
    m.attn_quant = "int4"
    with pytest.raises(ValueError, match="attn_quant"):
        _run(m, g)


# ---------------------------------------------------------------------------------------------------------------
# C ABI and SASS (no GPU needed)
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    from realtime_video_b200 import _lib
    _lib.build()
    return _lib.load()


def test_sage_header_is_bound_and_exported(lib):
    """include/krea_b200_sage.h (pulled in by krea_b200.h) declares exactly the entry points bound in
    _lib.SAGE_SIGNATURES, every one returns int, and the library exports them."""
    from pathlib import Path
    from realtime_video_b200 import _lib
    inc = Path(__file__).resolve().parent.parent / "include"
    assert '#include "krea_b200_sage.h"' in (inc / "krea_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", (inc / "krea_b200_sage.h").read_text(), flags=re.S)
    decl = re.findall(r"\b(\w+)\s+(kr_[a-z0-9_]+)\s*\(", text)
    assert {n for _, n in decl} == set(_lib.SAGE_SIGNATURES) == {"kr_sage_quantize", "kr_sage_attn"}
    assert all(t == "int" for t, _ in decl)
    for n in _lib.SAGE_SIGNATURES:
        assert hasattr(lib, n) and getattr(lib, n).restype is ctypes.c_int


def test_quantize_rejects_bad_arguments_before_any_cuda_call(lib):
    P = 4096                     # a 16-byte aligned stand-in address: never dereferenced on these paths
    ok = dict(q=P, ldq=256, k=P, ldk=256, v=P, ldv=256, Lq=16, Lkv=16, heads=2, q_i8=P, q_scale=P, k_mean=P, k_i8=P,
              k_scale=P, v_t8=P, v_scale=P)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.kr_sage_quantize(*a.values(), None), lib.kr_last_error()
    for bad, msg in ((dict(q=None), b"null"), (dict(v_t8=None), b"null"), (dict(Lkv=0), b"non-positive"),
                     (dict(heads=-1), b"non-positive"), (dict(ldk=128), b"pitch"), (dict(ldv=260), b"multiples"),
                     (dict(k=P + 2), b"aligned")):
        rc, err = call(**bad)
        assert rc == -1 and msg in err and b"kr_sage_quantize" in err, (bad, rc, err)


def test_attn_rejects_bad_arguments_before_any_cuda_call(lib):
    P = 4096
    ok = dict(q_i8=P, q_scale=P, k_i8=P, k_scale=P, v_t8=P, v_scale=P, out=P, ldo=256, Lq=16, Lkv=16, heads=2,
              softmax_scale=ctypes.c_float(1 / math.sqrt(128)))

    def call(**kw):
        a = dict(ok, **kw)
        return lib.kr_sage_attn(*a.values(), None), lib.kr_last_error()
    for bad, msg in ((dict(k_scale=None), b"null"), (dict(out=None), b"null"), (dict(Lq=0), b"non-positive"),
                     (dict(ldo=128), b"ldo"), (dict(softmax_scale=ctypes.c_float(0.0)), b"softmax_scale"),
                     (dict(softmax_scale=ctypes.c_float(float("nan"))), b"softmax_scale"),
                     (dict(out=P + 4), b"aligned")):
        rc, err = call(**bad)
        assert rc == -1 and msg in err and b"kr_sage_attn" in err, (bad, rc, err)


needs_cuobjdump = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@needs_cuobjdump
def test_sage_kernel_is_int8_and_e4m3_wgmma_fed_by_tma(lib):
    from realtime_video_b200 import _lib
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    bodies = re.split(r"\n\s*Function : ", out)
    sage = [b for b in bodies if b.split("\n", 1)[0].strip().find("sage_attn_kernel") >= 0]
    assert len(sage) == 1
    ops = set()
    for line in sage[0].splitlines()[1:]:
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*)", line)
        if m and m.group(1):
            t = m.group(1).split()
            ops.add(t[1] if t[0].startswith("@") else t[0])
    for need in ("IGMMA", "QGMMA", "UTMALDG", "MUFU.EX2"):
        assert any(o.startswith(need) for o in ops), need
    assert not any(o.startswith(("HMMA", "IMMA")) for o in ops)


@needs_cuobjdump
def test_sage_kernel_register_and_stack_budget(lib):
    """384 threads at launch allow 168 registers (the consumer warpgroups raise theirs with setmaxnreg); o, the fresh
    P.V accumulator and the packed P live together in registers."""
    from realtime_video_b200 import _lib
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", str(_lib.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    found = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line and "sage_" in name:
            found[name] = (int(re.search(r"REG:(\d+)", line).group(1)), int(re.search(r"STACK:(\d+)", line).group(1)))
            name = None
    attn = [v for n, v in found.items() if "sage_attn_kernel" in n]
    assert len(attn) == 1 and attn[0][0] <= 168 and attn[0][1] <= 64, found
    assert len(found) == 4 and all(stack == 0 for _, stack in found.values()), found
