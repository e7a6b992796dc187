"""The float64 kernel references of ``tests/kernel_refs.py`` checked on the CPU against ``oracle/dit_oracle.py``,
``oracle/vae_oracle.py`` and the torch functionals they restate, so a mistake in a reference cannot make a GPU
parity test pass vacuously.  Rounded references are compared with the oracle run in bf16 (the reference's eager
rounding points) to within one ulp; unrounded ones with the float64 oracle to 1e-12."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import dit_oracle as O
from oracle import vae_oracle as V
from tests import kernel_refs as R

BF = torch.bfloat16


def _close(a, b, tol=1e-12):
    a, b = a.double(), b.double()
    return float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


def test_r16_and_ulp():
    x = torch.tensor([1.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, 3.0, -0.75, 0.0], dtype=torch.float64)
    assert R.r16(x).tolist() == [1.0, 1.0, 1.0 + 2 ** -6, 3.0, -0.75, 0.0]       # ties to even
    assert R.ulp(x[:5]).tolist() == [2 ** -7, 2 ** -7, 2 ** -7, 2 ** -6, 2 ** -8]
    assert R.ulp(torch.tensor([1.0], dtype=torch.float64), torch.float16).item() == 2 ** -10
    m, frac = R.ulp_excess(torch.tensor([1.0 + 2 ** -7, 2.0]), torch.tensor([1.0, 2.0]))
    assert m == 1.0 and frac == 0.5


def test_ln_modulate_ref_vs_oracle():
    g = torch.Generator().manual_seed(0)
    L, D, fs = 12, 64, 4
    x = (torch.randn(L, D, generator=g) * 3 + 1).to(BF)
    w, b = (torch.randn(D, generator=g).to(BF) for _ in range(2))
    mod = (torch.randn(3, 6, D, generator=g) * 0.5).to(BF)
    out, exact, _ = R.ln_modulate(x, 1e-6)
    assert _close(exact, F.layer_norm(x.double(), (D,), eps=1e-6))
    assert R.ulp_excess(out, O.layer_norm(x, 1e-6))[0] <= 1
    out, exact, _ = R.ln_modulate(x, 1e-6, w, b)
    assert _close(exact, F.layer_norm(x.double(), (D,), w.double(), b.double(), 1e-6))
    assert R.ulp_excess(out, O.layer_norm(x, 1e-6, w, b))[0] <= 1
    # the DiT block's modulated norm (causal_model.py:466-471): per frame, shift = e[0], scale = e[1]
    out, exact, _ = R.ln_modulate(x, 1e-6, mod=mod, shift_idx=0, scale_idx=1, rows_per_frame=fs)
    e = mod.chunk(6, dim=1)
    want = (O.layer_norm(x, 1e-6).unflatten(0, (3, fs)) * (1 + e[1]) + e[0]).flatten(0, 1)     # bf16 eager
    assert R.ulp_excess(out, want)[0] <= 1
    want64 = (F.layer_norm(x.double(), (D,), eps=1e-6).unflatten(0, (3, fs)) * (1 + e[1].double()) +
              e[0].double()).flatten(0, 1)
    assert _close(exact, want64)
    # row_offset: rows of a shard starting at global row 5 use the frame of their global row
    part, _, _ = R.ln_modulate(x[5:], 1e-6, mod=mod, shift_idx=0, scale_idx=1, rows_per_frame=fs, row_offset=5)
    assert torch.equal(part, out[5:])


@pytest.mark.parametrize("start_frame", [0, 3])
def test_qk_norm_rope_ref_vs_oracle(start_frame):
    g = torch.Generator().manual_seed(1)
    gh, gw, heads, hd = 3, 5, 2, 128
    L = 2 * gh * gw
    x = torch.randn(L, heads * hd, generator=g).to(BF)
    w = (1 + 0.1 * torch.randn(heads * hd, generator=g)).to(BF)
    out, exact = R.qk_norm_rope(x, w, 1e-6, hd, gh, gw, start_frame)
    ang = O.rope_table(hd)
    want = O.rope_apply(O.rms_norm(x, w, 1e-6).view(L, heads, hd), (2, gh, gw), ang, start_frame).reshape(L, -1)
    m, frac = R.ulp_excess(out, want)
    assert m <= 1 and frac < 0.01, (m, frac)
    want64 = O.rope_apply((O.rms_norm(x.double(), torch.ones(heads * hd, dtype=torch.float64), 1e-6) *
                           w.double()).view(L, heads, hd), (2, gh, gw), ang, start_frame).reshape(L, -1)
    assert _close(exact, want64)
    # the three sub-bands are told apart: exchanging grid_h and grid_w changes the result
    assert not torch.equal(R.qk_norm_rope(x, w, 1e-6, hd, gw, gh, start_frame)[0], out)


def test_rope_table_is_the_products_table():
    from realtime_video_b200.dit import rope_angles
    d = 128
    ang = torch.cat([rope_angles(1024, d - 4 * (d // 6)), rope_angles(1024, 2 * (d // 6)),
                     rope_angles(1024, 2 * (d // 6))], dim=1)
    t = R.rope_table_f32(d, "cpu")
    assert torch.equal(t, torch.stack([ang.cos(), ang.sin()], dim=-1).float())


def test_rmsnorm_ref_vs_oracle():
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(7, 96, generator=g) * 4).to(BF)
    w = torch.randn(96, generator=g).to(BF)
    m, _ = R.ulp_excess(R.rmsnorm(x, w, 1e-6), O.rms_norm(x, w, 1e-6))
    assert m <= 1


def test_activation_refs():
    x = torch.linspace(-100, 100, 4001, dtype=torch.float64)
    assert _close(R.silu(x), x * torch.sigmoid(x))
    assert _close(R.gelu_tanh(x), 0.5 * x * (1 + torch.tanh(math.sqrt(2 / math.pi) * (x + 0.044715 * x ** 3))))


def test_patchify_ref_vs_conv3d():
    g = torch.Generator().manual_seed(3)
    C, Fr, H, W, D = 4, 2, 6, 8, 10
    x = torch.randn(C, Fr, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(D, C, 1, 2, 2, generator=g, dtype=torch.float64)
    tok = F.conv3d(x[None], w, stride=(1, 2, 2)).flatten(2).transpose(1, 2)[0]      # causal_model.py:874-877
    assert _close(R.patchify(x) @ w.flatten(1).t(), tok)


def test_unpatchify_ref_vs_oracle():
    g = torch.Generator().manual_seed(4)
    C, Fr, H, W = 3, 2, 4, 6
    out = torch.randn(Fr * (H // 2) * (W // 2), 4 * C, generator=g)
    u = out.reshape(Fr, H // 2, W // 2, 1, 2, 2, C)                                # dit_oracle.forward_inference
    want = torch.einsum("fhwpqrc->cfphqwr", u).reshape(C, Fr, H, W).transpose(0, 1)
    assert torch.equal(R.unpatchify(out, C, Fr, H, W), want)


def test_flow_to_x0_ref_vs_oracle():
    g = torch.Generator().manual_seed(5)
    sched = O.FlowMatchSchedulerOracle()
    t = sched.timesteps[torch.tensor([0, 250, 700])]
    flow = torch.randn(3, 2, 4, 4, generator=g).to(BF)
    xt = torch.randn(3, 2, 4, 4, generator=g).to(BF)
    sig = sched.sigmas.double()[torch.tensor([0, 250, 700])]
    assert torch.equal(R.flow_to_x0(flow, xt, sig), O.flow_to_x0(flow, xt, t, sched))


@pytest.mark.parametrize("Lq,Lkv,block_len,window,pad", [(40, 70, 0, 0, 0), (100, 100, 30, 0, 28),
                                                         (100, 100, 30, 60, 28), (130, 130, 40, 80, 126)])
def test_attention_ref_vs_oracle(Lq, Lkv, block_len, window, pad):
    g = torch.Generator().manual_seed(Lq + pad)
    heads = 2
    q, k, v = (torch.randn(n, heads * 128, generator=g, dtype=torch.float64) for n in (Lq, Lkv, Lkv))
    got = R.attention(q, k, v, heads, block_len, window, pad)
    if block_len:
        # the oracle's recompute branch: zero rows appended, mask over the padded length (dit_oracle self_attn)
        kk = torch.cat([k, k.new_zeros(pad, heads * 128)])
        vv = torch.cat([v, v.new_zeros(pad, heads * 128)])
        mask = O.block_causal_mask(Lq, Lkv + pad, block_len, window)
        want = O.attention(q.view(Lq, heads, 128), kk.view(-1, heads, 128), vv.view(-1, heads, 128), mask)
    else:
        want = O.attention(q.view(Lq, heads, 128), k.view(-1, heads, 128), v.view(-1, heads, 128))
    assert float((got - want.reshape(Lq, -1)).abs().max()) < 1e-5
    assert float(R.rel_rows_heads(want.reshape(Lq, -1).double(), got, heads).max()) < 1e-5
    scaled = R.attention(q, k, v, heads, softmax_scale=0.3)
    s = (q.view(Lq, heads, 128).transpose(0, 1) @ k.view(Lkv, heads, 128).transpose(0, 1).transpose(1, 2)) * 0.3
    assert _close(scaled, (torch.softmax(s, -1) @ v.view(Lkv, heads, 128).transpose(0, 1)).transpose(0, 1)
                  .reshape(Lq, -1))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_vae_rmsnorm_ref_vs_oracle(dtype):
    g = torch.Generator().manual_seed(6)
    C = 96
    x = (torch.randn(5, 3, 4, C, generator=g) * 2).to(dtype)          # channels-last [T, H, W, C]
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(dtype)
    y, exact = R.vae_rmsnorm(x, gamma, dtype)
    want = V.rms_norm(x.double().permute(3, 0, 1, 2)[None], gamma.double().view(C, 1, 1, 1))[0].permute(1, 2, 3, 0)
    assert _close(exact, want)
    # four rounding points, each within half an ulp of its own value: |y - exact| <= 4 ulp(exact) (and 0 at 0)
    assert float(((y - exact).abs() / R.ulp(exact, dtype)).max()) <= 4
    s, sexact = R.vae_rmsnorm_silu(x, gamma, dtype)
    assert _close(sexact, F.silu(want))
    assert torch.equal(s, F.silu(y).to(dtype).double())
    zero = torch.zeros(2, C, dtype=dtype)
    assert float(R.vae_rmsnorm(zero, gamma, dtype)[0].abs().max()) == 0


def test_softmax_ref():
    s = torch.randn(4, 33, dtype=torch.float32)
    assert _close(R.softmax_rows(s), torch.softmax(s.double(), -1))
    assert _close(R.softmax_rows(s).sum(-1), torch.ones(4, dtype=torch.float64))
