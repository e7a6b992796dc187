"""The float64 GEMM checker of ``tests/kernel_refs.py`` (``gemm_interval`` / ``check_gemm`` / ``guarded``) proven on
the CPU: an emulation of a correct kernel (fp32 accumulation over 64-wide k-blocks, then gemm_epilogue_row's chain
with its rounding points) passes for every epilogue and both 16-bit types, and each of eight plausible kernel bugs
is rejected.  The restatements are also compared with ``tests/cpu_ops_emulation.gemm`` and torch."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import cpu_ops_emulation as C
from tests import kernel_refs as R

DTYPES = [torch.bfloat16, torch.float16]
EPIS = [R.EPI_BIAS, R.EPI_BIAS_GELU, R.EPI_BIAS_GATE_RES, R.EPI_BIAS_RES, R.EPI_MUL, R.EPI_F32]
# two 128-row tiles and a 44-row tail; a 96-wide column tile leaves a 64-wide last one; K = 200 ends in a k tail;
# gate boundaries at rows 13, 63, 113, ... fall inside the 64-row halves of the tiles
M, N, K, BN = 300, 352, 200, 96
RPG, ROW_OFF, ALPHA = 50, 37, 1.0 / math.sqrt(384)


def _gelu32(x):
    """gelu_tanh of kr_common.cuh in fp32."""
    inner = 0.7978845608028654 * (x + 0.044715 * x * x * x)
    return 0.5 * x * (1.0 + torch.tanh(inner))


def emulate(epi, a, w, bias, dtype, out, *, residual=None, gate=None, out2=None, n_split=0, mutate=None):
    """What the kernel computes, written into ``out`` (and ``out2`` for the columns >= n_split); ``mutate`` names a
    deliberate bug."""
    rows = a.shape[0]
    acc = torch.zeros(rows, w.shape[0], dtype=torch.float32)
    for k0 in range(0, a.shape[1], 64):
        part = a[:, k0:k0 + 64].float() @ w[:, k0:k0 + 64].float().t()
        if mutate == "drop_kblock" and k0 == 64:
            part[128:256] = 0                          # the second row tile skips its second k-block
        acc += part
    v = acc + bias.float() if bias is not None else acc
    rnd = lambda t: t.to(dtype).float()   # noqa: E731
    y = rnd(v)
    if epi == R.EPI_F32:
        y = v * {"alpha_missing": 1.0, "alpha_twice": ALPHA * ALPHA}.get(mutate, ALPHA)
    elif epi == R.EPI_BIAS_GELU:
        y = _gelu32(v if mutate == "gelu_unrounded" else y)
    elif epi == R.EPI_BIAS_GATE_RES:
        r = torch.arange(rows) + (0 if mutate == "row_offset_ignored" else ROW_OFF)
        p = y * gate.float()[r // RPG]
        y = residual.float() + (p if mutate == "gate_unrounded" else rnd(p))
    elif epi == R.EPI_BIAS_RES:
        y = residual.float() + y
    elif epi == R.EPI_MUL:
        y = residual.float() * y
    y = y.to(out.dtype)
    if mutate == "zero_last_tile":
        y[:, (N - 1) // BN * BN:] = 0
    if out2 is not None:
        out.copy_(y[:, :n_split])
        out2.copy_(y[:, n_split:])
    else:
        out.copy_(y)
    if mutate == "row_past_m":
        torch.as_strided(out, (1, out.shape[1]), out.stride(), out.storage_offset() + rows * out.stride(0)).copy_(y[-1:, :out.shape[1]])


def _operands(dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(dtype)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dtype)
    b = (torch.randn(N, generator=g) * 0.5).to(dtype)
    res = torch.randn(M, N, generator=g).to(dtype)
    gate = (torch.randn((M + ROW_OFF) // RPG + 1, N, generator=g) * 0.5).to(dtype)
    return a, w, b, res, gate


def run_checked(epi, dtype, mutate=None, bias=True, split=False):
    """Emulate one launch into guarded buffers and hold it to the checker; returns the list of violations."""
    a, w, b, res, gate = _operands(dtype)
    b = b if bias else None
    z, m, E = R.gemm_interval(a, w, b)
    odt = torch.float32 if epi == R.EPI_F32 else dtype
    obuf, out = R.guarded(M, 256 if split else N, odt, "cpu")
    o2buf, out2 = R.guarded(M, N - 256, dtype, "cpu") if split else (None, None)
    rbuf, r = R.guarded(M, N, dtype, "cpu", fill=res)
    gbuf, gv = R.guarded(gate.shape[0], N, dtype, "cpu", fill=gate)
    emulate(epi, a, w, b, dtype, out, residual=r, gate=gv, out2=out2, n_split=256 if split else 0, mutate=mutate)
    got = torch.cat([out, out2], dim=1) if split else out
    ybuf, y16 = R.guarded(M, N, dtype, "cpu")
    emulate(R.EPI_BIAS, a, w, b, dtype, y16)
    gate_r = R.gate_rows(M, gate, RPG, ROW_OFF, "cpu")
    if mutate == "one_ulp":
        hi = R.r16(z[5, 7] + E[5, 7], dtype)
        got[5, 7] = R._bits_neighbour(hi.view(1), torch.tensor([True]), dtype)[0].to(got.dtype)
    viol, stats = R.check_gemm(epi, got, z, m, E, dtype, residual=res, gate_r=gate_r, alpha=ALPHA,
                               y16=None if epi == R.EPI_F32 else y16)
    for buf, cols in ((obuf, out.shape[1]), (o2buf, N - 256), (rbuf, N), (gbuf, N)):
        if buf is not None and not R.guard_intact(buf, buf.shape[0] - 2 * R.GUARD_ROWS, cols):
            viol.append("guard overwritten")
    return viol, stats


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("epi", EPIS)
def test_checker_accepts_a_correct_kernel(epi, dtype):
    for bias in (True, False):
        viol, stats = run_checked(epi, dtype, bias=bias)
        assert not viol, (R.EPI_NAMES[epi], bias, viol, stats)
        assert stats["excess"] == 0
    if epi != R.EPI_F32:
        viol, _ = run_checked(epi, dtype, split=True)
        assert not viol, viol


MUTATIONS = [("one_ulp", R.EPI_BIAS), ("drop_kblock", R.EPI_BIAS), ("drop_kblock", R.EPI_BIAS_RES),
             ("gate_unrounded", R.EPI_BIAS_GATE_RES), ("row_offset_ignored", R.EPI_BIAS_GATE_RES),
             ("gelu_unrounded", R.EPI_BIAS_GELU), ("zero_last_tile", R.EPI_BIAS), ("zero_last_tile", R.EPI_MUL),
             ("row_past_m", R.EPI_BIAS), ("row_past_m", R.EPI_F32), ("alpha_missing", R.EPI_F32),
             ("alpha_twice", R.EPI_F32)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mutate,epi", MUTATIONS)
def test_checker_rejects_each_kernel_bug(mutate, epi, dtype):
    viol, stats = run_checked(epi, dtype, mutate=mutate)
    assert viol, (mutate, stats)


def test_checker_rejects_a_wrong_split_destination():
    viol, _ = run_checked(R.EPI_BIAS, torch.bfloat16, mutate="row_past_m", split=True)
    assert viol


@pytest.mark.parametrize("dtype", DTYPES)
def test_gelu_error_of_fp32_is_within_the_allowance(dtype):
    """The fp32 GELU of a correct kernel rounds away from the float64 GELU on far fewer elements than
    GELU_MAX_FRAC; the unrounded-argument bug on far more."""
    _, stats = run_checked(R.EPI_BIAS_GELU, dtype)
    _, bad = run_checked(R.EPI_BIAS_GELU, dtype, mutate="gelu_unrounded")
    assert stats["chain_frac"] <= R.GELU_MAX_FRAC / 4 and bad["chain_frac"] >= 4 * R.GELU_MAX_FRAC, (stats, bad)


def test_a_dropped_kblock_is_far_outside_the_bound():
    """At K = 5120 with unit-variance outputs the bound is under half a bf16 ulp of a typical |z|; one missing
    64-wide k-block moves z by more than 100 E; with the e4m3 bound, one missing 128-wide k-block still moves z by
    more than E on most elements."""
    g = torch.Generator().manual_seed(3)
    a = torch.randn(64, 5120, generator=g, dtype=torch.float64)
    w = torch.randn(32, 5120, generator=g, dtype=torch.float64) / math.sqrt(5120)
    z, m, E = R.gemm_interval(a, w)
    assert float((E / R.ulp(z)).median()) < 0.5
    drop = (a[:, 64:128] @ w[:, 64:128].t()).abs()
    assert float((drop / E).median()) > 100
    _, _, E8 = R.gemm_interval(a, w, c_acc=R.C_ACC_E4M3)
    drop8 = (a[:, 128:256] @ w[:, 128:256].t()).abs()
    assert float((drop8 > E8).double().mean()) > 0.75


@pytest.mark.parametrize("dtype", DTYPES)
def test_restatements_against_cpu_emulation_and_torch(dtype):
    a, w, b, res, gate = _operands(dtype, seed=1)
    z, m, E = R.gemm_interval(a, w, b)
    assert torch.allclose(z, F.linear(a.double(), w.double(), b.double()), rtol=0, atol=1e-12)
    assert torch.equal(m, a.double().abs() @ w.double().abs().t())
    # per-row and per-column scales of the FP8 kernels
    rs, cs = torch.rand(M, dtype=torch.float64) + 0.5, torch.rand(N, dtype=torch.float64) + 0.5
    zs, _, _ = R.gemm_interval(a, w, b, row_scale=rs, col_scale=cs)
    assert torch.allclose(zs, (a.double() @ w.double().t()) * rs[:, None] * cs[None] + b.double(), atol=1e-12)
    y16 = R.r16(z, dtype)
    gate_r = R.gate_rows(M, gate, RPG, ROW_OFF, "cpu")
    for epi, kw in ((R.EPI_BIAS, {}), (R.EPI_BIAS_GELU, {}), (R.EPI_BIAS_RES, {"residual": res}),
                    (R.EPI_MUL, {"residual": res}),
                    (R.EPI_BIAS_GATE_RES, {"residual": res, "gate": gate, "rows_per_gate": RPG, "row_offset": ROW_OFF})):
        want = C.gemm(a, w, None if epi == R.EPI_MUL else b, epilogue=epi, **kw)
        if epi == R.EPI_MUL:        # the emulation multiplies (a w^T) without bias
            y16m = R.r16(z - b.double(), dtype)
            got = R.r16(R.epi_chain(epi, y16m, dtype, res, gate_r), dtype)
        else:
            got = R.r16(R.epi_chain(epi, y16, dtype, res, gate_r), dtype)
        # the emulation accumulates in fp32 and skips the intermediate roundings: one ulp of the result, plus the
        # first rounding and the fp32 error carried through the chain's slope, plus the gate product's rounding
        slope = {R.EPI_BIAS_GELU: 1.13, R.EPI_MUL: res.double().abs(), R.EPI_BIAS_GATE_RES: gate_r.abs()}.get(epi, 1.0)
        slack = R.ulp(want, dtype) + slope * (R.ulp(y16, dtype) + 2 ** -16 * m)
        if epi == R.EPI_BIAS_GATE_RES:
            slack = slack + R.ulp(y16 * gate_r, dtype)
        assert bool(((got - want.double()).abs() <= slack).all()), R.EPI_NAMES[epi]
    gl = R.epi_chain(R.EPI_BIAS_GELU, y16, dtype)
    assert torch.allclose(gl, F.gelu(y16, approximate="tanh"), atol=1e-15)
    f32 = C.gemm(a, w, b, epilogue=R.EPI_F32, alpha=ALPHA)
    assert float(((f32.double() - z * ALPHA).abs() / (m * ALPHA)).max()) < 2 ** -16


def test_gelu_interval_and_acc_ratio():
    x = torch.linspace(-3, 3, 60001, dtype=torch.float64)
    lo, hi = torch.tensor([-2.0, -1.0, 0.5, -0.8]), torch.tensor([-1.0, 0.3, 1.0, -0.7])
    mn, mx = R.gelu_interval(lo.double(), hi.double())
    g = R.gelu_tanh(x)
    for i in range(4):
        inside = g[(x >= lo[i]) & (x <= hi[i])]
        assert float(mn[i]) <= float(inside.min()) + 1e-12 and float(mx[i]) >= float(inside.max()) - 1e-12
        assert float(mn[i]) >= float(inside.min()) - 2e-4     # grid spacing 1e-4, |slope| < 1.13
    assert abs(float(R.gelu_tanh(torch.tensor(R.GELU_ARGMIN))) - R.GELU_MIN) < 1e-15
    z = torch.tensor([[1.0 + 2 ** -10, 3.0]], dtype=torch.float64)
    m = torch.ones_like(z)
    assert R.acc_ratio(R.r16(z), z, m, torch.bfloat16) == 0.0
    # 1 + 2^-10 rounds to 1; reading 1 + 2^-7 needs an accumulation error of at least 2^-8 - 2^-10
    y = torch.tensor([[1.0 + 2 ** -7, 3.0]], dtype=torch.float64)
    assert R.acc_ratio(y, z, m, torch.bfloat16) == 2 ** -8 - 2 ** -10
    # the neighbour walk crosses zero and keeps the sign-magnitude order
    v = torch.tensor([1.0, -1.0, 0.0], dtype=torch.float64)
    up = R._bits_neighbour(v, torch.tensor([True, True, True]), torch.float16)
    dn = R._bits_neighbour(v, torch.tensor([False, False, False]), torch.float16)
    assert up.tolist() == [1 + 2 ** -10, -(1 - 2 ** -11), 2 ** -24]
    assert dn.tolist() == [1 - 2 ** -11, -(1 + 2 ** -10), -(2 ** -24)]


def test_guarded_buffers():
    buf, v = R.guarded(5, 32, torch.bfloat16, "cpu", fill=torch.ones(5, 32))
    assert v.stride(0) == 56 and v.data_ptr() % 16 == 0 and R.guard_intact(buf, 5, 32)
    buf[R.GUARD_ROWS + 5, R.GUARD_COLS] = 0           # the row past M
    assert not R.guard_intact(buf, 5, 32)
    buf, v = R.guarded(5, 32, torch.float32, "cpu")
    assert torch.isnan(buf).all() and R.guard_intact(buf, 5, 32)
    buf[1, 0] = 1.0
    assert not R.guard_intact(buf, 5, 32)
