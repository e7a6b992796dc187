"""Static checks on the SASS of the built library (cuobjdump, no GPU needed): the hot kernels really are
wgmma / TMA code for sm_90a, there is no legacy mma.sync tensor path, and the single-thread TMA issue loops are
emitted back to back — `lane == 0` guards make ptxas wrap every UTMALDG in an ELECT + branch loop, `elect.sync`
guards do not (DESIGN.md §4 'Issue threads')."""
import re
import shutil
import subprocess

import pytest

from realtime_video_b200 import _lib

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="cuobjdump not on PATH")


@pytest.fixture(scope="module")
def sass():
    _lib.load()                      # builds the library if needed
    out = subprocess.run(["cuobjdump", "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    funcs, name, body = {}, None, []
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = body
            name, body = m.group(1), []
        elif name and re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            body.append(line.split("*/", 1)[1].strip())
    if name:
        funcs[name] = body
    return funcs


def _ops(body):
    return [(l.split()[1] if l.startswith("@") else l.split()[0]) for l in body if l]


def test_compiled_for_sm_90a_only():
    out = subprocess.run(["cuobjdump", "-lelf", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


@pytest.mark.parametrize("pattern,needs", [
    ("gemm_tn_kernel", ("HGMMA", "UTMALDG", "SYNCS")),
    ("gemm_flex_kernel", ("HGMMA", "UTMALDG", "SYNCS")),
    ("gemm2_tn_kernel", ("HGMMA", "UTMALDG", "UCGABAR")),
    ("gemm_sk_kernel", ("HGMMA", "UTMALDG", "SYNCS")),
    ("gemm_fp8_kernel", ("QGMMA", "UTMALDG", "SYNCS")),
    ("attn_fwd_kernel", ("HGMMA", "UTMALDG", "MUFU.EX2")),
    ("t5_attn_kernel", ("HGMMA", "UTMALDG", "MUFU.EX2")),
    ("conv_igemm_kernel", ("HGMMA", "UTMALDG", "SYNCS")),
    ("conv_halo_kernel", ("HGMMA", "UTMALDG", "SYNCS")),
])
def test_hot_kernels_are_wgmma_and_tma(sass, pattern, needs):
    hits = {k: v for k, v in sass.items() if pattern in k}
    assert hits, f"no kernel matching {pattern}"
    for name, body in hits.items():
        ops = _ops(body)
        for n in needs:
            assert any(o.startswith(n) for o in ops), f"{name}: no {n}"


def test_no_legacy_tensor_core_path(sass):
    for name, body in sass.items():
        assert not any(o.startswith(("HMMA", "IMMA")) for o in _ops(body)), name


def test_issue_threads_are_not_wrapped_in_elect_loops(sass):
    for name, body in sass.items():
        ops = _ops(body)
        for i, o in enumerate(ops):
            if o.startswith("UTMALDG"):
                assert not any(p.startswith("ELECT") for p in ops[max(0, i - 2):i]), f"{name}: {o} behind an ELECT loop"


def test_register_and_stack_budget():
    """Resource usage of the hot kernels (cuobjdump --dump-resource-usage): the GEMM and conv kernels keep their
    accumulators and epilogue in registers (no stack), the attention kernel stays within the 168 registers that
    384 threads per SM allow at launch (the consumer warpgroups raise theirs with setmaxnreg) with at most a few
    spill slots."""
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", str(_lib.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    usage = {}
    name = None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            name = m.group(1)
        elif name and "REG:" in line:
            usage[name] = (int(re.search(r"REG:(\d+)", line).group(1)), int(re.search(r"STACK:(\d+)", line).group(1)))
            name = None
    assert usage
    for fn, (reg, stack) in usage.items():
        head_conv = "conv_igemm_kernelILi96ELi16E" in fn      # 96 -> 3 head: runtime channel loop over a 16-entry array
        if any(k in fn for k in ("gemm_tn_kernel", "gemm_flex_kernel", "gemm2_tn_kernel", "conv_igemm_kernel",
                                 "conv_halo_kernel")) \
                and not head_conv:
            assert stack == 0, (fn, reg, stack)
        if "attn_fwd_kernel" in fn:
            assert reg <= 168 and stack <= 64, (fn, reg, stack)


def test_jpeg_kernels_keep_their_tables_out_of_local_memory(sass):
    """kr_jpeg.cu: the per-block DCT keeps its 64 coefficients in registers (zigzag / quant-table indices fold to
    constants after unrolling), the Huffman tables live in __constant__ memory built at compile time, the bit stream is
    assembled with global OR-reductions and the per-frame prefix sums with warp shuffles."""
    kern = {k: _ops(v) for k, v in sass.items() if "jpeg_" in k}
    assert len(kern) == 5, sorted(kern)                       # dct (2 loaders), scan, emit, stuff
    emit = next(v for k, v in kern.items() if "jpeg_emit" in k)
    assert any(o.startswith(("RED", "ATOMG")) and ".OR" in o for o in emit)
    for name in ("jpeg_scan", "jpeg_stuff"):
        ops = next(v for k, v in kern.items() if name in k)
        assert any(o.startswith("SHFL.UP") for o in ops), name
    out = subprocess.run(["cuobjdump", "--dump-resource-usage", str(_lib.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    for m in re.finditer(r"Function (\S*jpeg_\S*):\s*\n\s*(.*)", out):
        stack = int(re.search(r"STACK:(\d+)", m.group(2)).group(1))
        assert stack <= 16, (m.group(1), stack)               # a spilled temporary at most; no local arrays
