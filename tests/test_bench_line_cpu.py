"""bench.py assembles its ONE JSON line in a pure function: exercised here with fabricated measurements for every mode
the driver (or a user) can launch, so that a key error cannot cost a finished multi-minute GPU run its result.  Also
checks the contract's required keys and that the line is JSON-serialisable."""
import argparse
import json

import pytest

import bench

REQUIRED = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
            "vs_baseline", "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"]


def fake_args(**kw):
    d = dict(gpus=1, steps=4, warmup=3, layers=bench.LAYERS, block_fwd="off", graphs="off")
    d.update(kw)
    return argparse.Namespace(**d)


def fake_prof():
    return {"gemm": {"flops": 5.6e14, "ms": 800.0, "n": 1246},
            "gemm/gemm_flex_kernel": {"flops": 2.8e14, "ms": 380.0, "n": 400},
            "gemm/gemm_tn_kernel": {"flops": 2.8e14, "ms": 420.0, "n": 836},
            "attention": {"flops": 1.7e14, "ms": 190.0, "n": 400},
            "vae_conv": {"flops": 4.0e13, "ms": 44.0, "n": 73}}


def fake_run(sp=False, exchange=None, note=None):
    r = {"ms": 2772.0, "launches": 36156, "clocks": {"sm_mhz": 1537.0, "sm_max_mhz": 1965.0, "reasons": ["sw_power_cap"],
                                                     "samples": 19},
         "prof": fake_prof(), "ms_prof": 693.0, "decode": True}
    if sp:
        r["exchange"], r["exchange_note"] = exchange, note
    return r


E2E = {"ms": 2790.0, "h2d": 599040, "d2h": 57507840, "host_ref_ms": None}


@pytest.mark.parametrize("world,parallel,exchange", [(1, "sp", None), (2, "sp", "p2p"), (8, "sp", "nccl"), (4, "pp", None),
                                                     (4, "replicas", None)])
def test_line_for_every_mode(world, parallel, exchange):
    sp_mode = world > 1 and parallel in ("sp", "pp")
    pp_mode = world > 1 and parallel == "pp"
    args = fake_args(gpus=world)
    main_run = fake_run(sp=sp_mode and not pp_mode, exchange=exchange, note="RuntimeError: no peer access")
    egress = None if sp_mode else {"value": 17.2, "unit": "frames/s", "d2h_bytes_per_step": 14376960, "ms_per_step": 696.0}
    jpeg = None if world > 1 else {"value": 17.2, "unit": "frames/s", "d2h_bytes_per_step": 2520135, "ms_per_step": 695.0,
                                   "reference_host_egress_ms_per_step": 68.9}
    fp8 = None if world > 1 else {"value": 22.2, "unit": "frames/s"}
    secondary = None if world == 1 else {"mode": "replicas" if sp_mode else "sp", "scaling": "weak" if sp_mode else "strong",
                                         "value": 34.0, "unit": "frames/s", "ms_per_step": 700.0, "steps": 2}
    cpu = {"value": 0.0078, "unit": "frames/s", "cores": 32, "kind": "port", "sample": "2 layer-forwards"}
    line = bench.assemble_line(args, world, sp_mode, pp_mode, False, main_run, E2E, egress, jpeg, fp8, secondary, cpu)
    json.loads(json.dumps(line))
    for k in REQUIRED:
        assert k in line, k
    assert line["n_gpus"] == world and line["metric"] == "frames_per_second_832x480_4step_t2v"
    streams = 1 if sp_mode else world
    assert line["value"] == pytest.approx(streams * 4 * 12 / 2.772)
    assert line["scaling"] == ("strong" if sp_mode else "weak")
    assert (line["vs_baseline"] is None) == (world > 1)
    assert line["e2e"]["h2d_bytes_per_step"] == 599040 and line["e2e"]["value"] > 0
    assert 0 < line["roofline"]["frac"] <= 1.05 and line["roofline"]["unit"] == "TFLOP/s"
    par = line["config"]["parallelism"]
    if pp_mode:
        assert "configs[2]" in par
    elif sp_mode and exchange == "p2p":
        assert "NVLink peer memory" in par
    elif sp_mode:
        assert "falls back to NCCL" in par and "no peer access" in par
    if world > 1:
        assert secondary["mode"] in line
    else:
        assert "fp8" in line and line["egress_jpeg"]["reference_host_egress_ms_per_step"] == 68.9


def test_reference_arm_line_shape():
    """--impl reference prints the same metric / unit with impl=reference (contract); assembled without running the
    oracle by calling the describe helper on a fabricated time."""
    d = bench.CpuReference.fps_from_layer_time(8.0)
    assert 0 < d < 0.1
