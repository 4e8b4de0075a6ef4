"""bench.py's output contract (one JSON line and its keys). The reference arm runs anywhere (CPU); this repo's arm
needs an H100."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
             "vs_baseline", "dtype", "data", "config", "e2e"}


def _run(args, timeout=900):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + args, capture_output=True, text=True,
                         timeout=timeout, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, out.stdout
    return json.loads(lines[0])


def test_reference_arm_line():
    """`--impl reference` runs the UNMODIFIED reference module from oracle/_ref (oracle/fetch_ref.py, run by build())
    when it is there, the oracle port otherwise; a timed step is the full per-rank chunk, so steps x ms_per_step is the
    time the arm really spent."""
    have_ref = os.path.exists(os.path.join(ROOT, "oracle", "_ref", "distributed_sigmoid_loss.py"))
    d = _run(["--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "1", "--batch", "256", "--dim", "64"])
    assert d["impl"] == "reference" and BASE_KEYS <= set(d)
    assert d["metric"] == "image-text pairs/sec" and d["unit"] == "pairs/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["gpu_launches"] == 0 and d["steps"] == 2 and d["warmup"] == 1
    cb = d["cpu_baseline"]
    assert cb["kind"] == ("reference" if have_ref else "port")
    assert cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"] and "model" not in d["config"]
    # N = 1: the measured step IS the whole job
    assert abs(d["value"] - 256 / (d["ms_per_step"] * 1e-3)) <= 1e-6 * d["value"]
    # loss of the reference on the bench inputs: the product arm must print the same number (bench.py `loss`)
    assert 5.0 < d["loss"] < 20.0


def test_reference_arm_extrapolates_at_n_gt_1():
    d = _run(["--impl", "reference", "--gpus", "4", "--steps", "1", "--warmup", "0", "--batch", "128", "--dim", "64"])
    # one timed step is still ONE (B x B) chunk; the whole job is W ranks x W chunks of it on this host
    assert abs(d["extrapolated_job_step_ms"] - 16 * d["ms_per_step"]) <= 1e-9 * d["ms_per_step"] * 16
    assert abs(d["value"] - 4 * 128 / (d["extrapolated_job_step_ms"] * 1e-3)) <= 1e-6 * d["value"]
    assert "extrapolated" in d["cpu_baseline"]["sample"]


@pytest.mark.gpu
def test_product_arm_line():
    d = _run(["--gpus", "1", "--steps", "3", "--warmup", "3", "--batch", "2048", "--dim", "256", "--sustain-ms", "50",
              "--cpu-steps", "1"])
    assert "impl" not in d and BASE_KEYS | {"gpu_launches", "clocks", "roofline", "cpu_baseline", "burst", "parity",
                                            "per_rank"} <= set(d)
    assert d["n_gpus"] == 1 and d["steps"] == 3 and d["warmup"] >= 3 and d["dtype"] == "bf16"
    assert d["gpu_launches"] == 2 * 3          # one loss kernel + one gradient kernel per step
    r = d["roofline"]
    assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and 0 < r["frac"] < 1.2 and r["launches_timed"] == 3
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] == 2 * 2048 * 256 * 2 and e["d2h_bytes_per_step"] == 12 and e["value"] > 0
    assert e["first_steps_ms_per_step"] > 0 and "sustained" in e["api"]   # the headline e2e figure is the sustained one
    g = e["with_grads"]
    assert g["d2h_bytes_per_step"] == 2 * 2048 * 256 * 2 + 12 and g["value"] > 0 and g["loss"] == e["loss"]
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["value"] > 0
    assert d["clocks"]["samples"] >= 1
    par = d["parity"]
    assert par["pass"] is True and par["shape"] == [2048, 768]
    assert all(v <= 1e-3 for v in par["fused_fp32"].values())


@pytest.mark.gpu
def test_dump_outputs_of_the_timed_path(tmp_path):
    """--dump-outputs writes the last timed step's five outputs as float32 .npy files, at most 64 MB in all; the inputs
    are fixed by the arguments, so a second run computes the same outputs."""
    import numpy as np

    names = ("loss", "dimg", "dtxt", "dt_prime", "dbias")
    runs = []
    for i in range(2):
        out = tmp_path / f"run{i}"
        d = _run(["--gpus", "1", "--steps", "2", "--warmup", "1", "--batch", "2048", "--dim", "256", "--sustain-ms", "20",
                  "--no-cpu-baseline", "--no-parity", "--dump-outputs", str(out)])
        assert d["steps"] == 2
        assert sorted(p.name for p in out.iterdir()) == sorted(n + ".npy" for n in names)
        assert sum(p.stat().st_size for p in out.iterdir()) <= 64 << 20
        arrays = {n: np.load(out / (n + ".npy")) for n in names}
        assert all(a.dtype == np.float32 for a in arrays.values())
        assert arrays["dimg"].shape == arrays["dtxt"].shape == (2048, 256) and arrays["loss"].shape == (1,)
        assert np.isfinite(arrays["loss"]).all() and abs(float(arrays["loss"][0]) - d["loss"]) <= 1e-6 * abs(d["loss"])
        runs.append(arrays)
    for n in names:
        np.testing.assert_allclose(runs[1][n], runs[0][n], rtol=1e-6, atol=0)
    with pytest.raises(AssertionError):
        _run(["--impl", "reference", "--steps", "1", "--warmup", "0", "--batch", "64", "--dim", "64",
              "--dump-outputs", str(tmp_path / "ref")])
