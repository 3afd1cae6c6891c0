"""bench.py contract pieces that can be checked without a GPU: the reference arm prints ONE JSON line with the agreed keys,
and the product arm fails loudly (no JSON, non-zero exit) when there is no device -- there is no CPU fallback."""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


def _run(args, timeout=600):
    return subprocess.run([sys.executable, str(ROOT / "bench.py"), *args], capture_output=True, text=True, timeout=timeout, cwd=ROOT)


def test_reference_arm_prints_one_json_line():
    p = _run(["--impl", "reference", "--steps", "1", "--warmup", "0"])
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "GFLOPS" and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["gpu_launches"] == 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["cpu_baseline"]["value"] == d["value"] == d["e2e"]["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert "4096" in d["metric"] and "sample" in d["cpu_baseline"]


def test_product_arm_fails_loudly_without_a_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    p = _run(["--steps", "1", "--warmup", "0", "--no-cpu"], timeout=300)
    assert p.returncode != 0
    assert not [l for l in p.stdout.splitlines() if l.strip().startswith("{")]


def test_committed_product_line_has_the_contract_keys():
    """The product arm cannot run without a GPU; the line it printed on an H100 (README.md, Results) is committed under
    profiles/ -- check that artefact against the contract, so that a key dropped from bench.py's output is noticed on the CPU
    side too."""
    d = json.loads((ROOT / "profiles" / "h100_bench_n1.json").read_text().strip().splitlines()[-1])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "clocks", "gpu_launches", "sweep", "parity", "abft"):
        assert k in d, k
    assert d["n_gpus"] == 1 and d["steps"] == 20 and d["gpu_launches"] == d["steps"] and d["higher_is_better"] is True
    assert "workload" in d["config"] and "model" not in d["config"]
    r = d["roofline"]
    assert r["bound"] == "tensor" and r["unit"] == "TFLOP/s" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-3 and r["traffic"] > 0
    assert 0.25 < r["frac"] < 1.0
    assert d["cpu_baseline"]["kind"] in ("port", "reference") and d["cpu_baseline"]["cores"] >= 1 and "sample" in d["cpu_baseline"]
    e = d["e2e"]
    assert e["h2d_bytes_per_step"] == 3 * 4 * 4096 * 4096 and e["d2h_bytes_per_step"] == 4 * 4096 * 4096 and 0 < e["value"] < d["value"]
    assert d["clocks"]["sm_mhz"] > 0 and not set(d["clocks"]["reasons"]) & {"hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}
    assert d["parity"]["ok"] and d["parity"]["rel_fro"] < d["parity"]["tolerance"] == 1e-3
    sizes = [row["n"] for row in d["sweep"]]
    assert sizes == list(range(1024, 16385, 1024))
    for row in d["sweep"]:
        assert {"abft_gflops", "plain_gflops", "cublas_tf32_gflops", "overhead_pct_vs_cublas_tf32"} <= set(row)
    # the claims README.md (Results) and DESIGN.md §7 make about this line, as measured on an H100 at 400 W; the design
    # target of <= 10 % over cuBLAS-TF32 is not reached there yet (DESIGN.md §9.1 lists what is left)
    assert d["abft"]["overhead_pct_vs_cublas_tf32"] <= 42.5
    assert all(row["overhead_pct_vs_cublas_tf32"] <= 42.5 for row in d["sweep"] if row["n"] >= 4096)
