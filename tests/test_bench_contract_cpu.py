"""bench.py contract checks that need no GPU: the reference arm (the unmodified reference from oracle/_ref on the host
cores) prints ONE JSON line with the keys its consumers read, on rank 0 only."""

import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def _run(args, env=None):
    r = subprocess.run([sys.executable, str(ROOT / "bench.py"), *args], capture_output=True, text=True, timeout=600,
                       env={**os.environ, **(env or {})}, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    return [ln for ln in r.stdout.splitlines() if ln.startswith("{")]


def test_reference_arm_prints_one_contract_line():
    lines = _run(["--impl", "reference", "--workload", "aurora-small-17x32x4L", "--steps", "2", "--warmup", "1"])
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "forecast-steps/sec" and d["unit"] == "forecast-steps/s"
    assert d["higher_is_better"] is True and d["n_gpus"] == 1 and d["steps"] == 2 and d["warmup"] == 1
    # `ms_per_step` is the wall time of one timed (bounded-sample) step — K of them fit in the run — and a whole forecast
    # step is `sample_scale` of them, the factor measured against ONE complete reference forward in the same run
    assert d["value"] > 0 and abs(d["ms_per_whole_step"] - 1000.0 / d["value"]) < 1e-6 * d["ms_per_whole_step"]
    assert abs(d["ms_per_step"] * d["sample_scale"] / d["ms_per_whole_step"] - 1.0) < 1e-6
    assert d["config"]["workload"] == "aurora-small-17x32x4L" and d["config"]["parallelism"] == "single GPU"
    cb = d["cpu_baseline"]
    assert cb["kind"] == "reference" and cb["cores"] >= 1 and cb["value"] == d["value"] and "sample" in cb
    assert cb["complete_forward_seconds"] > 0 and cb["samples"] == 2
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["gpu_launches"] == 0


def test_reference_arm_is_silent_on_other_ranks():
    assert _run(["--impl", "reference", "--workload", "aurora-small-17x32x4L", "--steps", "1", "--warmup", "1", "--gpus", "2"],
                env={"RANK": "1", "WORLD_SIZE": "2", "LOCAL_RANK": "1"}) == []


def test_both_arms_report_the_same_config_and_parallelism():
    """`config` is computed from the command line alone, so the driver sees identical dicts from `--impl ours` and
    `--impl reference`; `auto` shards a forecast by latitude whenever the grid allows and falls back to replicas otherwise."""
    sys.path.insert(0, str(ROOT))
    import bench

    for wl in bench.WORKLOADS:
        for n in (1, 2, 4, 8):
            assert bench.workload_config(wl, n, "auto") == bench.workload_config(wl, n, "auto")
    assert bench.resolve_parallelism("aurora-0.25deg-721x1440x13L", 8, "auto") == "latshard"
    assert bench.resolve_parallelism("aurora-0.25deg-721x1440x13L", 1, "auto") == "single GPU"
    assert bench.resolve_parallelism("aurora-0.25deg-721x1440x13L", 8, "replicas") == "replicas"
    # 150 token rows: an odd 2x2 merge inside the U-Net -> cannot be banded -> replicas (explicit `latshard` raises)
    assert bench.resolve_parallelism("aurora-airpollution-0.4deg-451x900x13L", 8, "auto") == "replicas"
    import pytest

    with pytest.raises(NotImplementedError):
        bench.resolve_parallelism("aurora-airpollution-0.4deg-451x900x13L", 8, "latshard")
    cfg = bench.workload_config("aurora-0.25deg-721x1440x13L", 8, "auto")
    assert cfg["workload"] == "aurora-0.25deg-721x1440x13L" and "latitude-sharded over 8" in cfg["parallelism"]


def test_reference_copy_matches_its_manifest():
    """oracle/_ref (the copy of the unmodified reference made by oracle/build_ref.py) is byte-for-byte what its manifest
    says, and — where the checkout it was made from is present — what that checkout holds."""
    import hashlib

    sys.path.insert(0, str(ROOT))
    from oracle import build_ref

    ref = ROOT / "oracle" / "_ref"
    if not (ref / "MANIFEST.json").exists():
        import pytest

        pytest.skip("oracle/_ref not built")
    man = json.loads((ref / "MANIFEST.json").read_text())
    assert man["files"], "empty manifest"
    for rel, digest in man["files"].items():
        assert hashlib.sha256((ref / rel).read_bytes()).hexdigest() == digest, rel
        src = build_ref.REFERENCE / rel
        if src.exists():
            assert hashlib.sha256(src.read_bytes()).hexdigest() == digest, rel
