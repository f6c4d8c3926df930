"""The three tile schedules of the wgmma GEMM (ab_gemm_bf16), each forced with AB_GEMM_SCHEDULE: ping-pong, the
cooperative 128 x 256 tile, and the staggered one (the cooperative tile with warpgroup 1 kept 1-2 k-blocks behind
warpgroup 0).  Every schedule runs the same seeded cases: tile counts around the SM count (idle CTAs, one tile each,
uneven loads) with a last row block whose second warpgroup has no live row, M / N / K tails with fewer k-blocks than
the lag, no bias / bias / bias + GELU / the fp32 + residual epilogue, bf16 and fp16.  Each output is checked against
an fp32 PyTorch reference, and must be bit-identical across the three schedules (the accumulation order over K does
not depend on the schedule) and across two launches.

The schedule is read once per process, so each one runs in a child process (this file run as a script) that writes
a digest of every output and its worst tolerance excess."""

import hashlib
import json
import math
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
SCHEDULES = ["pingpong", "cooperative", "staggered"]
MODES = {  # bias, gelu, fp32 output + residual
    "none": (False, False, False),
    "bias": (True, False, False),
    "bias_gelu": (True, True, False),
    "bias_res_f32_dual": (True, False, True),
}
TAILS = [
    (131, 520, 64),     # one k-block (fewer than the lag); N tail inside a 64-column box
    (257, 200, 72),     # two k-blocks, the second 8 deep; one 256-column tile with 72 live columns
    (300, 1032, 136),   # three k-blocks; N tail of 8 columns, M tail of 44 rows
    (517, 264, 1024),   # sixteen k-blocks, one 256-column tile with 8 live columns in the second
    (1000, 300, 1096),  # a K tail past 1024
]


def cases(sms: int) -> list[tuple]:
    """(id, m, n, k, dtype, mode); the same list in every process of one machine."""
    out = []
    # N = 768: three 128 x 256 tiles (six 128 x 128 ping-pong tiles) per 128 rows; M = 128 (blocks - 1) + 40, so the
    # last row block has no live row for warpgroup 1 of the 128 x 256 tile.  Tile counts 3, about sms, sms + 3 (some
    # CTAs with two tiles) and about 2 sms + 3 (an odd count on most CTAs).
    for blocks in (1, math.ceil(sms / 3), math.ceil(sms / 3) + 1, math.ceil(2 * sms / 3) + 1):
        for mode in ("none", "bias_gelu"):
            out.append((f"tiles{3 * blocks}-{mode}", 128 * (blocks - 1) + 40, 768, 320, "bf16", mode))
    for m, n, k in TAILS:
        for mode in MODES:
            for dtype in ("bf16", "fp16"):
                out.append((f"{m}x{n}x{k}-{mode}-{dtype}", m, n, k, dtype, mode))
    # many tiles per CTA, the stage-2 width
    out.append(("many-bias_gelu", 2 * 128 * sms + 77, 1536, 1024, "bf16", "bias_gelu"))
    return out


def _digest(t) -> str:
    import torch

    return "" if t is None else hashlib.sha256(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _excess(o, y, tol: float) -> float:
    """Largest |o - y| - tol (1 + |y|); +inf if o holds a NaN (outputs start as NaN)."""
    import torch

    d = ((o.float() - y).abs() - tol * (1.0 + y.abs())).max().item()
    return math.inf if math.isnan(d) or bool(torch.isnan(o).any()) else d


def run_cases(out_path: str) -> None:
    """Child process: every case under the schedule in AB_GEMM_SCHEDULE; writes {id: record} as JSON."""
    import torch

    sys.path.insert(0, str(ROOT))
    from aurora_b200 import cabi

    torch.backends.cuda.matmul.allow_tf32 = False
    dts = {"bf16": torch.bfloat16, "fp16": torch.float16}
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    res = {}
    for cid, m, n, k, dtype, mode in cases(sms):
        bias_on, gelu, f32 = MODES[mode]
        g = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
        dt = dts[dtype]
        a = torch.randn(m, k, device="cuda", generator=g).to(dt)
        w = (torch.randn(n, k, device="cuda", generator=g) / k**0.5).to(dt)
        b = torch.randn(n, device="cuda", generator=g) if bias_on else None
        r = torch.randn(m, n, device="cuda", generator=g) if f32 else None
        outs = []
        for _ in range(2):
            o16 = torch.full((m, n), float("nan"), device="cuda", dtype=dt)
            o32 = torch.full((m, n), float("nan"), device="cuda") if f32 else None
            cabi.gemm(a, w, bias=b, residual=r, out_f32=o32, out_bf16=o16,
                      act=cabi.AB_ACT_GELU_ERF if gelu else cabi.AB_ACT_NONE)
            outs.append((o16, o32))
        torch.cuda.synchronize()
        y = a.float() @ w.float().t()
        if b is not None:
            y += b
        if gelu:
            y = torch.nn.functional.gelu(y)
        y16 = y + r if r is not None else y  # the residual is added to both outputs
        (o16, o32), (p16, p32) = outs
        res[cid] = {
            "hash16": _digest(o16), "hash32": _digest(o32),
            "excess16": _excess(o16, y16, 1e-2), "excess32": _excess(o32, y16, 1e-4) if f32 else -1.0,
            "repeat_same": bool(torch.equal(o16, p16)) and (o32 is None or bool(torch.equal(o32, p32))),
        }
        del a, w, b, r, outs, o16, o32, p16, p32, y, y16
    Path(out_path).write_text(json.dumps(res))


if __name__ == "__main__":
    run_cases(sys.argv[1])
    sys.exit(0)


pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def results(tmp_path_factory) -> dict:
    """{schedule: {case id: record}}, one child process per schedule."""
    out = {}
    for sched in SCHEDULES:
        path = tmp_path_factory.mktemp("sched") / f"{sched}.json"
        env = {**os.environ, "AB_GEMM_SCHEDULE": sched}
        subprocess.run([sys.executable, __file__, str(path)], check=True, env=env, cwd=ROOT, timeout=900)
        out[sched] = json.loads(path.read_text())
    return out


def _ids() -> list[str]:
    import torch

    return [c[0] for c in cases(torch.cuda.get_device_properties(0).multi_processor_count)] \
        if torch.cuda.is_available() else [c[0] for c in cases(132)]


@pytest.mark.parametrize("sched", SCHEDULES)
def test_every_case_matches_the_fp32_reference(results, sched):
    bad = {cid: (r["excess16"], r["excess32"]) for cid, r in results[sched].items()
           if r["excess16"] > 0 or r["excess32"] > 0}
    assert not bad, bad
    assert sorted(results[sched]) == sorted(_ids())


@pytest.mark.parametrize("sched", SCHEDULES)
def test_two_launches_are_bit_identical(results, sched):
    assert all(r["repeat_same"] for r in results[sched].values()), \
        [cid for cid, r in results[sched].items() if not r["repeat_same"]]


def test_schedules_are_bit_identical(results):
    base = results["pingpong"]
    for sched in SCHEDULES[1:]:
        diff = [cid for cid, r in results[sched].items()
                if (r["hash16"], r["hash32"]) != (base[cid]["hash16"], base[cid]["hash32"])]
        assert not diff, (sched, diff)


def test_unknown_schedule_is_refused():
    code = ("import sys, torch; sys.path.insert(0, '.'); from aurora_b200 import cabi\n"
            "a = torch.zeros(128, 64, device='cuda', dtype=torch.bfloat16); o = torch.empty(128, 256, device='cuda', "
            "dtype=torch.bfloat16)\n"
            "try:\n    cabi.gemm(a, torch.zeros(256, 64, device='cuda', dtype=torch.bfloat16), out_bf16=o)\n"
            "except Exception as e:\n    print('refused', e); sys.exit(0)\nsys.exit(1)")
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, "AB_GEMM_SCHEDULE": "fastest"}, cwd=ROOT,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "AB_GEMM_SCHEDULE" in r.stdout, r.stdout + r.stderr
