"""Per-shape timing of the wgmma GEMM (ab_gemm_bf16) on the shapes one forward step of a bench.py workload runs.

    python tools/gemm_shapes.py [--workload NAME] [--iters N]

1. Records every `cabi.gemm` call of one eager forward (the per-op path of bench.py's instrumented step): M, N, K,
   operand dtype, bias, activation and outputs.
2. Times each distinct shape in isolation on fresh seeded tensors (warm-up, then `--iters` launches between CUDA
   events): one JSON line per shape with launches per step, ms per launch, TFLOP/s and ms per step.
3. K-scan: the M x N of the bf16 shapes of the two largest-M Swin stages, also at 2K and 4K (fc1 with and without
   GELU).  A least-squares fit of t = t0 + c * K separates the fixed cost (epilogue, pipeline fill / drain) from the
   main-loop rate; `fixed_share` is t0 over the time at the shape's own K.
4. The card: name, power limit and max SM clock, read in the same run.

AB_GEMM_SCHEDULE=pingpong|cooperative|staggered in the environment times every N > 128 shape on that schedule.

Writes nothing; needs a GPU.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from aurora_b200 import cabi  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return {"kind": "card", "name": name, "power_limit": power, "max_sm_clock": clock}


def record_shapes(workload: str) -> dict:
    """{shape key: launches} of one eager forward of `workload`, as bench.py builds it."""
    import aurora_b200 as ab

    cls, h, w, levels = bench.WORKLOADS[workload]
    dev = torch.device("cuda")
    model = getattr(ab, cls)(_init="empty", autocast=True).to(dev).eval()
    bench.randomise_parameters_(model, seed=0)
    batch = bench.make_host_batch(model.config, h, w, levels, pinned=False, seed=0).to(dev)
    model.use_cuda_graph = False
    model.forward(batch)  # warm-up: packs weights, allocates the workspace

    counts: dict = {}
    inner = cabi.gemm

    def spy(a, wt, *, bias=None, residual=None, out_f32=None, out_bf16=None, act=cabi.AB_ACT_NONE, peer_push=None):
        key = (a.shape[0], wt.shape[0], a.shape[1], str(a.dtype).removeprefix("torch."), bias is not None, int(act),
               out_f32 is not None, None if out_bf16 is None else str(out_bf16.dtype).removeprefix("torch."),
               residual is not None)
        counts[key] = counts.get(key, 0) + 1
        return inner(a, wt, bias=bias, residual=residual, out_f32=out_f32, out_bf16=out_bf16, act=act,
                     peer_push=peer_push)

    cabi.gemm, cabi.PROFILE = spy, {}  # PROFILE: the per-op path of bench.py's instrumented step
    try:
        model.forward(batch)
        torch.cuda.synchronize()
    finally:
        cabi.gemm, cabi.PROFILE = inner, None
    del model, batch
    torch.cuda.empty_cache()
    return counts


def time_shape(key, iters: int) -> float:
    """ms per launch of one shape on fresh seeded operands."""
    m, n, k, dt, has_bias, act, f32, out16, has_res = key
    g = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
    dtype = getattr(torch, dt)
    a = torch.randn(m, k, device="cuda", generator=g).to(dtype)
    wt = (torch.randn(n, k, device="cuda", generator=g) / k**0.5).to(dtype)
    bias = torch.randn(n, device="cuda", generator=g) if has_bias else None
    res = torch.randn(m, n, device="cuda", generator=g) if has_res else None
    o32 = torch.empty(m, n, device="cuda") if f32 else None
    o16 = torch.empty(m, n, device="cuda", dtype=getattr(torch, out16)) if out16 else None

    def run():
        cabi.gemm(a, wt, bias=bias, residual=res, out_f32=o32, out_bf16=o16, act=act)

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def describe(key) -> dict:
    m, n, k, dt, has_bias, act, f32, out16, has_res = key
    return {"m": m, "n": n, "k": k, "dtype": dt, "bias": has_bias, "gelu": act == cabi.AB_ACT_GELU_ERF,
            "out_f32": f32, "out16": out16, "residual": has_res}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default=bench.DEFAULT_WORKLOAD, choices=sorted(bench.WORKLOADS))
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/gemm_shapes.py needs a CUDA device")
    print(json.dumps(card()), flush=True)

    counts = record_shapes(args.workload)
    total_ms = total_tflop = 0.0
    for key in sorted(counts, key=lambda q: -q[0] * q[1] * q[2] * counts[q]):
        ms = time_shape(key, args.iters)
        flop = 2.0 * key[0] * key[1] * key[2]
        total_ms += ms * counts[key]
        total_tflop += flop * counts[key] / 1e12
        print(json.dumps({"kind": "shape", **describe(key), "launches_per_step": counts[key], "ms_per_launch": round(ms, 4),
                          "tflops": round(flop / ms / 1e9, 1), "ms_per_step": round(ms * counts[key], 3)}), flush=True)
    print(json.dumps({"kind": "total", "distinct_shapes": len(counts), "launches_per_step": sum(counts.values()),
                      "tflop_per_step": round(total_tflop, 2), "ms_per_step": round(total_ms, 2),
                      "tflops": round(total_tflop / total_ms * 1e3, 1)}), flush=True)

    bf16_m = sorted({q[0] for q in counts if q[3] == "bfloat16"}, reverse=True)[:2]
    scan = sorted({q for q in counts if q[3] == "bfloat16" and q[0] in bf16_m}, key=lambda q: (-q[0], str(q)))
    for key in scan:
        variants = [key] + ([key[:5] + (cabi.AB_ACT_NONE,) + key[6:]] if key[5] == cabi.AB_ACT_GELU_ERF else [])
        for v in variants:
            ks = [v[2], 2 * v[2], 4 * v[2]]
            ts = [time_shape((v[0], v[1], kk) + v[3:], args.iters) for kk in ks]
            mk, mt = sum(ks) / 3, sum(ts) / 3
            c = sum((x - mk) * (y - mt) for x, y in zip(ks, ts)) / sum((x - mk) ** 2 for x in ks)
            t0 = mt - c * mk
            print(json.dumps({"kind": "kscan", **describe(v), "k_values": ks, "ms": [round(t, 4) for t in ts],
                              "intercept_ms": round(t0, 4), "fixed_share": round(t0 / ts[0], 3),
                              "mainloop_tflops": round(2.0 * v[0] * v[1] / c / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
