"""Cost of scoring every step of a roll-out of the 1.3 B model at 0.25 degrees (721 x 1440, 13 levels) against an
analysis and a climatology.

Seeded random weights and inputs (bench.py's recipe); the "analysis" and the climatology are two more seeded batches
on the same grid.  After a warm-up, three arms alternate, each an 8-step `aurora_b200.rollout`:

  rollout     the roll-out alone;
  scorer      plus `aurora_b200.Scorer`, with the truth and climatology resident on the GPU;
  host        plus the reference notebooks' workflow: `pred.to("cpu")`, then a numpy float64 pass over every plane
              (the same definitions as `Scorer`).

The scores of the two scoring arms are then compared (to 1e-9 of rmse, mae, mae and 1), the device-to-host bytes of one step of each
are profiled, and the scoring kernels' own time is taken with CUDA events over many calls on one step's fields and
set against the HBM bound of the bytes they read (the H100 SXM data-sheet 3.35 TB/s).  Prints the median and range
of ms per step of each arm, those figures, the card and its power limit as one JSON line.

    python tools/score_rollout.py [--rounds 5] [--steps 8]
"""

from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, limit = (out[0].split(", ") + ["?"])[:2] if out else (torch.cuda.get_device_name(), "not read")
    return {"name": name, "power_limit": limit}


def d2h_bytes(fn) -> int:
    """Device-to-host bytes of `fn()` as torch.profiler records them."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = Path(d) / "trace.json"
        prof.export_chrome_trace(str(path))
        events = json.loads(path.read_text())["traceEvents"]
    return sum(int(e.get("args", {}).get("bytes", 0)) for e in events
               if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", ""))


def host_scores(pred, truth: dict, clim: dict, w: np.ndarray) -> list[tuple]:
    """The reference workflow on a host copy of the prediction: (variable, level index, rmse, bias, mae, acc, count)
    per plane, in float64 with the definitions of `aurora_b200.Scorer`."""
    pred = pred.to("cpu")
    out = []
    h = len(w)
    for group in ("surf_vars", "atmos_vars"):
        for k, v in getattr(pred, group).items():
            p = v[0, -1].numpy()
            p = p[None] if p.ndim == 2 else p
            for lv in range(p.shape[0]):
                pp, tt, cc = (a[lv, :h].astype(np.float64) for a in (p, truth[k], clim[k]))
                ok = ~(np.isnan(pp) | np.isnan(tt) | np.isnan(cc))
                wv = np.where(ok, w[:, None], 0.0)
                d = np.where(ok, pp - tt, 0.0)
                af, ao = np.where(ok, pp - cc, 0.0), np.where(ok, tt - cc, 0.0)
                big_w = wv.sum()
                acc = (wv * af * ao).sum() / np.sqrt((wv * af * af).sum() * (wv * ao * ao).sum())
                out.append((k, lv, np.sqrt((wv * d * d).sum() / big_w), (wv * d).sum() / big_w,
                            (wv * np.abs(d)).sum() / big_w, acc, int(ok.sum())))
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--kernel-calls", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_rollout.py needs a CUDA device")

    import aurora_b200 as ab
    from aurora_b200 import cabi
    from aurora_b200.batch import Batch, Metadata
    from aurora_b200.scorer import _field
    from bench import LEVELS13, make_host_batch, randomise_parameters_

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = ab.Aurora(_init="empty", autocast=True).to(dev).eval()
    randomise_parameters_(model, seed=0)
    batch = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=0)
    last = lambda b: {k: v[0, -1].reshape(-1, *v.shape[-2:]).numpy()  # noqa: E731
                      for d in (b.surf_vars, b.atmos_vars) for k, v in d.items()}
    truth_host = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=1)
    clim_host = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=2)
    truth_np, clim_np = last(truth_host), last(clim_host)
    truth_dev, clim_dev = truth_host.to(dev), clim_host.to(dev)
    weights = np.cos(np.deg2rad(batch.metadata.lat[:720].double().numpy()))

    def truth_at(pred) -> Batch:  # the same analysis fields, stamped with the prediction's time
        md = truth_dev.metadata
        return Batch(truth_dev.surf_vars, truth_dev.static_vars, truth_dev.atmos_vars,
                     Metadata.derived(md.lat, md.lon, pred.metadata.time, md.atmos_levels))

    def arm(kind: str, keep: dict | None = None):
        scorer = ab.Scorer(climatology=clim_dev) if kind == "scorer" else None
        host = []
        torch.cuda.synchronize()
        start = time.perf_counter()
        with torch.inference_mode():
            for pred in ab.rollout(model, batch, steps=args.steps):
                if kind == "scorer":
                    scorer.step(pred, truth_at(pred))
                elif kind == "host":
                    host += host_scores(pred, truth_np, clim_np, weights)
            table = scorer.results() if scorer is not None else None
        torch.cuda.synchronize()
        ms = 1000.0 * (time.perf_counter() - start) / args.steps
        if keep is not None:
            keep[kind] = table if kind == "scorer" else host
        return ms

    kinds = ("rollout", "scorer", "host")
    results: dict = {}
    for kind in kinds:  # warm-up: captures every graph signature, loads the library
        arm(kind, results)
    times = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for kind in kinds:
            times[kind].append(arm(kind))

    # the two scoring arms agree
    table, host = results["scorer"], results["host"]
    assert len(table) == len(host), (len(table), len(host))
    got = table[["rmse", "bias", "mae", "acc"]].to_numpy()
    want = np.array([r[2:6] for r in host])
    scale = np.stack([want[:, 0], want[:, 2], want[:, 2], np.ones(len(want))], -1)  # bias and acc may be ~0
    worst = float(np.max(np.abs(got - want) / scale))
    assert worst < 1e-9 and (table["count"].to_numpy() == np.array([r[6] for r in host])).all(), worst

    # device-to-host bytes of one step of each scoring arm
    with torch.inference_mode():
        pred = next(iter(ab.rollout(model, batch, steps=1)))
        scorer = ab.Scorer(climatology=clim_dev)
        scorer.step(pred, truth_at(pred))
        bytes_scorer = d2h_bytes(lambda: scorer.step(pred, truth_at(pred)))
        bytes_results = d2h_bytes(scorer.results)
        bytes_host = d2h_bytes(lambda: host_scores(pred, truth_np, clim_np, weights))

        # the kernels alone: one call = the 9 fields (69 planes) of a step
        h = pred.metadata.lat.numel()
        fields, n_planes = [], 0
        for group in ("surf_vars", "atmos_vars"):
            for k, v in getattr(pred, group).items():
                t, c = getattr(truth_dev, group)[k][0, -1], getattr(clim_dev, group)[k][0, -1]
                fields.append(_field(v[0, -1], t[..., :h, :], c[..., :h, :]))
                n_planes += fields[-1].levels
        w_dev = torch.from_numpy(weights).to(dev)
        sums = torch.empty(n_planes, cabi.AB_SCORE_SUMS, dtype=torch.float64, device=dev)
        ws = torch.empty(cabi.score_workspace_bytes(fields), dtype=torch.uint8, device=dev)
        for _ in range(5):
            cabi.score_fields(fields, w_dev, sums, ws)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.kernel_calls):
            cabi.score_fields(fields, w_dev, sums, ws)
        e1.record()
        e1.synchronize()
        kernel_ms = e0.elapsed_time(e1) / args.kernel_calls
    read_bytes = 3 * n_planes * h * pred.metadata.lon.numel() * 4

    med = {k: statistics.median(v) for k, v in times.items()}
    line = {
        "card": card(), "grid": "721x1440 (model input), 13 levels; scored 720x1440, 69 planes", "steps_per_arm": args.steps,
        "rounds": args.rounds,
        "ms_per_step": {"median": med, "min": {k: min(v) for k, v in times.items()},
                        "max": {k: max(v) for k, v in times.items()}, "all": times},
        "scoring_ms_per_step": {"scorer": med["scorer"] - med["rollout"], "host": med["host"] - med["rollout"]},
        "d2h_bytes": {"scorer_step": bytes_scorer, "scorer_results_after_one_step": bytes_results,
                      "host_step": bytes_host},
        "kernel": {"ms_per_call": kernel_ms, "bytes_read": read_bytes,
                   "hbm_bound_ms": 1000.0 * read_bytes / HBM_BYTES_PER_S,
                   "share_of_hbm_bound": read_bytes / HBM_BYTES_PER_S / (kernel_ms / 1000.0)},
        "scores_agree_rel": worst,
    }
    print(json.dumps(line, default=float), flush=True)


if __name__ == "__main__":
    main()
