"""Cost of scoring ensembles with `aurora_b200.EnsembleScorer` at 0.25 degrees (720 x 1440 scored, 69 planes).

Kernel arm: synthetic seeded members, truth and climatology resident on the GPU, no model.  For each M the 9 fields
of one step (the 1.3 B model's 4 surface and 5 x 13 atmospheric planes) go through `ab_ensemble_score_fields`;
CUDA events over `--kernel-calls` calls after a warm-up give ms per call, set against the HBM bound of the
(M + 2) x 286 MB the call reads at the H100 SXM data-sheet 3.35 TB/s.

Rollout arm: the 1.3 B model with bench.py's seeded weights and inputs, M = 8 members (seeded perturbations of one
initial state), lock-step `rollout`s of `--steps` steps, the analysis and climatology two more seeded batches.  After a
warm-up, three arms alternate:

  rollout     the M roll-outs alone;
  ensemble    plus `EnsembleScorer`, truth and climatology resident on the GPU;
  host        plus the host workflow: `pred.to("cpu")` of every member, then a numpy float64 pass over every plane
              with the same definitions (the CRPS spread term from the sorted members).

The host arm runs `--host-rounds` rounds (fewer than the others: it is slow).  Prints one JSON line: the card and its
power limit, the kernel arm per M, the median and range of ms per step of each rollout arm, the device-to-host bytes
of one step of each scoring arm and how far the two scoring arms' tables agree.

    python tools/score_ensemble.py [--rounds 5] [--host-rounds 2] [--steps 8] [--members 8] [--skip-kernel]
                                   [--skip-rollout]
"""

from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from score_rollout import HBM_BYTES_PER_S, card, d2h_bytes  # noqa: E402

KERNEL_MEMBERS = (2, 8, 16, 32, 50, 64)
COLS = ("ens_rmse", "ens_bias", "spread", "crps_skill", "crps_spread", "acc")


def kernel_arm(calls: int) -> dict:
    from aurora_b200 import cabi
    from aurora_b200.scorer import _ensemble_field

    dev = torch.device("cuda", 0)
    h, w, levels = 720, 1440, [1] * 4 + [13] * 5
    g = torch.Generator(device=dev).manual_seed(0)
    field = lambda n, lv: (280.0 + 3.0 * torch.randn(n, lv, h, w, generator=g, device=dev))  # noqa: E731
    members = [field(max(KERNEL_MEMBERS), lv) for lv in levels]
    truth, clim = [field(1, lv)[0] for lv in levels], [field(1, lv)[0] for lv in levels]
    weights = torch.from_numpy(np.cos(np.deg2rad(np.linspace(90, -90, 721)[:720]))).to(dev)
    planes = sum(levels)
    out = {}
    for m in KERNEL_MEMBERS:
        fields = [_ensemble_field([x[k] for k in range(m)], t, c) for x, t, c in zip(members, truth, clim)]
        sums = torch.empty(planes, cabi.AB_ENS_SUMS, dtype=torch.float64, device=dev)
        ws = torch.empty(cabi.ensemble_score_workspace_bytes(fields), dtype=torch.uint8, device=dev)
        for _ in range(5):
            cabi.ensemble_score_fields(fields, weights, sums, ws)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            cabi.ensemble_score_fields(fields, weights, sums, ws)
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / calls
        read = (m + 2) * planes * h * w * 4
        out[m] = {"ms_per_call": ms, "bytes_read": read, "hbm_bound_ms": 1000.0 * read / HBM_BYTES_PER_S,
                  "share_of_hbm_bound": read / HBM_BYTES_PER_S / (ms / 1000.0)}
    del members, truth, clim
    torch.cuda.empty_cache()
    return out


def host_scores(members, truth: dict, clim: dict, w: np.ndarray) -> list[tuple]:
    """The host workflow on copies of the members: (variable, level index, *COLS, count) per plane, float64."""
    host = [b.to("cpu") for b in members]
    m, h = len(host), len(w)
    out = []
    for group in ("surf_vars", "atmos_vars"):
        for k in getattr(host[0], group):
            x = np.stack([getattr(b, group)[k][0, -1].numpy() for b in host])
            x = x[:, None] if x.ndim == 3 else x
            for lv in range(x.shape[1]):
                xs = np.sort(x[:, lv].astype(np.float64), axis=0)
                y, c = truth[k][lv, :h].astype(np.float64), clim[k][lv, :h].astype(np.float64)
                ok = ~(np.isnan(xs).any(0) | np.isnan(y) | np.isnan(c))
                wv = np.where(ok, w[:, None], 0.0)
                big_w = wv.sum()
                xm = xs.mean(0)
                d = np.where(ok, xm - y, 0.0)
                var = np.where(ok, xs.var(0, ddof=1), 0.0)
                skill = np.where(ok, np.abs(xs - y).mean(0), 0.0)
                coef = (2.0 * np.arange(1, m + 1) - m - 1)[:, None, None]
                pair = np.where(ok, 2.0 * (coef * xs).sum(0) / (m * (m - 1)), 0.0)
                af, ao = np.where(ok, xm - c, 0.0), np.where(ok, y - c, 0.0)
                acc = (wv * af * ao).sum() / np.sqrt((wv * af * af).sum() * (wv * ao * ao).sum())
                out.append((k, lv, np.sqrt((wv * d * d).sum() / big_w), (wv * d).sum() / big_w,
                            np.sqrt((wv * var).sum() / big_w), (wv * skill).sum() / big_w, (wv * pair).sum() / big_w,
                            acc, int(ok.sum())))
    return out


def rollout_arm(args) -> dict:
    import aurora_b200 as ab
    from aurora_b200.batch import Batch, Metadata
    from bench import LEVELS13, make_host_batch, randomise_parameters_

    dev = torch.device("cuda", 0)
    model = ab.Aurora(_init="empty", autocast=True).to(dev).eval()
    randomise_parameters_(model, seed=0)
    batch = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=0)
    gen = torch.Generator().manual_seed(1)

    def perturbed() -> Batch:
        noise = lambda d: {k: (v + 0.01 * v.std() * torch.randn(v.shape, generator=gen)).pin_memory()  # noqa: E731
                           for k, v in d.items()}
        return Batch(noise(batch.surf_vars), batch.static_vars, noise(batch.atmos_vars), batch.metadata)

    starts = [perturbed() for _ in range(args.members)]
    last = lambda b: {k: v[0, -1].reshape(-1, *v.shape[-2:]).numpy()  # noqa: E731
                      for d in (b.surf_vars, b.atmos_vars) for k, v in d.items()}
    truth_host = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=1)
    clim_host = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=2)
    truth_np, clim_np = last(truth_host), last(clim_host)
    truth_dev, clim_dev = truth_host.to(dev), clim_host.to(dev)
    weights = np.cos(np.deg2rad(batch.metadata.lat[:720].double().numpy()))

    def truth_at(pred) -> Batch:
        md = truth_dev.metadata
        return Batch(truth_dev.surf_vars, truth_dev.static_vars, truth_dev.atmos_vars,
                     Metadata.derived(md.lat, md.lon, pred.metadata.time, md.atmos_levels))

    def arm(kind: str, keep: dict | None = None) -> float:
        scorer = ab.EnsembleScorer(climatology=clim_dev) if kind == "ensemble" else None
        host = []
        torch.cuda.synchronize()
        start = time.perf_counter()
        with torch.inference_mode():
            for members in zip(*(ab.rollout(model, b, steps=args.steps) for b in starts)):
                if kind == "ensemble":
                    scorer.step(members, truth_at(members[0]))
                elif kind == "host":
                    host += host_scores(members, truth_np, clim_np, weights)
            table = scorer.results() if scorer is not None else None
        torch.cuda.synchronize()
        if keep is not None:
            keep[kind] = table if kind == "ensemble" else host
        ms = 1000.0 * (time.perf_counter() - start) / args.steps
        print(f"{kind}: {ms:.1f} ms per step", file=sys.stderr, flush=True)
        return ms

    results: dict = {}
    for kind in ("rollout", "ensemble"):  # warm-up: captures every graph signature, loads the library
        arm(kind, results)
    times = {"rollout": [], "ensemble": [], "host": []}
    for r in range(args.rounds):
        for kind in ("rollout", "ensemble", "host"):
            if kind == "host" and r >= args.host_rounds:
                continue
            times[kind].append(arm(kind, results if kind == "host" else None))

    table, host = results["ensemble"], results["host"]
    assert len(table) == len(host), (len(table), len(host))
    got = table[list(COLS)].to_numpy()
    want = np.array([r[2:8] for r in host])
    scale = np.stack([want[:, 0], want[:, 0], want[:, 2], want[:, 3], want[:, 4], np.ones(len(want))], -1)
    worst = float(np.max(np.abs(got - want) / scale))
    counts_agree = bool((table["count"].to_numpy() == np.array([r[8] for r in host])).all())

    with torch.inference_mode():
        members = [next(iter(ab.rollout(model, b, steps=1))) for b in starts]
        scorer = ab.EnsembleScorer(climatology=clim_dev)
        scorer.step(members, truth_at(members[0]))
        bytes_scorer = d2h_bytes(lambda: scorer.step(members, truth_at(members[0])))
        bytes_results = d2h_bytes(scorer.results)
        bytes_host = d2h_bytes(lambda: host_scores(members, truth_np, clim_np, weights))
    med = {k: statistics.median(v) for k, v in times.items()}
    return {
        "members": args.members, "steps_per_arm": args.steps, "rounds": {k: len(v) for k, v in times.items()},
        "ms_per_step": {"median": med, "min": {k: min(v) for k, v in times.items()},
                        "max": {k: max(v) for k, v in times.items()}, "all": times},
        "scoring_ms_per_step": {"ensemble": med["ensemble"] - med["rollout"], "host": med["host"] - med["rollout"]},
        "d2h_bytes": {"ensemble_step": bytes_scorer, "ensemble_results_after_one_step": bytes_results,
                      "host_step": bytes_host},
        "tables_agree_rel": worst, "counts_agree": counts_agree,
    }


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--host-rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--members", type=int, default=8)
    ap.add_argument("--kernel-calls", type=int, default=50)
    ap.add_argument("--skip-rollout", action="store_true")
    ap.add_argument("--skip-kernel", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("score_ensemble.py needs a CUDA device")
    torch.cuda.set_device(0)
    line = {"card": card(), "grid": "720x1440 scored, 69 planes (4 surface + 5 x 13 levels)"}
    if not args.skip_kernel:
        line["kernel"] = kernel_arm(args.kernel_calls)
        print(json.dumps(line["kernel"], default=float), file=sys.stderr, flush=True)
    if not args.skip_rollout:
        line["rollout"] = rollout_arm(args)
    print(json.dumps(line, default=float), flush=True)


if __name__ == "__main__":
    main()
