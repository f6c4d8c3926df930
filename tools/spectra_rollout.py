"""Cost of the zonal power spectra of every step of a roll-out of the 1.3 B model at 0.25 degrees (721 x 1440,
13 levels), and of the spectrum kernels alone at 0.25 and 0.1 degrees.

Seeded random weights and inputs (bench.py's recipe).  After a warm-up, three arms alternate, each an 8-step
`aurora_b200.rollout`:

  rollout     the roll-out alone;
  spectra     plus `aurora_b200.ZonalSpectra` on each prediction (bands global, tropics and nh);
  host        plus `pred.to("cpu")` and `numpy.fft.rfft` over every row of every plane, with the same definitions.

The two spectrum arms' tables are then compared (the largest |difference| over the (plane, band)'s total power), and
the kernels' own time is taken with CUDA events over many calls on one step's 9 fields (69 planes) at 720 x 1440 and
on 69 planes of 1800 x 3600.  Each time is set against both bounds: the bytes read over the H100 SXM data-sheet HBM
bandwidth (3.35 TB/s), and 5 N log2 N float64 operations per complex FFT of N points (two rows each) over the
data-sheet FP64 rate without tensor cores (34 TFLOP/s).  Prints the median and range of ms per step of each arm,
those figures, the card and its power limit as one JSON line.

    python tools/spectra_rollout.py [--rounds 5] [--steps 8]
"""

from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
FP64_FLOP_PER_S = 34e12  # H100 SXM data sheet, FP64 without tensor cores
BANDS = {"global": (-90, 90), "tropics": (-20, 20), "nh": (20, 90)}


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, limit = (out[0].split(", ") + ["?"])[:2] if out else (torch.cuda.get_device_name(), "not read")
    return {"name": name, "power_limit": limit}


def host_spectra(pred, lat: np.ndarray) -> np.ndarray:
    """The host workflow: a copy of the prediction, then numpy.fft.rfft per plane and the band means of
    `aurora_b200.ZonalSpectra`: [planes, bands, W // 2 + 1]."""
    pred = pred.to("cpu")
    w = np.cos(np.deg2rad(lat))
    masks = [(lat >= lo) & (lat <= hi) for lo, hi in BANDS.values()]
    out = []
    for group in ("surf_vars", "atmos_vars"):
        for v in getattr(pred, group).values():
            x = v[0, -1].numpy()
            x = x[None] if x.ndim == 2 else x
            n = x.shape[-1]
            c = np.full(n // 2 + 1, 2.0)
            c[0] = 1.0
            if n % 2 == 0:
                c[-1] = 1.0
            for plane in x:
                counted = np.isfinite(plane).all(-1)
                p = c * np.abs(np.fft.rfft(plane.astype(np.float64), axis=-1)) ** 2 / n ** 2
                out.append([(w[m & counted, None] * p[m & counted]).sum(0) / w[m & counted].sum() for m in masks])
    return np.asarray(out)


def kernel_ms(fields: list, bands: list, weights: torch.Tensor, calls: int) -> float:
    from aurora_b200 import cabi

    planes = sum(f.levels for f in fields)
    out = torch.empty(planes, len(bands) * (fields[0].w // 2 + 3), dtype=torch.float64, device=weights.device)
    ws = torch.empty(cabi.zonal_spectra_workspace_bytes(fields, bands), dtype=torch.uint8, device=weights.device)
    for _ in range(5):
        cabi.zonal_spectra(fields, bands, weights, out, ws)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        cabi.zonal_spectra(fields, bands, weights, out, ws)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / calls


def bounds(ms: float, planes: int, h: int, w: int) -> dict:
    """The kernel time against the HBM and FP64 bounds of one band (rows of overlapping bands are read again)."""
    read = planes * h * w * 4
    flops = planes * math.ceil(h / 2) * 5 * w * math.log2(w)
    hbm_ms, fp64_ms = 1000.0 * read / HBM_BYTES_PER_S, 1000.0 * flops / FP64_FLOP_PER_S
    return {"ms_per_call": ms, "planes": planes, "bytes_read": read, "fft_flops": flops, "hbm_bound_ms": hbm_ms,
            "fp64_bound_ms": fp64_ms, "bound": "hbm" if hbm_ms >= fp64_ms else "fp64",
            "share_of_bound": max(hbm_ms, fp64_ms) / ms}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--kernel-calls", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spectra_rollout.py needs a CUDA device")

    import aurora_b200 as ab
    from aurora_b200.spectra import _field
    from bench import LEVELS13, make_host_batch, randomise_parameters_

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = ab.Aurora(_init="empty", autocast=True).to(dev).eval()
    randomise_parameters_(model, seed=0)
    batch = make_host_batch(model.config, 721, 1440, LEVELS13, pinned=True, seed=0)
    lat = batch.metadata.lat[:720].double().numpy()

    def arm(kind: str, keep: dict | None = None):
        spectra = ab.ZonalSpectra(bands=BANDS) if kind == "spectra" else None
        host = []
        torch.cuda.synchronize()
        start = time.perf_counter()
        with torch.inference_mode():
            for pred in ab.rollout(model, batch, steps=args.steps):
                if kind == "spectra":
                    spectra.step(pred)
                elif kind == "host":
                    host.append(host_spectra(pred, lat))
            table = spectra.results() if spectra is not None else None
        torch.cuda.synchronize()
        ms = 1000.0 * (time.perf_counter() - start) / args.steps
        if keep is not None:
            keep[kind] = table if kind == "spectra" else host
        return ms

    kinds = ("rollout", "spectra", "host")
    results: dict = {}
    for kind in kinds:  # warm-up: captures every graph signature, loads the library
        arm(kind, results)
    times = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for kind in kinds:
            times[kind].append(arm(kind))

    # the two spectrum arms agree
    host = np.concatenate(results["host"])  # [steps * planes, bands, nk]
    got = results["spectra"]["power"].to_numpy().reshape(host.shape)
    agree = float(np.max(np.abs(got - host) / host.sum(-1, keepdims=True)))

    # the kernels alone: one step's 9 fields (69 planes) at 0.25 degrees, and 69 planes at 0.1 degrees
    with torch.inference_mode():
        pred = next(iter(ab.rollout(model, batch, steps=1)))
        fields = [_field(v[0, -1]) for d in (pred.surf_vars, pred.atmos_vars) for v in d.values()]
        n_planes = sum(f.levels for f in fields)
        w_dev = torch.from_numpy(np.cos(np.deg2rad(lat))).to(dev)
        one = [(0, 720)]
        k025 = bounds(kernel_ms(fields, one, w_dev, args.kernel_calls), n_planes, 720, 1440)
        k025["bands"] = 1
        rows3 = [(int(np.nonzero((lat >= lo) & (lat <= hi))[0][0]), int(np.nonzero((lat >= lo) & (lat <= hi))[0][-1]) + 1)
                 for lo, hi in BANDS.values()]
        k025_3 = {"ms_per_call": kernel_ms(fields, rows3, w_dev, args.kernel_calls), "bands": rows3}
        del pred, fields
        g = torch.Generator(device=dev).manual_seed(5)
        big = [torch.randn(lv, 1800, 3600, device=dev, generator=g) for lv in (1, 1, 1, 1, 13, 13, 13, 13, 13)]
        lat01 = np.linspace(89.95, -89.95, 1800)
        w01 = torch.from_numpy(np.cos(np.deg2rad(lat01))).to(dev)
        k01 = bounds(kernel_ms([_field(t) for t in big], [(0, 1800)], w01, args.kernel_calls), 69, 1800, 3600)
        k01["bands"] = 1

    med = {k: statistics.median(v) for k, v in times.items()}
    line = {
        "card": card(), "grid": "721x1440 (model input), 13 levels; spectra of 720x1440, 69 planes",
        "steps_per_arm": args.steps, "rounds": args.rounds, "bands": BANDS,
        "ms_per_step": {"median": med, "min": {k: min(v) for k, v in times.items()},
                        "max": {k: max(v) for k, v in times.items()}, "all": times},
        "spectra_ms_per_step": {"spectra": med["spectra"] - med["rollout"], "host": med["host"] - med["rollout"]},
        "kernel_0p25deg": k025, "kernel_0p25deg_3_bands": k025_3, "kernel_0p1deg": k01,
        "host_agrees_with_gpu": agree,
    }
    print(json.dumps(line, default=float), flush=True)


if __name__ == "__main__":
    main()
