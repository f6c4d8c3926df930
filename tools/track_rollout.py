"""Cost of tracking a tropical cyclone during a roll-out of the 1.3 B model at 0.25 degrees (721 x 1440, 13 levels).

Seeded random weights (bench.py's recipe) and a synthetic input carrying a storm over an all-ocean planet.  After a
warm-up, three arms alternate, each an 8-step `aurora_b200.rollout`:

  rollout     the roll-out alone;
  reference   plus the reference's `Tracker` (oracle/_ref), handed each prediction as a reference user would;
  ours        plus `aurora_b200.Tracker`.

Both trackers then follow one more roll-out side by side; the script fails unless their tracks are identical, and
the last step of each is profiled for its device-to-host bytes.  Prints the median ms per step of each arm, those
bytes, the card and its power limit as one JSON line.

    python tools/track_rollout.py [--rounds 5] [--steps 8]
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

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

STORM = (15.0, 140.0)  # lat, lon of the synthetic storm at the initial time


def card() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    name, limit = (out[0].split(", ") + ["?"])[:2] if out else (torch.cuda.get_device_name(), "not read")
    return {"name": name, "power_limit": limit}


def storm_batch(cfg, levels):
    from bench import make_host_batch

    batch = make_host_batch(cfg, 721, 1440, levels, pinned=True, seed=0)
    lat = batch.metadata.lat.double()[:, None]
    lon = batch.metadata.lon.double()[None, :]
    dlon = (torch.remainder(lon - STORM[1] + 180.0, 360.0) - 180.0) * torch.cos(torch.deg2rad(torch.tensor(STORM[0])))
    bump = torch.exp(-((lat - STORM[0]) ** 2 + dlon**2) / (2 * 2.0**2)).float()
    batch.surf_vars["msl"] -= 4000.0 * bump
    batch.atmos_vars["z"][:, :, levels.index(700)] -= 3000.0 * bump
    batch.static_vars["lsm"].zero_()
    return batch


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


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("track_rollout.py needs a CUDA device")

    import pandas as pd

    import aurora_b200 as ab
    from bench import LEVELS13, randomise_parameters_
    from oracle import ref as oracle_ref

    ref = oracle_ref.load()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    model = ab.Aurora(_init="empty", autocast=True).to(dev).eval()
    randomise_parameters_(model, seed=0)
    batch = storm_batch(model.config, LEVELS13)
    t0 = batch.metadata.time[0]

    def arm(kind: str):
        tracker = {"rollout": None, "reference": ref.Tracker, "ours": ab.Tracker}[kind]
        tracker = tracker(*STORM, t0) if tracker else None
        torch.cuda.synchronize()
        start = time.perf_counter()
        with torch.inference_mode():
            for pred in ab.rollout(model, batch, steps=args.steps):
                if kind == "reference":
                    tracker.step(oracle_ref.to_ref_batch(pred))
                elif kind == "ours":
                    tracker.step(pred)
        torch.cuda.synchronize()
        return 1000.0 * (time.perf_counter() - start) / args.steps

    kinds = ("rollout", "reference", "ours")
    for kind in kinds:  # warm-up: captures every graph signature, loads the library and the reference
        arm(kind)
    times = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for kind in kinds:
            times[kind].append(arm(kind))

    # side by side on the same predictions: the tracks must be identical; the last step of each is profiled
    ours, theirs = ab.Tracker(*STORM, t0), ref.Tracker(*STORM, t0)
    with torch.inference_mode():
        for i, pred in enumerate(ab.rollout(model, batch, steps=args.steps)):
            if i < args.steps - 1:
                ours.step(pred)
                theirs.step(oracle_ref.to_ref_batch(pred))
            else:
                bytes_ours = d2h_bytes(lambda: ours.step(pred))
                bytes_ref = d2h_bytes(lambda: theirs.step(oracle_ref.to_ref_batch(pred)))
    pd.testing.assert_frame_equal(ours.results(), theirs.results(), check_exact=True)
    assert ours.fails == theirs.fails

    med = {k: statistics.median(v) for k, v in times.items()}
    line = {
        "card": card(), "grid": "721x1440 (model input), 13 levels", "steps_per_arm": args.steps,
        "rounds": args.rounds,
        "ms_per_step": {"median": med, "all": times},
        "tracker_ms_per_step": {"reference": med["reference"] - med["rollout"], "ours": med["ours"] - med["rollout"]},
        "d2h_bytes_per_tracker_step": {"reference": bytes_ref, "ours": bytes_ours},
        "tracks_identical": True, "fails": ours.fails,
        "track": ours.results().astype({"time": str}).to_dict(orient="list"),
    }
    print(json.dumps(line, default=float), flush=True)


if __name__ == "__main__":
    main()
