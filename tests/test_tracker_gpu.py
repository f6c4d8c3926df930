"""The cyclone tracker on the GPU against SciPy / numpy and against the reference's `Tracker` (oracle/_ref):
the box kernel bit for bit, whole synthetic tracks on 0.25 and 0.1 degree grids, tracks on real predictions of a tiny
model, and the device-to-host traffic of a step."""

import json
from datetime import datetime, timedelta

import numpy as np
import pandas as pd
import pytest
import torch
from scipy.ndimage import gaussian_filter, minimum_filter

from aurora_b200 import Tracker, cabi, rollout
from aurora_b200 import tracker as ab_tracker
from aurora_b200.batch import Batch, Metadata
from oracle import ref as oracle_ref
from tests import fixtures as fx

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
T0 = datetime(2022, 9, 14, 0)


# ---- the box kernel against SciPy ------------------------------------------------------------------------------------
def _run_boxes(specs, planes):
    """specs: [(op, plane name, rows, cols)] -> (values, counts, [mask or None])."""
    index = np.concatenate([np.concatenate((r, c)) for _, _, r, c in specs]).astype(np.int32)
    boxes, off, moff = [], 0, 0
    for op, name, rows, cols in specs:
        t = planes[name]
        b = cabi.AbTrackBox(plane=t.data_ptr(), plane2=planes["v"].data_ptr() if op == cabi.AB_TRACK_WINDMAX else None,
                            h=t.shape[0], w=t.shape[1], ld=t.stride(0), op=op, rows_off=off, n_rows=len(rows),
                            cols_off=off + len(rows), n_cols=len(cols), mask_off=moff)
        off += len(rows) + len(cols)
        moff += len(rows) * len(cols) if op == cabi.AB_TRACK_MINIMA else 0
        boxes.append(b)
    n = len(specs)
    values = torch.full((n,), -7.0, device=DEV)
    counts = torch.full((n,), -7, dtype=torch.int32, device=DEV)
    masks = torch.full((max(moff, 1),), 7, dtype=torch.uint8, device=DEV)
    cabi.track_boxes(boxes, torch.from_numpy(index).to(DEV), values, counts, masks)
    m = masks.cpu().numpy()
    out, moff = [], 0
    for op, _, rows, cols in specs:
        if op == cabi.AB_TRACK_MINIMA:
            out.append(m[moff:moff + len(rows) * len(cols)].reshape(len(rows), len(cols)))
            moff += len(rows) * len(cols)
        else:
            out.append(None)
    return values.cpu().numpy(), counts.cpu().numpy(), out


def _scipy_minima(box):
    s = gaussian_filter(box, sigma=1)
    m = minimum_filter(s, size=(8, 8)) == s
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = False
    return m


def _index_lists(rng, shape, nr, nc, kind):
    h, w = shape
    if kind == "wrapped":  # the reference's wrapped longitude selection: [w - k, w) then [0, nc - k)
        k = int(rng.integers(1, nc + 1)) if nc > 1 else 1
        cols = np.concatenate((np.arange(w - k, w), np.arange(0, nc - k)))
        r0 = int(rng.integers(0, h - nr + 1))
        return np.arange(r0, r0 + nr), cols
    if kind == "scattered":  # non-contiguous, unsorted, repeated entries allowed
        return rng.integers(0, h, nr), rng.integers(0, w, nc)
    r0, c0 = int(rng.integers(0, h - nr + 1)), int(rng.integers(0, w - nc + 1))
    return np.arange(r0, r0 + nr), np.arange(c0, c0 + nc)


def test_box_kernel_matches_scipy_and_numpy_exactly():
    rng = np.random.default_rng(7)
    h, w = 211, 409
    sign = np.where(rng.random((h, w)) < 0.3, -1.0, 1.0)
    wide = (sign * 10.0 ** rng.uniform(-4.5, 4.5, (h, w))).astype(np.float32)  # values over 9 decades
    smooth = (1e5 + 300 * np.sin(np.arange(h)[:, None] / 7.0) * np.cos(np.arange(w)[None, :] / 5.0)
              + rng.normal(0, 30, (h, w))).astype(np.float32)
    u = (rng.normal(0, 12, (h, w))).astype(np.float32)
    v = (rng.normal(0, 12, (h, w))).astype(np.float32)
    host = {"wide": wide, "smooth": smooth, "u": u, "v": v}
    planes = {k: torch.from_numpy(a).to(DEV) for k, a in host.items()}
    shapes = [(1, 1), (1, 7), (9, 1), (2, 2), (3, 3), (2, 9), (4, 5), (7, 8), (8, 8), (13, 17), (25, 25), (33, 41),
              (41, 41), (61, 61), (81, 81), (101, 101), (101, 37), (1, 101)]
    shapes += [tuple(int(x) for x in rng.integers(1, 102, 2)) for _ in range(30)]
    specs = []
    for i, (nr, nc) in enumerate(shapes):
        kind = ("contiguous", "wrapped", "scattered")[i % 3]
        rows, cols = _index_lists(rng, (h, w), nr, nc, kind)
        plane = ("wide", "smooth")[i % 2]
        specs += [(cabi.AB_TRACK_MINIMA, plane, rows, cols), (cabi.AB_TRACK_MAX, plane, rows, cols),
                  (cabi.AB_TRACK_MIN, plane, rows, cols), (cabi.AB_TRACK_WINDMAX, "u", rows, cols)]
    n_minima = 0
    for s0 in range(0, len(specs), cabi.AB_TRACK_MAX_BOXES):
        chunk = specs[s0:s0 + cabi.AB_TRACK_MAX_BOXES]
        values, counts, masks = _run_boxes(chunk, planes)
        for j, (op, name, rows, cols) in enumerate(chunk):
            box = host[name][np.ix_(rows, cols)]
            what = (op, name, box.shape)
            if op == cabi.AB_TRACK_MINIMA:
                want = _scipy_minima(box)
                np.testing.assert_array_equal(masks[j], want.astype(np.uint8), err_msg=str(what))
                assert counts[j] == want.sum(), what
                n_minima += int(want.sum())
            elif op == cabi.AB_TRACK_MAX:
                assert values[j] == box.max() and counts[j] == 0, what
            elif op == cabi.AB_TRACK_MIN:
                assert values[j] == box.min(), what
            else:
                vb = v[np.ix_(rows, cols)]
                assert values[j] == np.sqrt(box * box + vb * vb).max(), what
    assert n_minima > 100  # the comparison is not vacuous


def test_box_kernel_flags_indices_outside_the_plane():
    planes = {"p": torch.zeros(10, 20, device=DEV), "v": torch.zeros(10, 20, device=DEV)}
    values, counts, _ = _run_boxes([(cabi.AB_TRACK_MAX, "p", np.arange(3), np.array([0, 20])),
                                    (cabi.AB_TRACK_MINIMA, "p", np.arange(3), np.arange(3)),
                                    (cabi.AB_TRACK_MIN, "p", np.array([-1]), np.arange(3))], planes)
    # the constant 3 x 3 box has one interior cell, and it equals its minimum filter
    assert counts.tolist() == [-1, 1, -1] and np.isnan(values[0]) and np.isnan(values[2])


# ---- synthetic storms: whole tracks against the reference ---------------------------------------------------------
def _grid(res):
    lat = torch.linspace(90, -90, round(180 / res) + 1, dtype=torch.float64)
    lon = torch.arange(round(360 / res), dtype=torch.float64) * res
    return lat.float(), lon.float()


def _bump(lat, lon, centre, sigma_deg):
    """exp(-d^2 / 2 sigma^2) around `centre` (lat, lon) on the device, planar distance with longitude wrapped."""
    la = lat.to(DEV, torch.float64)[:, None]
    lo = lon.to(DEV, torch.float64)[None, :]
    dlat = la - centre[0]
    dlon = torch.remainder(lo - centre[1] + 180.0, 360.0) - 180.0
    dlon = dlon * np.cos(np.deg2rad(centre[0]))
    return torch.exp(-(dlat**2 + dlon**2) / (2 * sigma_deg**2)), dlat, dlon


def _storm_batch(lat, lon, time, msl_centre, z_centre, lsm, noise_seed):
    la = torch.deg2rad(lat.to(DEV, torch.float64))[:, None]
    lo = torch.deg2rad(lon.to(DEV, torch.float64))[None, :]
    g = torch.Generator(device=DEV).manual_seed(noise_seed)
    shape = (lat.numel(), lon.numel())
    msl = 99000.0 + 3000.0 * torch.cos(la) + 300.0 * torch.sin(lo) + 0.5 * torch.randn(shape, generator=g, device=DEV,
                                                                                         dtype=torch.float64)
    z = 29000.0 + 1500.0 * torch.cos(la) + 150.0 * torch.sin(lo) + 0.2 * torch.randn(shape, generator=g, device=DEV,
                                                                             dtype=torch.float64)
    u = 5.0 * torch.randn(shape, generator=g, device=DEV, dtype=torch.float64)
    v = 5.0 * torch.randn(shape, generator=g, device=DEV, dtype=torch.float64)
    if msl_centre is not None:
        b, dlat, dlon = _bump(lat, lon, msl_centre, 1.5)
        msl = msl - 4000.0 * b
        speed = 25.0 * torch.sqrt(dlat**2 + dlon**2) * b
        r = torch.sqrt(dlat**2 + dlon**2).clamp_min(1e-6)
        u, v = u - speed * dlat / r, v + speed * dlon / r
    if z_centre is not None:
        msl_z, _, _ = _bump(lat, lon, z_centre, 2.0)
        z = z - 900.0 * msl_z
    levels = fx.LEVELS13
    atmos_z = torch.zeros(1, 1, len(levels), *shape, device=DEV)
    atmos_z[0, 0, levels.index(700)] = z.float()
    return Batch(
        surf_vars={"msl": msl.float()[None, None], "10u": u.float()[None, None], "10v": v.float()[None, None]},
        static_vars={"lsm": lsm},
        atmos_vars={"z": atmos_z},
        metadata=Metadata(lat=lat.to(DEV), lon=lon.to(DEV), time=(time,), atmos_levels=levels),
    )


def _land(lat, lon, boxes):
    lsm = torch.zeros(lat.numel(), lon.numel(), device=DEV)
    la, lo = lat.to(DEV)[:, None], lon.to(DEV)[None, :]
    for lat0, lat1, lon0, lon1 in boxes:
        lsm[((la >= lat0) & (la <= lat1) & (lo >= lon0) & (lo <= lon1)).expand_as(lsm)] = 1.0
    return lsm


def _line(start, step, n):
    return [(start[0] + k * step[0], (start[1] + k * step[1]) % 360) for k in range(n + 1)]


def _scenarios():
    """name -> (grid spacing, msl storm centres, z700 storm centres, land boxes); a centre of None: no storm."""
    s = {}
    # open ocean, both grids
    line = _line((15.0, 140.0), (0.5, -0.75), 9)
    s["ocean_025"] = (0.25, line, line, [])
    line = _line((12.0, 300.0), (0.4, -0.6), 8)
    s["ocean_01"] = (0.1, line, line, [])
    # land to the north: the big boxes stop being clear as the storm approaches, smaller deltas take over
    line = _line((20.0, 130.0), (0.5, -0.5), 9)
    s["land_025"] = (0.25, line, line, [(26.5, 40.0, 100.0, 160.0)])
    line = _line((18.0, 60.0), (0.4, 0.5), 8)
    s["land_01"] = (0.1, line, line, [(24.0, 40.0, 40.0, 90.0)])
    # msl without an interior minimum at steps 3-5 while z700 keeps the storm: the z700 path, refinement finds nothing
    line = _line((15.0, 150.0), (0.5, -0.75), 9)
    s["z700_025"] = (0.25, [None if k in (3, 4, 5) else c for k, c in enumerate(line)], line, [])
    # an island on the extrapolated position of step 4 and the storm 3 degrees north of it: no msl box around the
    # guess is clear, z700 finds the storm, and msl refines it once the boxes around it clear the island
    line = _line((14.0, 145.0), (0.5, -0.75), 9)
    moved = [(c[0] + 3.0, c[1]) if k == 4 else c for k, c in enumerate(line)]
    g = line[4]
    s["z700_refine_025"] = (0.25, moved, moved, [(g[0] - 0.5, g[0] + 0.5, g[1] - 0.5, g[1] + 0.5)])
    # no eye at step 5: fails is incremented and the position extrapolated
    line = [None if k == 5 else c for k, c in enumerate(_line((16.0, 135.0), (0.5, -0.75), 9))]
    s["no_eye_025"] = (0.25, line, line, [])
    # crossing 0 degrees E: the extrapolation does not unwrap longitude (the reference's behaviour)
    line = _line((15.0, 358.5), (0.25, 0.75), 9)
    s["dateline_025"] = (0.25, line, line, [])
    return s


SCENARIOS = _scenarios()


@pytest.fixture(scope="module")
def ref():
    return oracle_ref.load()


def _ref_batch(batch):
    return oracle_ref.to_ref_batch(batch, device="cpu")


def _compare(ours, theirs):
    pd.testing.assert_frame_equal(ours.results(), theirs.results(), check_exact=True)
    assert ours.fails == theirs.fails


@pytest.mark.parametrize("name", sorted(SCENARIOS))
def test_track_matches_the_reference(ref, name):
    res, msl_track, z_track, land = SCENARIOS[name]
    lat, lon = _grid(res)
    lsm = _land(lat, lon, land)
    ours = Tracker(msl_track[0][0], msl_track[0][1], T0)
    theirs = ref.Tracker(msl_track[0][0], msl_track[0][1], T0)
    three_launch_steps = 0
    for k in range(1, len(msl_track)):
        batch = _storm_batch(lat, lon, T0 + timedelta(hours=6 * k), msl_track[k], z_track[k], lsm, noise_seed=k)
        n0 = cabi.launch_count()
        ours.step(batch)
        launches = cabi.launch_count() - n0
        assert launches <= 3
        three_launch_steps += launches == 3
        theirs.step(_ref_batch(batch))
    _compare(ours, theirs)
    lons = ours.results()["lon"].to_numpy()
    if name == "no_eye_025":
        assert ours.fails == 1
    else:
        assert ours.fails == 0 or name == "dateline_025"
    if name.startswith("z700"):
        assert three_launch_steps >= 1, "the z700 path was not taken"
    if name == "dateline_025":
        assert (lons < 1.5).any() and (lons > 358.0).any()
        assert ((lons > 5) & (lons < 355)).any(), "the extrapolation quirk did not show"


def test_complete_failure_at_the_first_step(ref):
    lat, lon = _grid(0.25)
    batch = _storm_batch(lat, lon, T0 + timedelta(hours=6), None, None, _land(lat, lon, []), noise_seed=3)
    ours, theirs = Tracker(15.0, 140.0, T0), ref.Tracker(15.0, 140.0, T0)
    with pytest.raises(ab_tracker.NoEyeException, match="^Completely failed at the first step.$"):
        ours.step(batch)
    with pytest.raises(ref.tracker.NoEyeException, match="^Completely failed at the first step.$"):
        theirs.step(_ref_batch(batch))
    _compare(ours, theirs)
    assert ours.fails == 1


# ---- real predictions of a tiny model -------------------------------------------------------------------------------
def test_tracks_on_rollout_predictions_match_the_reference(ref):
    import aurora_b200 as ab

    cfg = fx.CONFIGS["tiny"]
    net = ab.Aurora(**fx.our_kwargs(cfg))
    net.load_state_dict(fx.make_state_dict(cfg, seed=5), strict=True)
    net = net.to(DEV).eval()
    h, w = 64, 128  # a regional grid at 0.25 degrees: on the default 17 x 32 global grid every box would be empty
    batch = fx.make_batch(cfg, h, w, levels=fx.LEVELS13, seed=5)
    lat = 30.0 - 0.25 * torch.arange(h, dtype=torch.float32)
    lon = 120.0 + 0.25 * torch.arange(w, dtype=torch.float32)
    centre = (22.0, 136.0)
    bump, _, _ = _bump(lat, lon, centre, 1.5)
    bump = bump.float().cpu()
    batch.surf_vars["msl"] = batch.surf_vars["msl"] - 8000.0 * bump
    z = batch.atmos_vars["z"]
    z[:, :, fx.LEVELS13.index(700)] -= 3000.0 * bump
    batch.static_vars["lsm"] = torch.zeros(h, w)
    batch = Batch(batch.surf_vars, batch.static_vars, batch.atmos_vars,
                  Metadata(lat=lat, lon=lon, time=batch.metadata.time, atmos_levels=fx.LEVELS13))
    ours = Tracker(centre[0], centre[1], batch.metadata.time[0])
    theirs = ref.Tracker(centre[0], centre[1], batch.metadata.time[0])
    steps = 0
    with torch.inference_mode():
        for pred in rollout(net, batch, steps=8):
            err_ours = err_theirs = None
            try:
                ours.step(pred)
            except ab_tracker.NoEyeException as e:
                err_ours = e
            try:
                theirs.step(_ref_batch(pred))
            except ref.tracker.NoEyeException as e:
                err_theirs = e
            assert (err_ours is None) == (err_theirs is None), (err_ours, err_theirs)
            if err_ours is not None:
                assert str(err_ours) == str(err_theirs)
                break
            steps += 1
    _compare(ours, theirs)


# ---- traffic: only boxes and masks come back -------------------------------------------------------------------------
def traffic(trace_path: str) -> dict:
    """Device-to-host copies and launches of the second step of a track, and the number of tracked positions."""
    from torch.profiler import ProfilerActivity, profile

    lat, lon = _grid(0.25)
    lsm = _land(lat, lon, [])
    track = _line((15.0, 140.0), (0.5, -0.75), 2)
    tr = Tracker(track[0][0], track[0][1], T0)
    tr.step(_storm_batch(lat, lon, T0 + timedelta(hours=6), track[1], track[1], lsm, noise_seed=1))
    batch = _storm_batch(lat, lon, T0 + timedelta(hours=12), track[2], track[2], lsm, noise_seed=2)
    torch.cuda.synchronize()
    n0 = cabi.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        tr.step(batch)
        torch.cuda.synchronize()
    launches = cabi.launch_count() - n0
    prof.export_chrome_trace(trace_path)
    events = json.loads(open(trace_path).read())["traceEvents"]
    return {"launches": launches, "tracked": len(tr.tracked_lats),
            "d2h": [int(e.get("args", {}).get("bytes", 0)) for e in events
                    if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]}


def test_step_reads_back_only_small_buffers(tmp_path):
    """Profiled in a child process: a profiling session earlier in the test process (other files profile in-process)
    can leave this one without CUDA activity records."""
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parent.parent
    code = ("import json, sys; from tests.test_tracker_gpu import traffic; "
            f"print(json.dumps(traffic({str(tmp_path / 'trace.json')!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert r["launches"] <= 3
    assert r["d2h"], "no device-to-host copy was recorded"
    assert max(r["d2h"]) <= 256 * 1024, r["d2h"]
    assert r["tracked"] == 3
