"""The scorer on the GPU against a numpy float64 restatement of its definitions (`aurora_b200/scorer.py`): the kernel's
sums on shapes from 1 x 1 to the 0.1-degree plane, with and without 16-byte loads; `Scorer` on cropped, strided,
batched and multi-level inputs; NaN, inf, empty and constant planes; exact identities; repeatability; rollouts of a
tiny model; and the device-to-host traffic of `step` and `results`.

Sums are compared to a relative 1e-12 of the summed magnitudes (the order of the additions differs, the arithmetic
does not); the scores derived from them to 1e-11 of the magnitude that bounds each one's rounding."""

import json
from datetime import datetime

import numpy as np
import pandas as pd
import pytest
import torch

from aurora_b200 import Scorer, cabi, rollout
from aurora_b200.batch import Batch, Metadata
from aurora_b200.scorer import _field
from tests import fixtures as fx

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
T0 = datetime(2020, 6, 1, 12, 0)


# ---- the restatement --------------------------------------------------------------------------------------------------
def ref_sums(p, t, c, w):
    """p, t, c (or None): float32 arrays [..., H, W]; w: float64 [H].  -> (sums [..., 8], summed magnitudes [..., 8])"""
    p64, t64 = p.astype(np.float64), t.astype(np.float64)
    valid = ~np.isnan(p) & ~np.isnan(t)
    if c is not None:
        valid &= ~np.isnan(c)
    wv = np.where(valid, w[:, None], 0.0)
    d = np.where(valid, p64 - t64, 0.0)
    terms = [wv, wv * d, wv * d * d, wv * np.abs(d)]
    if c is None:
        terms += [np.zeros_like(wv)] * 3
    else:
        c64 = c.astype(np.float64)
        af, ao = np.where(valid, p64 - c64, 0.0), np.where(valid, t64 - c64, 0.0)
        terms += [wv * af * ao, wv * af * af, wv * ao * ao]
    terms.append(valid.astype(np.float64))
    return (np.stack([x.sum(axis=(-2, -1)) for x in terms], -1),
            np.stack([np.abs(x).sum(axis=(-2, -1)) for x in terms], -1))


def ref_scores(s, m, with_clim):
    """Scores from sums `s` and magnitudes `m` [n, 8]: {name: (value, tolerance)}."""
    with np.errstate(divide="ignore", invalid="ignore"):
        w = s[:, 0]
        den = np.sqrt(s[:, 5] * s[:, 6])
        ok = with_clim & (den != 0)
        return {"rmse": (np.sqrt(s[:, 2] / w), 1e-11 * np.sqrt(s[:, 2] / w)),
                "bias": (s[:, 1] / w, 1e-11 * m[:, 1] / w),
                "mae": (s[:, 3] / w, 1e-11 * s[:, 3] / w),
                "acc": (np.where(ok, s[:, 4] / den, np.nan), 1e-11 * np.where(ok, m[:, 4] / den, 0.0)),
                "count": (s[:, 7], 0.0)}


def weights_of(lat) -> np.ndarray:
    return np.cos(np.deg2rad(np.asarray(lat, dtype=np.float64)))


def assert_close(got, want, tol, what=""):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=f"NaN pattern {what}")
    inf = np.isinf(want)
    np.testing.assert_array_equal(got[inf], want[inf], err_msg=f"inf {what}")
    fin = np.isfinite(want)
    err = np.abs(got - want)[fin]
    bound = np.broadcast_to(tol, want.shape)[fin]
    assert (err <= bound).all(), (what, float((err / np.maximum(bound, 1e-300)).max()))


def assert_sums(got, want, mags, what=""):
    assert_close(got, want, 1e-12 * mags, what)


def assert_table(df, ref_rows):
    """`ref_rows`: [(member, variable, level, p, t, c, w)] in the scorer's row order."""
    s, m, clim = [], [], []
    for _, _, _, p, t, c, w in ref_rows:
        a, b = ref_sums(p, t, c, w)
        s.append(a.reshape(-1, 8))
        m.append(b.reshape(-1, 8))
        clim += [c is not None] * s[-1].shape[0]
    s, m = np.concatenate(s), np.concatenate(m)
    assert len(df) == s.shape[0]
    keys = [(mb, v, lv) for mb, v, lvs, *_ in ref_rows for lv in lvs]
    got_keys = list(zip(df["member"], df["variable"], df["level"]))
    assert [(a, b) for a, b, _ in got_keys] == [(a, b) for a, b, _ in keys]
    np.testing.assert_array_equal(np.array([k[2] for k in got_keys]), np.array([k[2] for k in keys], dtype=np.float64))
    for name, (want, tol) in ref_scores(s, m, np.array(clim)).items():
        assert_close(df[name].to_numpy(), want, tol, name)


# ---- the kernel -------------------------------------------------------------------------------------------------------
def run_kernel(fields, w: torch.Tensor) -> np.ndarray:
    planes = sum(f.levels for f in fields)
    sums = torch.full((planes, cabi.AB_SCORE_SUMS), float("nan"), dtype=torch.float64, device=DEV)
    ws = torch.empty(cabi.score_workspace_bytes(fields), dtype=torch.uint8, device=DEV)
    cabi.score_fields(fields, w, sums, ws)
    return sums.cpu().numpy()


def _planes(rng, shape, scale, offset=0.0):
    return (offset + scale * rng.standard_normal(shape)).astype(np.float32)


SHAPES = [(1, 1, 1), (1, 1, 37), (1, 1, 1440), (1, 3, 4), (1, 7, 13), (2, 5, 1441), (3, 33, 65), (1, 720, 1440),
          (1, 1800, 3600)]


@pytest.mark.parametrize("with_clim", [False, True], ids=["no_clim", "clim"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_kernel_sums_match_numpy(shape, with_clim):
    rng = np.random.default_rng(sum(shape))
    levels, h, w = shape
    p = _planes(rng, shape, 3.0, 280.0)
    t = _planes(rng, shape, 3.0, 279.0)
    c = _planes(rng, shape, 10.0, 275.0) if with_clim else None
    lat = np.linspace(90, -90, h).astype(np.float32) if h > 1 else np.array([37.5], np.float32)
    wt = weights_of(lat)
    dev = [None if a is None else torch.from_numpy(a).to(DEV) for a in (p, t, c)]
    views = [None if a is None else (a[0] if levels == 1 else a) for a in dev]
    got = run_kernel([_field(*views)], torch.from_numpy(wt).to(DEV))
    want, mags = ref_sums(p, t, c, wt)
    assert_sums(got, want.reshape(-1, 8), mags.reshape(-1, 8), str(shape))
    assert got[:, 7].sum() == p.size


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
def test_kernel_pitched_and_misaligned_views(offset):
    """Row pitch larger than the width and pointers off the 16-byte grid: the scalar path, or the vector path with a
    tail, must give the same sums."""
    rng = np.random.default_rng(10 + offset)
    h, w, ld = 61, 203, 212
    base = [_planes(rng, (3, h, ld), 2.0, 10.0 * k) for k in range(3)]
    host = [b[..., offset:offset + w] for b in base]
    dev = [torch.from_numpy(b).to(DEV)[..., offset:offset + w] for b in base]
    wt = weights_of(np.linspace(80, -80, h))
    got = run_kernel([_field(*dev)], torch.from_numpy(wt).to(DEV))
    want, mags = ref_sums(*host, wt)
    assert_sums(got, want, mags)


def test_kernel_many_fields_in_one_call():
    rng = np.random.default_rng(3)
    wt = weights_of(np.linspace(90, -90, 40))
    host, fields, keep = [], [], []
    for i in range(cabi.AB_SCORE_MAX_FIELDS):
        lv, h, w = 1 + i % 3, 1 + (7 * i) % 40, 1 + (13 * i) % 97
        arrs = [_planes(rng, (lv, h, w), 1.0 + i, i) for _ in range(3)]
        dev = [torch.from_numpy(a).to(DEV) for a in arrs]
        keep += dev
        fields.append(_field(*dev))
        host.append(ref_sums(*arrs, wt[:h]))
    got = run_kernel(fields, torch.from_numpy(wt).to(DEV))
    want = np.concatenate([a.reshape(-1, 8) for a, _ in host])
    mags = np.concatenate([b.reshape(-1, 8) for _, b in host])
    assert_sums(got, want, mags)


def test_kernel_sums_are_bit_identical_on_repeated_launches():
    rng = np.random.default_rng(4)
    arrs = [torch.from_numpy(_planes(rng, (13, 720, 1440), 5.0, 100.0 * k)).to(DEV) for k in range(3)]
    wt = torch.from_numpy(weights_of(np.linspace(90, -90, 721)[:720])).to(DEV)
    f = _field(*arrs)
    sums = torch.empty(5, 13, cabi.AB_SCORE_SUMS, dtype=torch.float64, device=DEV)
    ws = torch.empty(cabi.score_workspace_bytes([f]), dtype=torch.uint8, device=DEV)
    for i in range(5):
        cabi.score_fields([f], wt, sums[i], ws)
    bits = sums.view(torch.int64).cpu()
    for i in range(1, 5):
        assert torch.equal(bits[0], bits[i]), i


# ---- Scorer -----------------------------------------------------------------------------------------------------------
def _on_device(b: Batch, time=None, lat=None) -> Batch:
    md = b.metadata
    out = b.to(DEV)
    out.metadata = Metadata.derived(out.metadata.lat if lat is None else lat, out.metadata.lon,
                                    md.time if time is None else time, md.atmos_levels, md.rollout_step)
    return out


def _rows(pred, truth, clim, surf, atmos):
    """The restatement's view of a step: [(member, variable, levels, p, t, c, w)] from host copies."""
    pred, truth = pred.to("cpu"), truth.to("cpu")
    clim = None if clim is None else clim.to("cpu")
    h = pred.metadata.lat.numel()
    w = weights_of(pred.metadata.lat.numpy())
    plevels = list(pred.metadata.atmos_levels)
    out = []
    for b in range(len(pred.metadata.time)):
        for k in surf:
            p = pred.surf_vars[k][b, -1].numpy()
            t = truth.surf_vars[k][b, -1, :h].numpy()
            c = None if clim is None else clim.surf_vars[k][min(b, clim.surf_vars[k].shape[0] - 1), -1, :h].numpy()
            out.append((b, k, [np.nan], p, t, c, w))
        for k in atmos:
            p = pred.atmos_vars[k][b, -1].numpy()
            ti = [list(truth.metadata.atmos_levels).index(lv) for lv in plevels]
            t = truth.atmos_vars[k][b, -1].numpy()[ti, :h]
            c = None
            if clim is not None:
                ci = [list(clim.metadata.atmos_levels).index(lv) for lv in plevels]
                c = clim.atmos_vars[k][min(b, clim.atmos_vars[k].shape[0] - 1), -1].numpy()[ci, :h]
            out.append((b, k, [float(lv) for lv in plevels], p, t, c, w))
    return out


def _as_prediction(b: Batch) -> Batch:
    """One history slice, like `Aurora.forward`'s output."""
    one = lambda d: {k: v[:, -1:].contiguous() for k, v in d.items()}  # noqa: E731
    return Batch(one(b.surf_vars), b.static_vars, one(b.atmos_vars), b.metadata)


def test_scorer_crops_a_721_row_truth_and_climatology():
    cfg = fx.CONFIGS["tiny"]
    truth = fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, seed=1)  # T = 2: the last history slice is a view
    clim = fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, t=1, seed=2)
    pred = _as_prediction(fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, t=1, seed=3).crop(4))
    pred = _on_device(pred)
    truth_d, clim_d = _on_device(truth), _on_device(clim)
    names = ("msl", "2t", "z", "q")
    sc = Scorer(climatology=clim_d, variables=names)
    sc.step(pred, truth_d)
    df = sc.results()
    assert (df["count"] == 720 * 1440).all() and len(df) == 2 + 2 * 13
    assert_table(df, _rows(pred, truth, clim, ["msl", "2t"], ["z", "q"]))
    assert (df["time"] == pd.Timestamp(T0)).all() and (df["rollout_step"] == 0).all()


def test_scorer_batch_of_two_with_strided_and_gathered_levels():
    """B = 2; the truth holds every level and two history slices (strided level view with step 2), the climatology its
    levels in reverse order (gathered) and batch size 1 (shared by both members)."""
    cfg = fx.CONFIGS["tiny"]
    plev = fx.LEVELS13[::2]
    pred = _on_device(_as_prediction(fx.make_batch(cfg, 33, 64, levels=plev, b=2, t=1, seed=4)))
    truth = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS13, b=2, seed=5)
    clim = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS13[::-1], b=1, seed=6)
    sc = Scorer(climatology=_on_device(clim))
    sc.step(pred, _on_device(truth))
    df = sc.results()
    assert list(df["member"].unique()) == [0, 1]
    assert list(df["time"].unique()) == [pd.Timestamp(t) for t in pred.metadata.time]
    assert_table(df, _rows(pred, truth, clim, list(cfg.surf_vars), list(cfg.atmos_vars)))


def _surface_batch(fields: dict, h, w, lat=None, time=T0):
    lat = torch.linspace(80, -80, h) if lat is None else lat
    md = Metadata(lat=lat.to(DEV), lon=torch.linspace(0, 360, w + 1)[:-1].to(DEV), time=(time,),
                  atmos_levels=fx.LEVELS4)
    return Batch({k: torch.as_tensor(v).reshape(1, 1, h, w).to(DEV) for k, v in fields.items()}, {}, {}, md)


@pytest.mark.parametrize("hw", [(9, 20), (8, 64)], ids=["scalar", "vector"])
def test_scorer_nan_inf_empty_and_constant_planes(hw):
    h, w = hw
    rng = np.random.default_rng(h * w)
    base = lambda s: _planes(rng, (h, w), 2.0, s)  # noqa: E731
    p, t, c = {}, {}, {}
    # NaN in each input, overlapping in places
    p["nan"], t["nan"], c["nan"] = base(10.0), base(9.0), base(5.0)
    p["nan"][0, :3] = np.nan
    t["nan"][0, 2:6] = np.nan
    c["nan"][h - 1, -4:] = np.nan
    c["nan"][0, 0] = np.nan
    # +inf in the prediction and in the truth at two valid points (differences of both signs), a NaN besides
    p["inf"], t["inf"], c["inf"] = base(1.0), base(1.0), base(0.0)
    p["inf"][1, 1] = np.inf
    t["inf"][2, 3] = np.inf
    p["inf"][3, 0] = np.nan
    # only +inf: rmse, bias and mae are inf
    p["pinf"], t["pinf"], c["pinf"] = base(1.0), base(1.0), base(0.0)
    p["pinf"][h // 2, w // 2] = np.inf
    # all NaN in one input
    p["empty"], t["empty"], c["empty"] = base(1.0), base(1.0), np.full((h, w), np.nan, np.float32)
    # a prediction equal to the climatology: no forecast anomaly, ACC NaN
    p["const"], t["const"], c["const"] = np.full((h, w), 3.0, np.float32), base(3.0), np.full((h, w), 3.0, np.float32)
    lat = torch.linspace(80, -80, h)
    pred, truth, clim = (_surface_batch(x, h, w, lat) for x in (p, t, c))
    sc = Scorer(climatology=clim)
    sc.step(pred, truth)
    df = sc.results().set_index("variable")
    wt = weights_of(lat.numpy())
    rows = [(0, k, [np.nan], p[k], t[k], c[k], wt) for k in p]
    assert_table(df.reset_index(), rows)
    nan_pts = np.isnan(p["nan"]) | np.isnan(t["nan"]) | np.isnan(c["nan"])
    assert df.loc["nan", "count"] == h * w - nan_pts.sum() == h * w - 10
    assert np.isinf(df.loc["pinf", "rmse"]) and df.loc["pinf", "bias"] == np.inf and df.loc["pinf", "mae"] == np.inf
    assert np.isnan(df.loc["inf", "bias"]) and df.loc["inf", "rmse"] == np.inf and df.loc["inf", "count"] == h * w - 1
    assert df.loc["empty", "count"] == 0
    assert df.loc["empty", ["rmse", "bias", "mae", "acc"]].isna().all()
    assert np.isnan(df.loc["const", "acc"]) and np.isfinite(df.loc["const", "rmse"])


def test_scorer_identities():
    h, w = 181, 360
    rng = np.random.default_rng(8)
    x = _planes(rng, (h, w), 4.0, 270.0)
    c = _planes(rng, (h, w), 4.0, 268.0)
    t = np.round(x)  # small integers: t + k is exact in float32
    lat = torch.linspace(90, -90, h)
    k = 0.5
    sc = Scorer(climatology=_surface_batch({"a": c, "b": c}, h, w, lat))
    sc.step(_surface_batch({"a": x, "b": t + np.float32(k)}, h, w, lat), _surface_batch({"a": x, "b": t}, h, w, lat))
    df = sc.results().set_index("variable")
    assert df.loc["a", "rmse"] == 0 and df.loc["a", "bias"] == 0 and df.loc["a", "mae"] == 0
    assert df.loc["a", "acc"] == 1
    assert df.loc["b", "bias"] == k and df.loc["b", "mae"] == k and df.loc["b", "rmse"] == k
    sc2 = Scorer()
    sc2.step(_surface_batch({"a": x}, h, w, lat), _surface_batch({"a": x}, h, w, lat))
    assert np.isnan(sc2.results()["acc"]).all()  # no climatology


# ---- rollouts of a tiny model -----------------------------------------------------------------------------------------
def _model(cfg_name, cls_name, seed):
    import aurora_b200 as ab

    cfg = fx.CONFIGS[cfg_name]
    net = getattr(ab, cls_name)(**fx.our_kwargs(cfg, cls_name))
    net.load_state_dict(fx.make_state_dict(cfg, seed=seed), strict=True)
    return cfg, net.to(DEV).eval()


@pytest.mark.parametrize("variant", ["tiny", "tiny_wave"])
def test_rollout_scores_match_numpy_on_host_copies(variant):
    wave = variant == "tiny_wave"
    cfg, net = _model(variant, "AuroraWave" if wave else "Aurora", 12)
    make = (lambda seed, **kw: fx.make_wave_batch(cfg, 33, 64, seed=seed, with_dwi=False, **kw)) if wave else (
        lambda seed, **kw: fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, seed=seed, **kw))
    batch = fx.make_wave_batch(cfg, 33, 64, seed=12, with_dwi=True) if wave else make(12)
    clim = make(40)
    sc = Scorer(climatology=clim)  # on the host: copied to the device once
    steps = []
    with torch.inference_mode():
        for i, pred in enumerate(rollout(net, batch, steps=3)):
            truth = make(20 + i)
            truth = Batch(truth.surf_vars, truth.static_vars, truth.atmos_vars,
                          Metadata.derived(truth.metadata.lat, truth.metadata.lon, pred.metadata.time,
                                           truth.metadata.atmos_levels))
            sc.step(pred, truth)  # a host truth: copied with Batch.to
            surf = [k for k in pred.surf_vars if k in truth.surf_vars]
            atmos = [k for k in pred.atmos_vars if k in truth.atmos_vars]
            steps.append(_rows(pred, truth, clim, surf, atmos))
    df = sc.results()
    assert list(df["rollout_step"].unique()) == [1, 2, 3]
    assert_table(df, [r for rows in steps for r in rows])
    if wave:
        assert (df["count"] < 32 * 64).any()  # the NaN masks of the wave fields


# ---- traffic ----------------------------------------------------------------------------------------------------------
def _d2h(fn, tmp_path) -> list[int]:
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    events = json.loads(trace.read_text())["traceEvents"]
    return [int(e.get("args", {}).get("bytes", 0)) for e in events
            if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]


def test_step_reads_nothing_back_and_results_copies_once(tmp_path):
    cfg = fx.CONFIGS["tiny"]
    truth = _on_device(fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, seed=1))
    clim = _on_device(fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, t=1, seed=2))
    pred = _on_device(_as_prediction(fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, t=1, seed=3).crop(4)))
    sc = Scorer(climatology=clim)
    for _ in range(2):
        sc.step(pred, truth)  # the first step copies the coordinates and uploads the row weights
    n0 = cabi.launch_count()

    def step_then_results():
        sc.step(pred, truth)
        assert cabi.launch_count() - n0 == 2  # one call: partial sums and their reduction
        sc.results()

    # one profiling session: the single copy it records is the whole table of three steps, so the step made none
    planes = 3 * (len(cfg.surf_vars) + 13 * len(cfg.atmos_vars))
    sizes = _d2h(step_then_results, tmp_path)
    assert sizes == [planes * cabi.AB_SCORE_SUMS * 8], sizes
