"""The zonal spectra on the GPU against a numpy float64 restatement of their definition (`aurora_b200/spectra.py`):
`np.fft.rfft` of the float64 rows.  Widths from 1 to 4096 with every radix, heights from 1 to 1800, pitched,
misaligned, level-strided and gathered views, 64 fields in one call; overlapping, single-row and empty bands; NaN and
inf rows; exact cases (a pure tone, the Nyquist alternation, a constant, Parseval, a longitude roll); repeated calls
bit for bit; rollouts of tiny models, eager and from CUDA graphs; and the device-to-host traffic of `step` and
`results`.

Every weighted spectrum sum is compared to 1e-12 of the sum of that (plane, band)'s reference spectrum over all
wavenumbers; the float64 FFT's own error is about 5e-15 of it.  Row counts must match exactly."""

import json
from datetime import datetime

import numpy as np
import pytest
import torch

from aurora_b200 import ZonalSpectra, cabi, rollout
from aurora_b200.batch import Batch, Metadata
from aurora_b200.spectra import _field
from tests import fixtures as fx

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
T0 = datetime(2020, 6, 1, 12, 0)
TOL = 1e-12


# ---- the restatement --------------------------------------------------------------------------------------------------
def row_spectra(x: np.ndarray) -> np.ndarray:
    """x: float32 [..., W] -> P [..., W // 2 + 1] in float64 (NaN rows stay NaN)."""
    n = x.shape[-1]
    c = np.full(n // 2 + 1, 2.0)
    c[0] = 1.0
    if n % 2 == 0:
        c[-1] = 1.0
    return c * np.abs(np.fft.rfft(x.astype(np.float64), axis=-1)) ** 2 / n ** 2


def ref_sums(x: np.ndarray, w: np.ndarray, bands) -> np.ndarray:
    """x: float32 [L, H, W]; w: float64 [H]; bands: [(r0, r1)] -> [L, bands, W // 2 + 3]: Σw, rows, Σ w P(k)."""
    counted = np.isfinite(x).all(axis=-1)  # [L, H]
    with np.errstate(invalid="ignore", over="ignore"):
        p = np.where(counted[..., None], row_spectra(x), 0.0)
    out = np.zeros((x.shape[0], len(bands), x.shape[-1] // 2 + 3))
    for b, (r0, r1) in enumerate(bands):
        wc = np.where(counted[:, r0:r1], w[None, r0:r1], 0.0)
        out[:, b, 0] = wc.sum(-1)
        out[:, b, 1] = counted[:, r0:r1].sum(-1)
        out[:, b, 2:] = (wc[..., None] * p[:, r0:r1]).sum(-2)
    return out


def assert_sums(got: np.ndarray, want: np.ndarray, what=""):
    got, want = got.reshape(want.shape), want
    np.testing.assert_array_equal(got[..., 1], want[..., 1], err_msg=f"rows {what}")
    np.testing.assert_allclose(got[..., 0], want[..., 0], rtol=TOL, atol=0, err_msg=f"weights {what}")
    bound = TOL * want[..., 2:].sum(-1, keepdims=True)
    err = np.abs(got[..., 2:] - want[..., 2:])
    assert (err <= bound).all(), (what, float((err / np.maximum(bound, 1e-300)).max()))


# ---- the kernel -------------------------------------------------------------------------------------------------------
def run_kernel(fields, bands, w: torch.Tensor) -> np.ndarray:
    planes = sum(f.levels for f in fields)
    width = fields[0].w // 2 + 3
    out = torch.full((planes, len(bands) * width), float("nan"), dtype=torch.float64, device=DEV)
    ws = torch.empty(max(cabi.zonal_spectra_workspace_bytes(fields, bands), 8), dtype=torch.uint8, device=DEV)
    cabi.zonal_spectra(fields, bands, w, out, ws)
    return out.cpu().numpy().reshape(planes, len(bands), width)


def _lat(h):
    return np.linspace(90, -90, h) if h > 1 else np.array([37.5])


def _weights(h):
    return np.cos(np.deg2rad(_lat(h).astype(np.float32).astype(np.float64)))


def _check(x: np.ndarray, bands, view=None, what=""):
    """x: float32 [L, H, W] on the host; `view` maps its device copy to the (L, H, W) view the kernel reads."""
    d = torch.from_numpy(x).to(DEV)
    v = d if view is None else view(d)
    wt = _weights(x.shape[1])
    got = run_kernel([_field(v)], bands, torch.from_numpy(wt).to(DEV))
    assert_sums(got, ref_sums(x, wt, bands), what)
    return got


def _fields(rng, shape, offset=0.0):
    """Zero-mean noise with a few tones, or with an offset (k = 0 dominant)."""
    x = rng.standard_normal(shape)
    n = shape[-1]
    cols = np.arange(n)
    for m in (1, 3, n // 3):
        x += rng.standard_normal(shape[:-1] + (1,)) * np.cos(2 * np.pi * m * cols / n + rng.uniform(0, 6))
    return (offset + 4.0 * x).astype(np.float32)


WIDTHS = [1, 2, 3, 4, 5, 8, 9, 25, 27, 32, 64, 90, 120, 125, 900, 1024, 1440, 2048, 3600, 4000, 4096]


@pytest.mark.parametrize("w", WIDTHS)
def test_widths_match_numpy(w):
    rng = np.random.default_rng(w)
    for h, levels in ((1, 2), (7, 1), (65, 2)):
        for offset in (0.0, 280.0):
            x = _fields(rng, (levels, h, w), offset)
            bands = [(0, h), (h // 3, h // 3 + max(1, h // 2))]
            _check(x, bands, what=f"w={w} h={h} offset={offset}")


@pytest.mark.parametrize("h,w", [(721, 1440), (1800, 3600), (361, 4096), (1800, 90)])
def test_large_planes_match_numpy(h, w):
    rng = np.random.default_rng(h + w)
    x = _fields(rng, (1, h, w))
    _check(x, [(0, h), (h // 2 - 80, h // 2 + 81), (0, 1)], what=f"{h}x{w}")


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
@pytest.mark.parametrize("w", [32, 90])
def test_pitched_misaligned_and_level_strided_views(offset, w):
    """Row pitch larger than the width, pointers off the 16-byte grid and every other level: only offset 0 at w = 32
    takes cp.async.bulk; the others take cp.async and must give the same sums."""
    rng = np.random.default_rng(offset + w)
    ld, h = w + 12, 37
    base = _fields(rng, (6, h, ld), 3.0)
    x = np.ascontiguousarray(base[::2, :, offset:offset + w])
    _check(x, [(0, h), (5, 30)], view=lambda d: torch.from_numpy(base).to(DEV)[::2, :, offset:offset + w])


def test_gathered_levels_and_many_fields_in_one_call():
    rng = np.random.default_rng(3)
    h, w = 40, 120
    wt = _weights(h)
    bands = [(0, h), (10, 11), (3, 3), (0, 20), (15, 40)]
    fields, keep, want = [], [], []
    for i in range(cabi.AB_SPEC_MAX_FIELDS):
        lv = 1 + i % 3
        base = _fields(rng, (4, h, w), 10.0 * (i % 2))
        d = torch.from_numpy(base).to(DEV)
        idx = [0, 2, 3][:lv] if i % 4 == 0 else list(range(lv))
        v = d[idx] if i % 4 == 0 else d[:lv]  # a gathered copy, or a strided view
        keep.append(v)
        fields.append(_field(v))
        want.append(ref_sums(base[idx], wt, bands))
    got = run_kernel(fields, bands, torch.from_numpy(wt).to(DEV))
    assert_sums(got, np.concatenate(want))
    assert (got[:, 2, :2] == 0).all() and (got[:, 1, 1] == 1).all()  # the empty and the single-row band


def test_nan_and_inf_rows_are_skipped():
    rng = np.random.default_rng(5)
    h, w = 24, 64
    x = _fields(rng, (3, h, w), 1.0)
    x[0, 0, 5] = np.nan
    x[0, 7, :] = np.nan
    x[0, 8, 63] = np.inf
    x[0, 9, 0] = -np.inf
    x[1, 23, 1] = np.nan  # the last row, alone in its pair of an odd band
    x[2] = np.nan  # an all-NaN plane
    got = _check(x, [(0, h), (0, 23), (9, 10)])
    np.testing.assert_array_equal(got[:, 0, 1], [h - 4, h - 1, 0])
    assert got[0, 2, 1] == 0 and np.isnan(_power(got)[0, 2]).all() and np.isnan(_power(got)[2]).all()
    assert np.isfinite(got[:2, :2]).all()


def _power(got):
    with np.errstate(invalid="ignore", divide="ignore"):
        return got[..., 2:] / got[..., :1]


def test_exact_cases():
    n, h = 360, 9
    cols = np.arange(n)
    wt = torch.from_numpy(_weights(h)).to(DEV)
    one = [(0, h)]
    for m in (1, 7, 60, 179):
        a, theta = 3.5, 0.3 * m
        x = np.tile(a * np.cos(2 * np.pi * m * cols / n + theta), (1, h, 1)).astype(np.float32)
        d = torch.from_numpy(x).to(DEV)  # held while the kernel reads it
        p = _power(run_kernel([_field(d)], one, wt))[0, 0]
        ref = _power(ref_sums(x, _weights(h), one))[0, 0]
        assert abs(p[m] - ref[m]) <= TOL * a * a and abs(p[m] - a * a / 2) <= 1e-6 * a * a  # float32 input
        assert (np.abs(np.delete(p, m)) <= TOL * a * a).all(), m
    # the Nyquist alternation (+1, -1, ...): all power at k = N/2 with c = 1; a constant: all at k = 0
    for x, k in ((np.where(cols % 2 == 0, 1.0, -1.0), n // 2), (np.full(n, 2.5), 0)):
        x = np.tile(x, (1, h, 1)).astype(np.float32)
        d = torch.from_numpy(x).to(DEV)
        p = _power(run_kernel([_field(d)], one, wt))[0, 0]
        want = np.mean(x[0, 0].astype(np.float64) ** 2)
        assert abs(p[k] - want) <= TOL * want and (np.abs(np.delete(p, k)) <= TOL * want).all(), k
    # Parseval, and invariance under a longitude roll
    rng = np.random.default_rng(6)
    x = _fields(rng, (2, h, n), 5.0)
    rolled = np.roll(x, 77, axis=-1)
    d, dr = torch.from_numpy(x).to(DEV), torch.from_numpy(rolled).to(DEV)
    got = run_kernel([_field(d), _field(dr)], one, wt)
    w64 = _weights(h)
    parseval = (w64[None] * (x.astype(np.float64) ** 2).mean(-1)).sum(-1)
    np.testing.assert_allclose(got[:2, 0, 2:].sum(-1), parseval, rtol=TOL)
    assert (np.abs(got[:2, 0, 2:] - got[2:, 0, 2:]) <= TOL * got[:2, 0, 2:].sum(-1, keepdims=True)).all()


def test_repeated_calls_are_bit_identical():
    rng = np.random.default_rng(4)
    x = torch.from_numpy(_fields(rng, (5, 720, 1440), 3.0)).to(DEV)
    wt = torch.from_numpy(_weights(721)[:720]).to(DEV)
    bands = [(0, 720), (200, 520), (100, 300)]
    f = [_field(x)]
    ws = torch.empty(cabi.zonal_spectra_workspace_bytes(f, bands), dtype=torch.uint8, device=DEV)
    out = torch.empty(4, 5, 3 * 723, dtype=torch.float64, device=DEV)
    for i in range(4):
        cabi.zonal_spectra(f, bands, wt, out[i], ws)
    bits = out.view(torch.int64).cpu()
    for i in range(1, 4):
        assert torch.equal(bits[0], bits[i]), i


# ---- ZonalSpectra -----------------------------------------------------------------------------------------------------
def _surface_batch(fields: dict, h, w, lat=None, step=0):
    lat = torch.linspace(80, -80, h) if lat is None else lat
    b = {np.asarray(v).reshape(-1, h, w).shape[0] for v in fields.values()}.pop()
    md = Metadata(lat=lat.to(DEV), lon=torch.linspace(0, 360, w + 1)[:-1].to(DEV), time=(T0,) * b,
                  atmos_levels=fx.LEVELS4, rollout_step=step)
    return Batch({k: torch.as_tensor(np.asarray(v)).reshape(b, 1, h, w).to(DEV) for k, v in fields.items()}, {}, {},
                 md)


BANDS = {"global": (-90, 90), "tropics": (-20, 20), "nh": (20, 90), "overlap": (0, 45), "one": (46, 46),
         "none": (0.1, 0.2)}


def _key(level) -> float:
    return -1.0 if np.isnan(level) else float(level)  # NaN (surface) never equals itself as a dict key


def _host_table(batch: Batch, label: str, bands=BANDS) -> dict:
    """The restatement's (power, rows) per (member, variable, level) of one `step`, from a host copy."""
    b = batch.to("cpu")
    md = b.metadata
    lat = md.lat.numpy().astype(np.float64)
    w = np.cos(np.deg2rad(lat))
    ranges = []
    for lo, hi in bands.values():
        idx = np.nonzero((lat >= lo) & (lat <= hi))[0]
        ranges.append((int(idx[0]), int(idx[-1]) + 1) if idx.size else (0, 0))
    out = {}
    for j in range(len(md.time)):
        for k, v in list(b.surf_vars.items()) + list(b.atmos_vars.items()):
            x = v[j, -1].numpy()
            x = x[None] if x.ndim == 2 else x
            s = ref_sums(x, w, ranges)
            levels = md.atmos_levels if k in b.atmos_vars else (np.nan,)
            for li, lv in enumerate(levels):
                out[(label, j, k, _key(lv))] = s[li]
    return out


def assert_table(df, tables: list, bands=BANDS):
    ref = {}
    for step, t in enumerate(tables):
        ref.update({(step,) + key: v for key, v in t.items()})
    nb = len(bands)
    assert len(df) % nb == 0
    groups = df.groupby(["rollout_step", "label", "member", "variable", "level"], sort=False, dropna=False,
                        observed=True)
    assert len(groups) == len(ref)
    steps = sorted(df["rollout_step"].unique())
    for (step, label, member, variable, level), g in groups:
        want = ref[(steps.index(step), label, member, variable, _key(level))]
        assert list(g["band"].unique()) == list(bands)
        nk = want.shape[1] - 2
        power = g["power"].to_numpy().reshape(nb, nk)
        rows = g["rows"].to_numpy().reshape(nb, nk)
        np.testing.assert_array_equal(rows[:, 0], want[:, 1])
        with np.errstate(invalid="ignore", divide="ignore"):
            ref_power = want[:, 2:] / want[:, :1]
        np.testing.assert_array_equal(np.isnan(power), np.isnan(ref_power))
        ok = ~np.isnan(ref_power)
        bound = np.broadcast_to(TOL * ref_power.sum(-1, keepdims=True) * 2, ref_power.shape)
        assert (np.abs(power - ref_power)[ok] <= bound[ok]).all(), (variable, level)


def test_step_and_results_match_numpy():
    cfg = fx.CONFIGS["tiny"]
    x = fx.make_batch(cfg, 91, 180, levels=fx.LEVELS4, b=2, t=1, seed=3).to(DEV)
    sp = ZonalSpectra(bands=BANDS)
    sp.step(x)
    sp.step(x, label="truth")
    df = sp.results()
    nv = len(cfg.surf_vars) + 4 * len(cfg.atmos_vars)
    assert len(df) == 2 * 2 * nv * len(BANDS) * 91
    assert list(df["label"].unique()) == ["prediction", "truth"]
    assert (df[df["band"] == "none"]["rows"] == 0).all() and df[df["band"] == "none"]["power"].isna().all()
    assert (df[df["band"] == "one"]["rows"] == 1).all()
    g = df[(df["band"] == "global")]
    assert np.isinf(g[g["wavenumber"] == 0]["wavelength_km"]).all()
    assert_table(df[df["label"] == "prediction"], [_host_table(x, "prediction")])
    f64 = Batch({"v": x.surf_vars["2t"].double()}, {}, {}, x.metadata)
    with pytest.raises(TypeError, match="needs float32 fields, the batch's v is torch.float64"):
        sp.step(f64)


def _model(cfg_name, cls_name, seed):
    import aurora_b200 as ab

    cfg = fx.CONFIGS[cfg_name]
    net = getattr(ab, cls_name)(**fx.our_kwargs(cfg, cls_name))
    net.load_state_dict(fx.make_state_dict(cfg, seed=seed), strict=True)
    return cfg, net.to(DEV).eval()


@pytest.mark.parametrize("variant", ["tiny", "tiny_wave"])
def test_rollouts_match_numpy_eager_and_from_cuda_graphs(variant):
    wave = variant == "tiny_wave"
    cfg, net = _model(variant, "AuroraWave" if wave else "Aurora", 12)
    batch = (fx.make_wave_batch(cfg, 33, 64, seed=12, with_dwi=True) if wave
             else fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, seed=12))
    bands = {"global": (-90, 90), "tropics": (-30, 30)}
    tables, ref = [], []
    for graph in (False, True):
        net.use_cuda_graph = graph
        sp = ZonalSpectra(bands=bands)
        with torch.inference_mode():
            for pred in rollout(net, batch, steps=3):
                sp.step(pred)
                if not graph:
                    ref.append(_host_table(pred, "prediction", bands))
        tables.append(sp.results())
    net.use_cuda_graph = False
    eager, graphed = tables
    assert list(eager["rollout_step"].unique()) == [1, 2, 3]
    assert_table(eager, ref, bands)
    num = [c for c in eager.columns if eager[c].dtype == np.float64]
    np.testing.assert_array_equal(graphed[num].to_numpy().view(np.int64), eager[num].to_numpy().view(np.int64))
    if wave:
        assert (eager["rows"] < 32).any()  # the NaN masks of the wave fields drop rows


# ---- traffic ----------------------------------------------------------------------------------------------------------
def traffic(trace_path: str) -> dict:
    """Device-to-host copies of one `step` followed by `results` after two warm steps, and the launches of `step`."""
    from torch.profiler import ProfilerActivity, profile

    cfg = fx.CONFIGS["tiny"]
    x = fx.make_batch(cfg, 720, 1440, levels=fx.LEVELS13, t=1, seed=3).to(DEV)
    sp = ZonalSpectra(bands={"global": (-90, 90), "tropics": (-20, 20)})
    for _ in range(2):
        sp.step(x)  # the first step copies the coordinates and uploads the row weights
    torch.cuda.synchronize()
    n0 = cabi.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        sp.step(x)
        launches = cabi.launch_count() - n0
        sp.results()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace_path)
    events = json.loads(open(trace_path).read())["traceEvents"]
    return {"launches": launches, "values": 3 * (len(cfg.surf_vars) + 13 * len(cfg.atmos_vars)) * 2 * 723,
            "d2h": [int(e.get("args", {}).get("bytes", 0)) for e in events
                    if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]}


def test_step_reads_nothing_back_and_results_copies_once(tmp_path):
    """Profiled in a child process, so that this file leaves the profiler of the test process untouched."""
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parent.parent
    code = ("import json, sys; from tests.test_zonal_spectra_gpu import traffic; "
            f"print(json.dumps(traffic({str(tmp_path / 'trace.json')!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert r["launches"] == 2  # one call (9 variables): partial sums and their reduction
    # one profiling session: the single copy it records is everything of three steps, so the step made none
    assert r["d2h"] == [r["values"] * 8], r
