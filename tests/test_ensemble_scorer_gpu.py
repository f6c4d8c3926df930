"""The ensemble scorer on the GPU against a numpy float64 restatement of its definitions (`aurora_b200/scorer.py`) that
forms the CRPS spread term pairwise, Σ_{k≠l} |x_k - x_l|, and so does not share the kernel's sorted formula: member
counts in every sort-capacity bucket and at its edges, shapes from 1 x 1 to the 0.1-degree plane, with and without
16-byte loads; member permutations and repeated calls (bit for bit); NaN and inf; exact identities; one batch of M
against M batches of one; rollouts of a tiny model, eager and from CUDA graphs; and the device-to-host traffic of
`step` and `results`.

Sums are compared to a relative 1e-12 of the summed magnitudes, as in `test_scorer_gpu.py`."""

import json
from datetime import datetime

import numpy as np
import pytest
import torch

from aurora_b200 import EnsembleScorer, Scorer, cabi, rollout
from aurora_b200.batch import Batch, Metadata
from aurora_b200.scorer import _ensemble_field
from tests import fixtures as fx

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
T0 = datetime(2020, 6, 1, 12, 0)
S = cabi.AB_ENS_SUMS


# ---- the restatement --------------------------------------------------------------------------------------------------
def ref_sums(x, y, c, w):
    """x: float32 [M, ..., H, W]; y, c (or None): float32 [..., H, W]; w: float64 [H].
    -> (sums [..., 10], summed magnitudes [..., 10])"""
    m = x.shape[0]
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    valid = ~np.isnan(y) & ~np.isnan(x).any(axis=0)
    if c is not None:
        valid &= ~np.isnan(c)
    with np.errstate(invalid="ignore", over="ignore"):
        xm = x64.mean(axis=0)
        var = ((x64 - xm) ** 2).sum(axis=0) / (m - 1)
        skill = np.abs(x64 - y64).mean(axis=0)
        pair = np.zeros_like(xm)
        for k in range(m):  # the pairwise form, k != l (|inf - inf| on the diagonal would be NaN)
            pair += np.abs(x64[k] - np.delete(x64, k, axis=0)).sum(axis=0)
        pair /= m * (m - 1)
        wv = np.where(valid, w[:, None], 0.0)
        z = lambda a: np.where(valid, a, 0.0)  # noqa: E731
        d = z(xm - y64)
        terms = [wv, wv * d, wv * d * d, wv * z(var), wv * z(skill), wv * z(pair)]
        if c is None:
            terms += [np.zeros_like(wv)] * 3
        else:
            c64 = c.astype(np.float64)
            af, ao = z(xm - c64), z(y64 - c64)
            terms += [wv * af * ao, wv * af * af, wv * ao * ao]
        terms.append(valid.astype(np.float64))
        return (np.stack([t.sum(axis=(-2, -1)) for t in terms], -1),
                np.stack([np.abs(t).sum(axis=(-2, -1)) for t in terms], -1))


def ref_scores(s, m, members, with_clim):
    """The table's columns from restated sums `s` [n, 10]: {name: value}."""
    with np.errstate(divide="ignore", invalid="ignore"):
        w = s[:, 0]
        rmse, spread = np.sqrt(s[:, 2] / w), np.sqrt(s[:, 3] / w)
        den = np.sqrt(s[:, 7] * s[:, 8])
        return {"ens_rmse": rmse, "ens_bias": s[:, 1] / w, "spread": spread,
                "ssr": np.sqrt((members + 1) / members) * spread / rmse, "crps_skill": s[:, 4] / w,
                "crps_spread": s[:, 5] / w, "crps": s[:, 4] / w - s[:, 5] / w / 2,
                "acc": np.where(with_clim & (den != 0), s[:, 6] / den, np.nan), "count": s[:, 9]}


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
    assert_close(got, want.reshape(-1, S), 1e-12 * mags.reshape(-1, S), what)


# ---- the kernel -------------------------------------------------------------------------------------------------------
def run_kernel(fields, w: torch.Tensor) -> np.ndarray:
    planes = sum(f.levels for f in fields)
    sums = torch.full((planes, S), float("nan"), dtype=torch.float64, device=DEV)
    ws = torch.empty(cabi.ensemble_score_workspace_bytes(fields), dtype=torch.uint8, device=DEV)
    cabi.ensemble_score_fields(fields, w, sums, ws)
    return sums.cpu().numpy()


def _planes(rng, shape, scale, offset=0.0):
    return (offset + scale * rng.standard_normal(shape)).astype(np.float32)


def _ensemble(rng, m, shape, spread=1.5):
    """M members scattered around a common field, a truth and a climatology near it: [M, *shape], shape, shape."""
    base = _planes(rng, shape, 3.0, 280.0)
    x = (base + _planes(rng, (m, *shape), spread)).astype(np.float32)
    return x, (base + _planes(rng, shape, 2.0)).astype(np.float32), _planes(rng, shape, 10.0, 275.0)


def _views(x, y, c, levels):
    """Device copies, each an (H, W) view for one level and (L, H, W) otherwise; the members as a list."""
    dx, dy = torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)
    dc = None if c is None else torch.from_numpy(c).to(DEV)
    pick = (lambda t: t[0]) if levels == 1 else (lambda t: t)  # noqa: E731
    return [pick(dx[k]) for k in range(x.shape[0])], pick(dy), None if dc is None else pick(dc), dx


def _lat(h):
    return np.linspace(90, -90, h).astype(np.float32) if h > 1 else np.array([37.5], np.float32)


def _check_kernel(m, shape, with_clim, seed):
    rng = np.random.default_rng(seed)
    levels, h, w = shape
    x, y, c = _ensemble(rng, m, shape)
    c = c if with_clim else None
    wt = weights_of(_lat(h))
    xs, ty, tc, keep = _views(x, y, c, levels)
    got = run_kernel([_ensemble_field(xs, ty, tc)], torch.from_numpy(wt).to(DEV))
    want, mags = ref_sums(x, y, c, wt)
    assert_sums(got, want, mags, f"M={m} {shape}")
    assert got[:, 9].sum() == y.size
    return got


MEMBERS = [2, 3, 5, 8, 9, 17, 32, 33, 51, 64]  # every sort capacity (8 / 16 / 32 / 64) and its edges
SMALL = [(1, 1, 1), (1, 1, 37), (1, 3, 4), (2, 7, 13), (3, 33, 64), (1, 9, 1441)]


@pytest.mark.parametrize("with_clim", [False, True], ids=["no_clim", "clim"])
@pytest.mark.parametrize("shape", SMALL, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("m", MEMBERS)
def test_kernel_sums_match_pairwise_numpy(m, shape, with_clim):
    _check_kernel(m, shape, with_clim, seed=m * 1000 + sum(shape))


@pytest.mark.parametrize("m,shape", [(2, (1, 720, 1440)), (9, (1, 720, 1440)), (64, (1, 45, 1440)),
                                     (3, (1, 1800, 3600))], ids=lambda v: str(v) if isinstance(v, int) else
                         "x".join(map(str, v)))
@pytest.mark.parametrize("with_clim", [False, True], ids=["no_clim", "clim"])
def test_kernel_sums_match_pairwise_numpy_on_large_planes(m, shape, with_clim):
    _check_kernel(m, shape, with_clim, seed=m + shape[1])


@pytest.mark.parametrize("offset", [0, 1, 2, 3])
@pytest.mark.parametrize("w", [204, 203])
def test_kernel_pitched_and_misaligned_views(offset, w):
    """Row pitch larger than the width and pointers off the 16-byte grid: only offset 0 with an even width of 204
    takes the 16-byte path; the others take the scalar one and must give the same sums."""
    rng = np.random.default_rng(10 + offset + w)
    m, h, ld = 6, 37, 212
    base_x = _planes(rng, (m, 3, h, ld), 2.0, 10.0)
    base_y, base_c = _planes(rng, (3, h, ld), 2.0, 11.0), _planes(rng, (3, h, ld), 5.0, 9.0)
    host = [b[..., offset:offset + w] for b in (base_x, base_y, base_c)]
    dx = torch.from_numpy(base_x).to(DEV)[..., offset:offset + w]
    dy, dc = (torch.from_numpy(b).to(DEV)[..., offset:offset + w] for b in (base_y, base_c))
    wt = weights_of(np.linspace(80, -80, h))
    got = run_kernel([_ensemble_field([dx[k] for k in range(m)], dy, dc)], torch.from_numpy(wt).to(DEV))
    want, mags = ref_sums(*host, wt)
    assert_sums(got, want, mags)


def test_kernel_many_fields_in_one_call():
    rng = np.random.default_rng(3)
    wt = weights_of(np.linspace(90, -90, 40))
    want, mags, fields, keep = [], [], [], []
    for i in range(cabi.AB_ENS_MAX_FIELDS):
        m, lv, h, w = 2 + (5 * i) % 40, 1 + i % 3, 1 + (7 * i) % 40, 4 * (1 + (13 * i) % 25) + (i % 2)
        x, y, c = _ensemble(rng, m, (lv, h, w))
        c = c if i % 4 else None
        xs, ty, tc, dx = _views(x, y, c, 2)
        keep += [dx, ty, tc]
        fields.append(_ensemble_field(xs, ty, tc))
        a, b = ref_sums(x, y, c, wt[:h])
        want.append(a.reshape(-1, S))
        mags.append(b.reshape(-1, S))
    got = run_kernel(fields, torch.from_numpy(wt).to(DEV))
    assert_sums(got, np.concatenate(want), np.concatenate(mags))


def test_kernel_sums_are_bit_identical_under_member_permutation_and_repeats():
    rng = np.random.default_rng(4)
    m = 20
    x, y, c = _ensemble(rng, m, (3, 720, 1440))  # 90 partials per plane
    xs, ty, tc, keep = _views(x, y, c, 3)
    wt = torch.from_numpy(weights_of(np.linspace(90, -90, 721)[:720])).to(DEV)
    perms = [np.arange(m), np.arange(m)[::-1]] + [rng.permutation(m) for _ in range(3)]
    sums = torch.empty(len(perms) + 2, 3, S, dtype=torch.float64, device=DEV)
    f = _ensemble_field(xs, ty, tc)
    ws = torch.empty(cabi.ensemble_score_workspace_bytes([f]), dtype=torch.uint8, device=DEV)
    for i, p in enumerate(perms):
        cabi.ensemble_score_fields([_ensemble_field([xs[k] for k in p], ty, tc)], wt, sums[i], ws)
    for i in range(len(perms), len(perms) + 2):
        cabi.ensemble_score_fields([f], wt, sums[i], ws)
    bits = sums.view(torch.int64).cpu()
    for i in range(1, bits.shape[0]):
        assert torch.equal(bits[0], bits[i]), i


def test_kernel_nan_and_inf():
    """NaN in one member, in the truth, in the climatology and in a whole plane invalidates exactly those points for
    every sum; +inf in one member or in the truth is not skipped and propagates as the restatement says."""
    rng = np.random.default_rng(5)
    m, h, w = 7, 24, 64
    wt = weights_of(np.linspace(80, -80, h))
    cases = {}
    x, y, c = _ensemble(rng, m, (h, w))
    x[3, 0, :5] = np.nan
    x[6, 5, 7] = np.nan
    y[1, 2:4] = np.nan
    c[h - 1, -3:] = np.nan
    cases["nan"] = (x, y, c, 5 + 1 + 2 + 3)
    x, y, c = _ensemble(rng, m, (h, w))
    x[:] = np.nan
    cases["all_nan"] = (x, y, c, h * w)
    x, y, c = _ensemble(rng, m, (h, w))
    x[2, 3, 3] = np.inf
    cases["inf_member"] = (x, y, c, 0)
    x, y, c = _ensemble(rng, m, (h, w))
    y[4, 4] = np.inf
    cases["inf_truth"] = (x, y, c, 0)
    fields, keep, ref = [], [], []
    for name, (x, y, c, dropped) in cases.items():
        xs, ty, tc, dx = _views(x[:, None], y[None], c[None], 1)
        keep += [dx, ty, tc]
        fields.append(_ensemble_field(xs, ty, tc))
        ref.append(ref_sums(x, y, c, wt))
    got = run_kernel(fields, torch.from_numpy(wt).to(DEV))
    for i, (name, (x, y, c, dropped)) in enumerate(cases.items()):
        assert_sums(got[i:i + 1], *ref[i], name)
        assert got[i, 9] == h * w - dropped, name
    assert (got[1] == 0).all()  # all NaN: nothing is valid
    assert np.isinf(got[2, 2]) and np.isinf(got[2, 4]) and np.isinf(got[2, 5]) and np.isnan(got[2, 3])
    assert got[3, 1] == -np.inf and np.isinf(got[3, 4]) and np.isfinite(got[3, 5]) and np.isfinite(got[3, 3])


# ---- EnsembleScorer ---------------------------------------------------------------------------------------------------
def _surface_batch(fields: dict, h, w, lat=None, time=T0, step=0):
    """fields: {name: [B, H, W] or [H, W]} -> a one-history-slice `Batch` on the device."""
    lat = torch.linspace(80, -80, h) if lat is None else lat
    b = {np.asarray(v).reshape(-1, h, w).shape[0] for v in fields.values()}.pop()
    md = Metadata(lat=lat.to(DEV), lon=torch.linspace(0, 360, w + 1)[:-1].to(DEV), time=(time,) * b,
                  atmos_levels=fx.LEVELS4, rollout_step=step)
    return Batch({k: torch.as_tensor(np.asarray(v)).reshape(b, 1, h, w).to(DEV) for k, v in fields.items()}, {}, {},
                 md)


def test_identities():
    h, w, m = 91, 180, 6
    rng = np.random.default_rng(8)
    x = _planes(rng, (h, w), 4.0, 270.0)
    t = _planes(rng, (h, w), 4.0, 270.0)
    lat = torch.linspace(90, -90, h)
    # every member equal to the truth ("a") / every member equal to one field x ("b")
    members = [_surface_batch({"a": t, "b": x}, h, w, lat) for _ in range(m)]
    sc = EnsembleScorer()
    sc.step(members, _surface_batch({"a": t, "b": t}, h, w, lat))
    df = sc.results().set_index("variable")
    for col in ("crps", "crps_skill", "crps_spread", "spread", "ens_rmse", "ens_bias"):
        assert df.loc["a", col] == 0, col
    assert df.loc["b", "crps_spread"] == 0 and df.loc["b", "spread"] == 0
    det = Scorer()
    det.step(_surface_batch({"b": x}, h, w, lat), _surface_batch({"b": t}, h, w, lat))
    mae = det.results().set_index("variable").loc["b", "mae"]
    assert abs(df.loc["b", "crps_skill"] - mae) <= 1e-12 * mae
    assert df.loc["b", "crps"] == df.loc["b", "crps_skill"]
    # M = 2 in closed form: crps_spread = Σ w |x1 - x2| / W, spread² = Σ w (x1 - x2)² / 2 / W
    x2 = _planes(rng, (h, w), 4.0, 270.0)
    sc2 = EnsembleScorer()
    sc2.step([_surface_batch({"b": x}, h, w, lat), _surface_batch({"b": x2}, h, w, lat)],
             _surface_batch({"b": t}, h, w, lat))
    row = sc2.results().iloc[0]
    wv = np.broadcast_to(weights_of(lat.numpy())[:, None], (h, w))
    d12 = x.astype(np.float64) - x2
    big_w = wv.sum()
    assert abs(row["crps_spread"] - (wv * np.abs(d12)).sum() / big_w) <= 1e-12 * row["crps_spread"]
    assert abs(row["spread"] ** 2 - (wv * d12 ** 2 / 2).sum() / big_w) <= 1e-12 * row["spread"] ** 2
    skill = (wv * (np.abs(x - t.astype(np.float64)) + np.abs(x2 - t.astype(np.float64))) / 2).sum() / big_w
    assert abs(row["crps_skill"] - skill) <= 1e-12 * skill


def _restamp(b: Batch, time) -> Batch:
    md = b.metadata
    return Batch(b.surf_vars, b.static_vars, b.atmos_vars,
                 Metadata.derived(md.lat, md.lon, time, md.atmos_levels, md.rollout_step))


def _as_prediction(b: Batch) -> Batch:
    """One history slice, like `Aurora.forward`'s output."""
    one = lambda d: {k: v[:, -1:].contiguous() for k, v in d.items()}  # noqa: E731
    return Batch(one(b.surf_vars), b.static_vars, one(b.atmos_vars), b.metadata)


def _host_rows(members: list, truth: Batch, clim, names):
    """The restatement's rows of one step, from host copies: [(variable, levels, x [M, L, H, W], y, c, w)]."""
    ms = [b.to("cpu") for b in members]
    truth = truth.to("cpu")
    clim = None if clim is None else clim.to("cpu")
    md = ms[0].metadata
    h = md.lat.numel()
    w = weights_of(md.lat.numpy())
    out = []
    for k in names:
        group = "atmos_vars" if k in ms[0].atmos_vars else "surf_vars"
        x = np.stack([getattr(b, group)[k][j, -1].numpy() for b in ms for j in range(len(b.metadata.time))])
        y = getattr(truth, group)[k][0, -1].numpy()
        c = None if clim is None else getattr(clim, group)[k][0, -1].numpy()
        if group == "atmos_vars":
            y = y[[list(truth.metadata.atmos_levels).index(lv) for lv in md.atmos_levels], :h]
            c = None if c is None else c[[list(clim.metadata.atmos_levels).index(lv) for lv in md.atmos_levels], :h]
            levels = [float(lv) for lv in md.atmos_levels]
        else:
            x, y, c = x[:, None], y[None, :h], None if c is None else c[None, :h]
            levels = [np.nan]
        out.append((k, levels, x, y, c, w))
    return out


def assert_table(df, rows, members):
    s, mags, clim = [], [], []
    for _, _, x, y, c, w in rows:
        a, b = ref_sums(x, y, c, w)
        s.append(a.reshape(-1, S))
        mags.append(b.reshape(-1, S))
        clim += [c is not None] * s[-1].shape[0]
    s, mags = np.concatenate(s), np.concatenate(mags)
    assert len(df) == s.shape[0]
    assert list(df["variable"]) == [k for k, lvs, *_ in rows for _ in lvs]
    np.testing.assert_array_equal(df["level"].to_numpy(), np.array([lv for _, lvs, *_ in rows for lv in lvs]))
    assert (df["members"] == members).all()
    # scores against restated ones: 1e-10 of the magnitudes that bound their rounding
    with np.errstate(divide="ignore", invalid="ignore"):
        w = s[:, 0]
        tol = {"ens_bias": mags[:, 1] / w, "crps": mags[:, 4] / w + mags[:, 5] / w,
               "acc": np.where(np.array(clim), mags[:, 6] / np.sqrt(s[:, 7] * s[:, 8]), 0.0), "count": 0.0 * w}
    for name, want in ref_scores(s, mags, members, np.array(clim)).items():
        assert_close(df[name].to_numpy(), want, 1e-10 * tol.get(name, np.abs(want)), name)


def _entries(b: Batch, j0: int, j1: int) -> Batch:
    """Batch entries [j0, j1) as views."""
    md = b.metadata
    return Batch({k: v[j0:j1] for k, v in b.surf_vars.items()}, b.static_vars,
                 {k: v[j0:j1] for k, v in b.atmos_vars.items()},
                 Metadata.derived(md.lat, md.lon, md.time[j0:j1], md.atmos_levels, md.rollout_step))


def test_one_batch_of_m_equals_m_batches_of_one():
    cfg, m = fx.CONFIGS["tiny"], 5
    big = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, b=m, t=1, seed=30)  # staggered by 6 h per entry
    big = _restamp(big, (T0,) * m).to(DEV)
    ones = [_entries(big, j, j + 1) for j in range(m)]
    truth = _restamp(fx.make_batch(cfg, 33, 64, levels=fx.LEVELS13, seed=31), (T0,)).to(DEV)
    clim = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS13[::-1], t=1, seed=32).to(DEV)
    tables = []
    for members in (big, ones, [_entries(big, 0, 2), _entries(big, 2, m)]):
        sc = EnsembleScorer(climatology=clim)
        sc.step(members, truth)
        tables.append(sc.results())
    num = [c for c in tables[0].columns if tables[0][c].dtype == np.float64]
    for t in tables[1:]:
        assert list(t["variable"]) == list(tables[0]["variable"])
        np.testing.assert_array_equal(t[num].to_numpy().view(np.int64), tables[0][num].to_numpy().view(np.int64))
    assert_table(tables[0], _host_rows([big], truth, clim, list(cfg.surf_vars) + list(cfg.atmos_vars)), m)


def test_member_and_field_layouts_are_refused_or_conformed():
    h, w = 12, 32
    rng = np.random.default_rng(9)
    a, b, t = (_planes(rng, (h, w), 1.0, 5.0) for _ in range(3))
    lat = torch.linspace(80, -80, h)
    pa = _surface_batch({"v": a}, h, w, lat)
    pb = _surface_batch({"v": b}, h, w, lat)
    # a member with another row pitch (a column slice of a wider tensor): made contiguous, same sums
    wide = torch.from_numpy(np.pad(b, ((0, 0), (0, 8)))).to(DEV)[:, :w].reshape(1, 1, h, w)
    pb2 = Batch({"v": wide}, {}, {}, pb.metadata)
    truth = _surface_batch({"v": t}, h, w, lat)
    tables = []
    for ms in ([pa, pb], [pa, pb2], [pb2, pa]):
        sc = EnsembleScorer()
        sc.step(ms, truth)
        tables.append(sc.results())
    num = [c for c in tables[0].columns if tables[0][c].dtype == np.float64]
    for tb in tables[1:]:
        np.testing.assert_array_equal(tb[num].to_numpy().view(np.int64), tables[0][num].to_numpy().view(np.int64))
    f64 = Batch({"v": pb.surf_vars["v"].double()}, {}, {}, pb.metadata)
    with pytest.raises(TypeError, match="needs float32 fields, the member's v is torch.float64"):
        EnsembleScorer().step([pa, f64], truth)


# ---- rollouts of a tiny model -----------------------------------------------------------------------------------------
def _model(cfg_name, seed):
    import aurora_b200 as ab

    cfg = fx.CONFIGS[cfg_name]
    net = ab.Aurora(**fx.our_kwargs(cfg, "Aurora"))
    net.load_state_dict(fx.make_state_dict(cfg, seed=seed), strict=True)
    return cfg, net.to(DEV).eval()


def _perturbed(batch: Batch, seed: int) -> Batch:
    g = torch.Generator().manual_seed(seed)
    noise = lambda d: {k: v + 0.01 * v.std() * torch.randn(v.shape, generator=g) for k, v in d.items()}  # noqa: E731
    return Batch(noise(batch.surf_vars), batch.static_vars, noise(batch.atmos_vars), batch.metadata)


def test_rollout_ensembles_match_numpy_and_cuda_graphs():
    cfg, net = _model("tiny", 12)
    m, steps = 4, 3
    batch = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, seed=12)
    starts = [_perturbed(batch, 100 + k) for k in range(m)]
    clim = fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, t=1, seed=40)
    tables, rows = [], []
    for graph in (False, True):
        net.use_cuda_graph = graph
        sc = EnsembleScorer(climatology=clim)  # on the host: copied to the device once
        with torch.inference_mode():
            for i, members in enumerate(zip(*(rollout(net, b, steps=steps) for b in starts))):
                truth = _restamp(fx.make_batch(cfg, 33, 64, levels=fx.LEVELS4, seed=20 + i), members[0].metadata.time)
                sc.step(members, truth)  # a host truth: copied with Batch.to
                if not graph:
                    rows += _host_rows(list(members), truth, clim, list(cfg.surf_vars) + list(cfg.atmos_vars))
        tables.append(sc.results())
    net.use_cuda_graph = False
    eager, graphed = tables
    assert list(eager["rollout_step"].unique()) == [1, 2, 3]
    assert_table(eager, rows, m)
    num = [c for c in eager.columns if eager[c].dtype == np.float64]
    np.testing.assert_array_equal(graphed[num].to_numpy().view(np.int64), eager[num].to_numpy().view(np.int64))
    assert (eager["spread"] > 0).all()


# ---- traffic ----------------------------------------------------------------------------------------------------------
def traffic(trace_path: str) -> dict:
    """Device-to-host copies of one `step` followed by `results` after two warm steps, and the launches of `step`."""
    from torch.profiler import ProfilerActivity, profile

    cfg, m = fx.CONFIGS["tiny"], 3
    truth = _restamp(fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, seed=1), (T0,)).to(DEV)
    clim = fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, t=1, seed=2).to(DEV)
    members = [_restamp(_as_prediction(fx.make_batch(cfg, 721, 1440, levels=fx.LEVELS13, t=1, seed=3 + k).crop(4)),
                        (T0,)).to(DEV) for k in range(m)]
    sc = EnsembleScorer(climatology=clim)
    for _ in range(2):
        sc.step(members, truth)  # the first step copies the coordinates and uploads the row weights
    torch.cuda.synchronize()
    n0 = cabi.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        sc.step(members, truth)
        launches = cabi.launch_count() - n0
        sc.results()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace_path)
    events = json.loads(open(trace_path).read())["traceEvents"]
    return {"launches": launches, "planes": 3 * (len(cfg.surf_vars) + 13 * len(cfg.atmos_vars)),
            "d2h": [int(e.get("args", {}).get("bytes", 0)) for e in events
                    if e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]}


def test_step_reads_nothing_back_and_results_copies_once(tmp_path):
    """Profiled in a child process, so that this file leaves the profiler of the test process untouched."""
    import subprocess
    import sys
    from pathlib import Path

    root = Path(__file__).resolve().parent.parent
    code = ("import json, sys; from tests.test_ensemble_scorer_gpu import traffic; "
            f"print(json.dumps(traffic({str(tmp_path / 'trace.json')!r})))")
    flags = ["-s"] if sys.flags.no_user_site else []
    out = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    r = json.loads(out.stdout.strip().splitlines()[-1])
    assert r["launches"] == 2  # one call (9 variables): partial sums and their reduction
    # one profiling session: the single copy it records is the whole table of three steps, so the step made none
    assert r["d2h"] == [r["planes"] * S * 8], r
