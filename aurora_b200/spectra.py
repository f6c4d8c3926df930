"""``ZonalSpectra``: latitude-band zonal power spectra of predictions (or any `Batch`), computed where the fields live.
The usual way to see whether a forecast loses small-scale variance as lead time grows, which RMSE and ACC reward
rather than show.

Every `step` is one `ab_zonal_spectra` call per 64 fields (`csrc/spectra.cu`): one descriptor per variable and batch
member, and per level plane and band the weight sum, the row count and the weighted sums of the row spectra, appended
to a device tensor the object owns.  Nothing is read back until `results`, which copies everything accumulated to the
host at once.

Definitions.  For one row x_0 … x_{N-1} of a plane (N = W longitudes), X_k = Σ_n x_n e^{−2πikn/N} in float64 from the
float32 values, and the one-sided variance spectrum is

    P(k) = c_k |X_k|² / N²,   k = 0 … ⌊N/2⌋,   c_0 = 1, c_{N/2} = 1 when N is even, otherwise c_k = 2,

so that Σ_k P(k) = (1/N) Σ_n x_n² (Parseval).  A row counts only when all N values are finite (unlike `Scorer`, which
lets ±inf through: an inf would turn the row's whole transform into NaN).  For a band b of latitudes [lo, hi]
(inclusive), with the row weights w_r = cos(deg2rad(lat_r)) in float64 that `Scorer` uses,

    power(k) = Σ_{r∈b, counted} w_r P_r(k) / Σ_{r∈b, counted} w_r,      rows = the number of counted rows,

and an empty band gives rows = 0 and power = NaN.  ``wavelength_km = 2π · 6371 · c̄_b / k`` with
c̄_b = Σ cos²φ / Σ cos φ over all the band's rows: a geometric label, inf at k = 0, independent of which rows counted.
"""

from __future__ import annotations

from typing import Iterable, Optional

import numpy as np
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch
from aurora_b200.scorer import _StepScorer, _layout

__all__ = ["ZonalSpectra"]

COLUMNS = ("time", "rollout_step", "label", "member", "variable", "level", "band", "wavenumber", "wavelength_km",
           "power", "rows")
EARTH_RADIUS_KM = 6371.0


def _field(x: torch.Tensor) -> cabi.AbSpectrumField:
    """Descriptor of an (H, W) or (C, H, W) view with unit column stride."""
    f = cabi.AbSpectrumField()
    f.levels, f.h, f.w, f.ld, f.level_stride = _layout(x)
    f.x = x.data_ptr()
    return f


def _supported_width(w: int) -> bool:
    if w < 1 or w > cabi.AB_SPEC_MAX_WIDTH:
        return False
    for p in (2, 3, 5):
        while w % p == 0:
            w //= p
    return w == 1


class ZonalSpectra(_StepScorer):
    """Zonal power spectra of device-resident fields, step by step, without copying them to the host.

    Args:
        bands: Latitude bands, name → (lat_lo, lat_hi) in degrees, inclusive; at most 8, they may overlap.  By
            default ``{"global": (-90, 90)}``.
        variables: Surface / atmospheric variable names.  By default every surface and atmospheric variable of each
            batch.  Static variables are never used.
    """

    def __init__(self, bands: Optional[dict] = None, variables: Optional[Iterable[str]] = None) -> None:
        super().__init__(None, variables)
        bands = {"global": (-90.0, 90.0)} if bands is None else bands
        if not isinstance(bands, dict) or not bands:
            raise ValueError("ZonalSpectra needs bands as a non-empty dict of name -> (lat_lo, lat_hi)")
        if len(bands) > cabi.AB_SPEC_MAX_BANDS:
            raise ValueError(f"ZonalSpectra takes at most {cabi.AB_SPEC_MAX_BANDS} bands, got {len(bands)}")
        self.bands: dict[str, tuple[float, float]] = {}
        for name, band in bands.items():
            lo, hi = (float(v) for v in band)
            if not -90.0 <= lo <= hi <= 90.0:
                raise ValueError(f"band {name!r} = ({lo}, {hi}) needs -90 <= lo <= hi <= 90")
            self.bands[str(name)] = (lo, hi)
        self._geometry: dict[tuple, tuple] = {}

    def _grid(self, batch: Batch) -> tuple:
        """(band row ranges, wavelengths [bands, W/2 + 1]) of the batch's grid; refuses grids the kernel does not
        take."""
        md = batch.metadata
        lat, lon = self._coords(md.lat).astype(np.float64), self._coords(md.lon).astype(np.float64)
        w = lon.size
        key = (lat.tobytes(), lon.tobytes())
        hit = self._geometry.get(key)
        if hit is not None:
            return hit
        if lat.size > 1:
            d = np.diff(lat)
            if not ((d > 0).all() or (d < 0).all()):
                raise ValueError("ZonalSpectra.step needs strictly monotonic latitudes")
        spacing = 360.0 / max(w, 1)
        if w < 1 or (w > 1 and not (np.abs(np.diff(lon) - spacing) <= 1e-3 * spacing).all()):
            raise ValueError(f"ZonalSpectra.step needs {w} longitudes equally spaced by {spacing} degrees to cover "
                             "360 degrees")
        if not _supported_width(w):
            raise ValueError(f"ZonalSpectra.step takes grids of up to {cabi.AB_SPEC_MAX_WIDTH} longitudes whose "
                             f"count has no prime factor above 5; this one has {w}")
        cos = np.cos(np.deg2rad(lat))
        rows, wavelengths = [], []
        k = np.arange(w // 2 + 1, dtype=np.float64)
        for lo, hi in self.bands.values():
            idx = np.nonzero((lat >= lo) & (lat <= hi))[0]
            rows.append((int(idx[0]), int(idx[-1]) + 1) if idx.size else (0, 0))
            with np.errstate(divide="ignore", invalid="ignore"):
                cbar = (cos[idx] ** 2).sum() / cos[idx].sum()
                wavelengths.append(2 * np.pi * EARTH_RADIUS_KM * cbar / k)
        hit = (rows, np.stack(wavelengths))
        self._geometry[key] = hit
        return hit

    # -- public -----------------------------------------------------------------------------------------------------
    def step(self, batch: Batch, label: str = "prediction") -> None:
        """Add the spectra of one `Batch`.  Enqueues the work on the current stream; nothing is read back.

        Args:
            batch: A prediction as `Aurora.forward` returns it, a truth or an analysis, on a CUDA device, with 1-D
                coordinates, whole grids, strictly monotonic latitudes and W equally spaced longitudes covering 360
                degrees (W ≤ 4096 with no prime factor above 5).  Every batch entry is one member; the last history
                slice is used.
            label: A name for these rows of the table, such as "prediction" or "truth".
        """
        if not isinstance(label, str):
            raise TypeError(f"ZonalSpectra.step needs a str label, got {type(label).__name__}")
        md = batch.metadata
        self._check_prediction(batch, "batch")
        surf, atmos = self._names(batch, batch)
        self._check_tensors(batch, surf, atmos, "batch")
        band_rows, wavelengths = self._grid(batch)
        h, w = md.lat.numel(), md.lon.numel()
        for k in surf + atmos:
            t = batch.atmos_vars[k] if k in atmos else batch.surf_vars[k]
            if tuple(t.shape[-2:]) != (h, w):
                raise ValueError(f"{k} has shape {tuple(t.shape)}, the grid is {h} x {w}")
        device = batch.surf_vars[surf[0]].device if surf else batch.atmos_vars[atmos[0]].device
        geometry = (tuple(self.bands), wavelengths)

        with torch.cuda.device(device):
            weights = self._row_weights(md.lat, device)
            fields, rows, keep = [], [], []
            for b, time in enumerate(md.time):
                for k in surf + atmos:
                    is_atmos = k in atmos
                    x = (batch.atmos_vars if is_atmos else batch.surf_vars)[k][b, -1]
                    x = x if x.stride(-1) == 1 else x.contiguous()
                    keep.append(x)
                    fields.append(_field(x))
                    levels = md.atmos_levels if is_atmos else (float("nan"),)
                    rows += [(time, md.rollout_step, label, b, k, float(lv), geometry) for lv in levels]
            self._score(fields, rows, weights, device, cabi.AB_SPEC_MAX_FIELDS,
                        lambda chunk: cabi.zonal_spectra_workspace_bytes(chunk, band_rows),
                        lambda chunk, wt, out, ws: cabi.zonal_spectra(chunk, band_rows, wt, out, ws),
                        width=len(band_rows) * (w // 2 + 3))

    def results(self):
        """The spectra as a long pandas DataFrame, one row per (step call, batch member, variable, level, band,
        wavenumber), with columns time, rollout_step, label, member, variable, level (NaN for surface variables),
        band, wavenumber, wavelength_km, power and rows (counted latitude rows); label, variable and band are
        categorical.  One device-to-host copy of everything accumulated so far."""
        import pandas as pd

        s = self._host_sums()
        n = len(self._rows)
        time, step, label, member, variable, level, geometry = zip(*self._rows) if n else ((),) * 7
        nb = np.array([len(g[0]) for g in geometry], dtype=np.int64)
        nk = np.array([g[1].shape[1] for g in geometry], dtype=np.int64)
        # every plane's values are [bands][Σw, rows, Σ w P(0 .. nk - 1)]; split them into per-(band, k) columns
        lead = np.repeat(np.cumsum(np.concatenate([[0], nb * (nk + 2)]))[:-1], nb) + \
            (nk + 2).repeat(nb) * np.concatenate([np.arange(b) for b in nb] or [np.zeros(0, np.int64)])
        per_band = nk.repeat(nb)  # wavenumbers of every (plane, band)
        k = np.arange(per_band.sum()) - np.repeat(np.cumsum(per_band) - per_band, per_band)
        at = np.repeat(lead, per_band)  # index of Σw of each output row
        with np.errstate(divide="ignore", invalid="ignore"):
            power = s[at + 2 + k] / s[at]
        per_plane = nb * nk
        rep = lambda values, dtype=None: np.repeat(np.asarray(values, dtype=dtype), per_plane)  # noqa: E731

        def names(values, repeats):  # a categorical column: millions of rows, a handful of distinct strings
            categories, codes = np.unique(np.asarray(values, dtype=str), return_inverse=True)
            return pd.Categorical.from_codes(np.repeat(codes, repeats), categories=categories)

        bands = [b for g in geometry for b in g[0]]
        wavelengths = np.concatenate([g[1].reshape(-1) for g in geometry] or [np.zeros(0)])
        return pd.DataFrame({
            "time": pd.Series(rep(time, "datetime64[ns]"), dtype="datetime64[ns]"),
            "rollout_step": rep(step, np.int64), "label": names(label, per_plane),
            "member": rep(member, np.int64), "variable": names(variable, per_plane),
            "level": rep(level, np.float64), "band": names(bands, per_band),
            "wavenumber": k.astype(np.int64), "wavelength_km": wavelengths.astype(np.float64), "power": power,
            "rows": s[at + 1].astype(np.int64)})
