"""``Tracker``: tropical-cyclone tracking on predictions that stay on the GPU, track for track with the reference's
tracker (`aurora/tracker.py:123-282`).

The field work — gathering the boxes around a position, the Gaussian smoothing and 8 x 8 minimum filter that find the
local minima of msl / z700, the land test and the msl / wind crop — runs in `ab_track_boxes` (`csrc/tracker.cu`), which
writes a uint8 mask or a single value per box.  The scalar decisions stay here, in numpy, with the reference's numpy
types: the extrapolated guess, the box bounds, the distances to the minima, the delta cascade, the z700 fallback and
the failure counter.  A step makes at most three launches, each followed by one small read-back into pinned memory:

1. around the guess, speculatively: msl minima and the land maximum for every delta, and the z700 minima at delta 5;
2. only when msl finds no eye but z700 does: msl minima and the land maximum around the z700 position;
3. the msl minimum and the wind-speed maximum around the final position.

No field plane leaves the device; latitudes and longitudes are copied to the host once per grid.
"""

from __future__ import annotations

import logging
from datetime import datetime
from typing import Optional

import numpy as np
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch

__all__ = ["Tracker", "NoEyeException"]

logger = logging.getLogger(__name__)

DELTAS = (5, 4, 3, 2, 1.5)  # box half-widths in degrees, tried largest first (tracker.py:202, 233)
Z700_DELTA = 5  # (tracker.py:222-230)
CROP_DELTA = 1.5  # msl / wind crop around the final position (tracker.py:262-280)


class NoEyeException(Exception):
    """Raised when no eye can be found."""


def _box_indices(lats: np.ndarray, lons: np.ndarray, lat, lon, delta) -> tuple[np.ndarray, np.ndarray]:
    """Row and column index lists of the box [lat - delta, lat + delta] x [lon - delta, lon + delta] (tracker.py:21-49).
    The bounds keep the numpy type of `lat` / `lon`, so under NEP 50 a Python float is compared in the grid's float32
    and an np.float64 in float64, as in the reference.  A longitude range that wraps past 360 lists the columns from
    its lower bound to the end first, then those from 0."""
    lat_min, lat_max = lat - delta, lat + delta
    rows = np.flatnonzero((lat_min <= lats) & (lats <= lat_max))
    lon_min, lon_max = (lon - delta) % 360, (lon + delta) % 360
    if lon_min <= lon_max:
        cols = np.flatnonzero((lon_min <= lons) & (lons <= lon_max))
    else:
        cols = np.concatenate((np.flatnonzero(lon_min <= lons), np.flatnonzero(lons <= lon_max)))
    return rows, cols


def _haversine_km(lat1, lon1, lat2, lon2):
    """Great-circle distance in km (tracker.py:52-58), with the reference's operations in its order so that the
    distances, and therefore the closest minimum, round the same way."""
    lat1, lat2 = np.deg2rad(lat1), np.deg2rad(lat2)
    lon1, lon2 = np.deg2rad(lon1), np.deg2rad(lon2)
    inner = 1 - np.cos(lat2 - lat1) + np.cos(lat1) * np.cos(lat2) * (1 - np.cos(lon2 - lon1))
    return 2 * 6371 * np.arcsin(np.sqrt(0.5 * inner))


def _extrapolate(lats: list, lons: list):
    """First guess for the next position (tracker.py:107-120): the last position after one step, else the degree-1
    least-squares line through the last eight positions evaluated one step ahead (np.float64).  Longitude is not
    unwrapped, like the reference: a track crossing 0 degrees E extrapolates through the jump."""
    if len(lats) == 1:
        return lats[0], lons[0]
    n = min(len(lats), 8)
    fit = np.polyfit(np.arange(n), np.stack((lats[-n:], lons[-n:]), axis=-1), 1)
    lat, lon = np.polyval(fit, n)
    return lat, lon


def _raise_like_empty_reduction(shape: tuple[int, int], reduction: str) -> None:
    """The reference reduces an empty crop with numpy and fails there; fail with numpy's own error."""
    getattr(np.empty(shape, dtype=np.float32), reduction)()


def _raise_like_empty_minima(shape: tuple[int, int]) -> None:
    """The reference's border clearing on an empty box (tracker.py:90-93) raises numpy's IndexError; so do we."""
    m = np.zeros(shape, dtype=bool)
    m[0, :], m[-1, :], m[:, 0], m[:, -1] = 0, 0, 0, 0


class _Plane:
    """A float32 field plane on the device, as `ab_track_boxes` addresses it."""

    def __init__(self, name: str, t: torch.Tensor, shape: tuple[int, int]):
        if not t.is_cuda:
            raise cabi.AbError(f"Tracker.step needs the prediction on a CUDA device ({name} is on {t.device}); "
                               "libaurora_b200 has no CPU path")
        if t.dtype != torch.float32:
            raise TypeError(f"Tracker.step needs float32 fields, {name} is {t.dtype}")
        if tuple(t.shape) != shape:
            raise ValueError(f"{name} has shape {tuple(t.shape)}, the grid is {shape}")
        if t.stride(1) != 1:
            t = t.contiguous()
        self.t, self.h, self.w = t, shape[0], shape[1]
        self.ld = t.stride(0) if self.h > 1 else self.w


class _Launch:
    """The boxes of one `ab_track_boxes` launch and their read-back."""

    def __init__(self, tracker: "Tracker", device: torch.device):
        self.tracker, self.device = tracker, device
        self.boxes: list = []
        self.index: list[np.ndarray] = []
        self.n_index = 0
        self.mask_bytes = 0
        self.shapes: list[tuple[int, int]] = []
        self.mask_offs: list[int] = []

    def add(self, op: int, plane: _Plane, rows: np.ndarray, cols: np.ndarray, plane2: Optional[_Plane] = None):
        """Queue a box; returns its slot, or None for an empty box (which is never launched)."""
        if rows.size == 0 or cols.size == 0:
            return None
        b = cabi.AbTrackBox(plane=plane.t.data_ptr(), plane2=None if plane2 is None else plane2.t.data_ptr(),
                            h=plane.h, w=plane.w, ld=plane.ld, op=op, rows_off=self.n_index, n_rows=rows.size,
                            cols_off=self.n_index + rows.size, n_cols=cols.size)
        self.index += [rows, cols]
        self.n_index += rows.size + cols.size
        self.shapes.append((rows.size, cols.size))
        self.mask_offs.append(self.mask_bytes)
        if op == cabi.AB_TRACK_MINIMA:
            b.mask_off = self.mask_bytes
            self.mask_bytes += rows.size * cols.size
        self.boxes.append(b)
        return len(self.boxes) - 1

    def run(self) -> "_Results":
        n = len(self.boxes)
        if n == 0:
            return _Results(np.empty(0, np.float32), np.empty(0, np.int32), np.empty(0, np.uint8), [], [])
        idx = self.tracker._pinned("index", 4 * self.n_index).view(torch.int32)
        idx.numpy()[:] = np.concatenate(self.index)
        index = idx.to(self.device, non_blocking=True)
        nbytes = 8 * n + self.mask_bytes
        out = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        values, counts = out[:4 * n].view(torch.float32), out[4 * n:8 * n].view(torch.int32)
        masks = out[8 * n:] if self.mask_bytes else None
        cabi.track_boxes(self.boxes, index, values, counts, masks)
        host = self.tracker._pinned("out", nbytes)
        host.copy_(out, non_blocking=True)
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
        h = host.numpy()
        res = _Results(h[:4 * n].view(np.float32).copy(), h[4 * n:8 * n].view(np.int32).copy(), h[8 * n:].copy(),
                       self.shapes, self.mask_offs)
        if (res.counts < 0).any():
            raise cabi.AbError("ab_track_boxes: an index lies outside its field plane")
        return res


class _Results:
    def __init__(self, values, counts, masks, shapes, mask_offs):
        self.values, self.counts, self.masks, self.shapes, self.mask_offs = values, counts, masks, shapes, mask_offs

    def mask(self, slot: int) -> np.ndarray:
        nr, nc = self.shapes[slot]
        return self.masks[self.mask_offs[slot]:self.mask_offs[slot] + nr * nc].reshape(nr, nc)


class Tracker:
    """Simple tropical-cyclone tracker with the reference's interface and results (`aurora/tracker.py:123-282`; the
    algorithm is Anna Allen's design as implemented by Wessel Bruinsma).

    Args:
        init_lat: Latitude of the cyclone at `init_time`.
        init_lon: Longitude of the cyclone at `init_time`.
        init_time: Time of the initial condition.
    """

    def __init__(self, init_lat: float, init_lon: float, init_time: datetime) -> None:
        self.tracked_times: list[datetime] = [init_time]
        self.tracked_lats: list[float] = [init_lat]
        self.tracked_lons: list[float] = [init_lon]
        self.tracked_msls: list[float] = [np.nan]
        self.tracked_winds: list[float] = [np.nan]
        self.fails: int = 0
        self._grid_key = None
        self._lats = self._lons = None
        self._host: dict[str, torch.Tensor] = {}

    def results(self):
        """The track as a pandas DataFrame with columns time, lat, lon, msl and wind."""
        import pandas as pd

        return pd.DataFrame({"time": self.tracked_times, "lat": self.tracked_lats, "lon": self.tracked_lons,
                             "msl": self.tracked_msls, "wind": self.tracked_winds})

    # -- helpers ----------------------------------------------------------------------------------------------------
    def _pinned(self, name: str, nbytes: int) -> torch.Tensor:
        buf = self._host.get(name)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(nbytes, 4096), dtype=torch.uint8, pin_memory=True)
            self._host[name] = buf
        return buf[:nbytes]

    def _grid(self, lat: torch.Tensor, lon: torch.Tensor) -> tuple[np.ndarray, np.ndarray]:
        """Host copies of the coordinates, made once per grid (the rollout hands every prediction the same tensors)."""
        if self._grid_key is None or self._grid_key[0] is not lat or self._grid_key[1] is not lon:
            self._lats, self._lons = lat.detach().cpu().numpy(), lon.detach().cpu().numpy()
            self._grid_key = (lat, lon)
        return self._lats, self._lons

    def _queue_cascade(self, launch: _Launch, msl: _Plane, lsm: _Plane, lat, lon) -> list:
        out = []
        for delta in DELTAS:
            rows, cols = _box_indices(self._lats, self._lons, lat, lon, delta)
            out.append((rows, cols, launch.add(cabi.AB_TRACK_MAX, lsm, rows, cols),
                        launch.add(cabi.AB_TRACK_MINIMA, msl, rows, cols)))
        return out

    def _closest_min(self, res: _Results, slot, rows: np.ndarray, cols: np.ndarray, lat, lon):
        """The local minimum of the box closest to (lat, lon), first in row-major order among equals
        (tracker.py:95-104), or None when the box has none."""
        if slot is None:
            _raise_like_empty_minima((rows.size, cols.size))
        if res.counts[slot] == 0:
            return None
        box_lats, box_lons = self._lats[rows], self._lons[cols]
        r, c = np.nonzero(res.mask(slot))
        i = np.argmin(_haversine_km(box_lats[r], box_lons[c], lat, lon))
        return box_lats[r[i]], box_lons[c[i]]

    def _cascade(self, res: _Results, queued: list, lat, lon):
        """First delta whose box is clear of land (max lsm < 0.5) and has an msl minimum (tracker.py:201-217)."""
        for rows, cols, land, slot in queued:
            if land is None:
                _raise_like_empty_reduction((rows.size, cols.size), "max")
            if res.values[land] < 0.5:
                hit = self._closest_min(res, slot, rows, cols, lat, lon)
                if hit is not None:
                    return hit
        return None

    # -- public -----------------------------------------------------------------------------------------------------
    def step(self, batch: Batch) -> None:
        """Track the next step.

        Args:
            batch: Prediction (batch size one), on a CUDA device, with 700 hPa among its levels.
        """
        if len(batch.metadata.time) != 1:
            raise RuntimeError("Predictions don't have batch size one.")
        if getattr(batch, "slab_plans", None) is not None:
            raise ValueError("Tracker.step needs a whole-grid prediction; gather the latitude bands first "
                             "(aurora_b200.sharding.gather_bands)")
        md = batch.metadata
        z700_index = list(md.atmos_levels).index(700)
        if md.lat.dim() != 1 or md.lon.dim() != 1:
            raise ValueError("Tracker.step needs 1-D latitudes and longitudes")
        shape = (md.lat.numel(), md.lon.numel())
        z700 = _Plane("z at 700 hPa", batch.atmos_vars["z"][0, 0, z700_index], shape)
        msl = _Plane("msl", batch.surf_vars["msl"][0, 0], shape)
        u10 = _Plane("10u", batch.surf_vars["10u"][0, 0], shape)
        v10 = _Plane("10v", batch.surf_vars["10v"][0, 0], shape)
        lsm = _Plane("lsm", batch.static_vars["lsm"], shape)
        time = md.time[0]
        device = msl.t.device

        with torch.cuda.device(device):
            lats, lons = self._grid(md.lat, md.lon)
            lat, lon = _extrapolate(self.tracked_lats, self.tracked_lons)
            lat = max(min(lat, 90), -90)
            lon = lon % 360

            launch = _Launch(self, device)
            queued = self._queue_cascade(launch, msl, lsm, lat, lon)
            z_rows, z_cols = _box_indices(lats, lons, lat, lon, Z700_DELTA)
            z_slot = launch.add(cabi.AB_TRACK_MINIMA, z700, z_rows, z_cols)
            res = launch.run()

            hit = self._cascade(res, queued, lat, lon)
            snap = hit is not None
            if snap:
                lat, lon = hit
            else:
                # msl found no eye: take the z700 minimum and refine it with msl where possible (tracker.py:219-249)
                hit = self._closest_min(res, z_slot, z_rows, z_cols, lat, lon)
                if hit is not None:
                    lat, lon = hit
                    snap = True
                    launch = _Launch(self, device)
                    queued = self._queue_cascade(launch, msl, lsm, lat, lon)
                    refined = self._cascade(launch.run(), queued, lat, lon)
                    if refined is not None:
                        lat, lon = refined

            if not snap:
                self.fails += 1
                if len(self.tracked_lats) > 1:
                    logger.info(f"Failed at time {time}. Extrapolating in a silly way.")
                else:
                    raise NoEyeException("Completely failed at the first step.")

            self.tracked_times.append(time)
            self.tracked_lats.append(lat)
            self.tracked_lons.append(lon)

            rows, cols = _box_indices(lats, lons, lat, lon, CROP_DELTA)
            if rows.size == 0 or cols.size == 0:
                _raise_like_empty_reduction((rows.size, cols.size), "min")
            launch = _Launch(self, device)
            msl_slot = launch.add(cabi.AB_TRACK_MIN, msl, rows, cols)
            wind_slot = launch.add(cabi.AB_TRACK_WINDMAX, u10, rows, cols, plane2=v10)
            res = launch.run()
            self.tracked_msls.append(res.values[msl_slot])
            self.tracked_winds.append(res.values[wind_slot])
