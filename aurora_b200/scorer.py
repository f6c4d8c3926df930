"""``Scorer``: latitude-weighted RMSE, bias, MAE and anomaly correlation of predictions against a truth (an analysis
such as ERA5 or HRES T0) and, optionally, a climatology, computed where the prediction lives.

Every `step` is one `ab_score_fields` call (`csrc/score.cu`): one descriptor per variable and batch member, seven
float64 sums and a count per level plane, appended to a device tensor the scorer owns.  Nothing is read back until
`results`, which copies all accumulated sums to the host at once and forms the scores there.

Definitions, with row weights ``w_i = cos(deg2rad(lat_i))`` (float64, from the prediction's latitudes) and a point
valid when prediction, truth and (if given) climatology are all not NaN (±inf is not skipped and propagates); every
sum runs over the valid points, ``d = p - t``, ``af = p - c``, ``ao = t - c`` in float64 and ``W = Σ w``:

    rmse = sqrt(Σ w d² / W)      bias = Σ w d / W      mae = Σ w |d| / W
    acc  = Σ w af ao / sqrt(Σ w af² · Σ w ao²)         (uncentred, as WeatherBench 2; NaN for a zero denominator)

Normalising by the valid weights makes the common ``cos / mean(cos)`` convention cancel.
"""

from __future__ import annotations

from typing import Iterable, Optional

import numpy as np
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch

__all__ = ["Scorer"]

COLUMNS = ("time", "rollout_step", "member", "variable", "level", "rmse", "bias", "mae", "acc", "count")


def _select_levels(t: torch.Tensor, idx: list[int]) -> torch.Tensor:
    """Levels `idx` of a (C, H, W) tensor: a strided view when they are evenly spaced, else a gathered copy."""
    step = idx[1] - idx[0] if len(idx) > 1 else 1
    if step > 0 and all(b - a == step for a, b in zip(idx, idx[1:])):
        return t[idx[0]:idx[-1] + 1:step]
    return t[idx]


def _field(pred: torch.Tensor, truth: torch.Tensor, clim: Optional[torch.Tensor]) -> cabi.AbScoreField:
    """Descriptor of (H, W) or (C, H, W) views with equal shapes."""
    f = cabi.AbScoreField()
    for name, t in (("pred", pred), ("truth", truth), ("clim", clim)):
        if t is None:
            continue
        levels, h, w = (1, *t.shape) if t.dim() == 2 else t.shape
        setattr(f, name, t.data_ptr())
        setattr(f, f"ld_{name}", t.stride(-2) if h > 1 else max(t.stride(-2), w))
        setattr(f, f"{name}_level_stride", t.stride(0) if t.dim() == 3 and levels > 1 else 0)
        f.h, f.w, f.levels = h, w, levels
    return f


class Scorer:
    """Scores predictions against a truth, step by step, without copying them to the host.

    Args:
        climatology: Optional `Batch` with the scored variables on the truth's levels and grid; its last history
            slice is the climatology of every step (batch size 1, or that of the predictions).  Needed for `acc`.
            A climatology that is not on the predictions' device is copied there once with `Batch.to`.
        variables: Surface / atmospheric variable names to score.  By default every variable present in both the
            prediction and the truth.  Static variables are never scored.
    """

    def __init__(self, climatology: Optional[Batch] = None, variables: Optional[Iterable[str]] = None) -> None:
        self.climatology = climatology
        self.variables = None if variables is None else tuple(variables)
        self._rows: list[tuple] = []  # (time, rollout_step, member, variable, level, with climatology) per plane
        self._sums: Optional[torch.Tensor] = None  # float64 [capacity, 8] on the predictions' device
        self._workspace: Optional[torch.Tensor] = None
        self._host: dict[int, tuple[torch.Tensor, np.ndarray]] = {}  # coordinate tensors seen, by identity
        self._weights: dict[tuple, torch.Tensor] = {}
        self._clim_on: dict[torch.device, Batch] = {}

    # -- helpers ----------------------------------------------------------------------------------------------------
    def _coords(self, t: torch.Tensor) -> np.ndarray:
        """Host copy of a coordinate vector, made once per tensor (the rollout hands every prediction the same one)."""
        hit = self._host.get(id(t))
        if hit is None or hit[0] is not t:
            hit = (t, t.detach().cpu().numpy())
            self._host[id(t)] = hit
        return hit[1]

    def _row_weights(self, lat: torch.Tensor, device: torch.device) -> torch.Tensor:
        key = (id(lat), device)
        w = self._weights.get(key)
        if w is None:
            w = torch.from_numpy(np.cos(np.deg2rad(self._coords(lat).astype(np.float64)))).to(device)
            self._weights[key] = w
        return w

    def _names(self, pred: Batch, truth: Batch) -> tuple[list[str], list[str]]:
        if self.variables is None:
            surf = [k for k in pred.surf_vars if k in truth.surf_vars]
            atmos = [k for k in pred.atmos_vars if k in truth.atmos_vars]
        else:
            surf = [k for k in self.variables if k in pred.surf_vars]
            atmos = [k for k in self.variables if k in pred.atmos_vars]
            unknown = [k for k in self.variables if k not in surf and k not in atmos]
            if unknown:
                raise ValueError(f"{unknown} are not surface or atmospheric variables of the prediction")
        if not surf and not atmos:
            raise ValueError("the prediction and the truth have no variable in common to score")
        return surf, atmos

    def _check(self, what: str, other: Batch, pred: Batch, surf: list[str], atmos: list[str]) -> tuple[int, list]:
        """Refuse `other` (truth or climatology) unless it has the variables, levels and grid of the prediction;
        returns its batch size and the index in its levels of every prediction level."""
        md, om = pred.metadata, other.metadata
        if om.lat.dim() != 1 or om.lon.dim() != 1:
            raise ValueError(f"Scorer.step needs 1-D latitudes and longitudes (the {what}'s are not)")
        for group, names in (("surf_vars", surf), ("atmos_vars", atmos)):
            missing = [k for k in names if k not in getattr(other, group)]
            if missing:
                raise ValueError(f"the {what} lacks the variables {missing}")
        h = md.lat.numel()
        lat = self._coords(om.lat)
        if lat.size not in (h, h + 1):
            raise ValueError(f"the {what} has {lat.size} latitudes, the prediction {h} (one more is cropped)")
        if not np.array_equal(lat[:h], self._coords(md.lat)):
            raise ValueError(f"the {what}'s latitudes differ from the prediction's")
        if not np.array_equal(self._coords(om.lon), self._coords(md.lon)):
            raise ValueError(f"the {what}'s longitudes differ from the prediction's")
        levels = list(om.atmos_levels)
        missing = [lv for lv in md.atmos_levels if lv not in levels]
        if atmos and missing:
            raise ValueError(f"the {what} lacks the pressure levels {missing} of the prediction")
        b = len(md.time)
        tensors = [other.surf_vars[k] for k in surf] + [other.atmos_vars[k] for k in atmos]
        sizes = {t.shape[0] for t in tensors}
        if not sizes <= ({b} if what == "truth" else {1, b}):
            raise ValueError(f"the {what} has batch size {sorted(sizes)}, the prediction {b}")
        for t in tensors:
            if t.dtype != torch.float32:
                raise TypeError(f"Scorer.step needs float32 fields, the {what} has {t.dtype}")
            if t.shape[-2] != lat.size or t.shape[-1] != md.lon.numel():
                raise ValueError(f"a field of the {what} has shape {tuple(t.shape)}, its grid is "
                                 f"{lat.size} x {md.lon.numel()}")
        return sizes.pop(), [levels.index(lv) for lv in md.atmos_levels if lv in levels]

    def _append(self, n: int, device: torch.device) -> torch.Tensor:
        """`n` fresh rows at the end of the device sums (grown by copying on the device, never read back)."""
        used = len(self._rows)
        if self._sums is not None and self._sums.device != device:
            raise ValueError(f"Scorer holds scores on {self._sums.device}; the prediction is on {device}")
        if self._sums is None or self._sums.shape[0] < used + n:
            cap = max(used + n, 256, 0 if self._sums is None else 2 * self._sums.shape[0])
            grown = torch.empty(cap, cabi.AB_SCORE_SUMS, dtype=torch.float64, device=device)
            if used:
                grown[:used].copy_(self._sums[:used])
            self._sums = grown
        return self._sums[used:used + n]

    # -- public -----------------------------------------------------------------------------------------------------
    def step(self, pred: Batch, truth: Batch) -> None:
        """Score one prediction.  Enqueues the work on the current stream; nothing is read back.

        Args:
            pred: A prediction as `Aurora.forward` returns it, on a CUDA device, with 1-D coordinates and whole
                grids.  Every batch member is scored separately.
            truth: A `Batch` valid at the prediction's time, with its variables, every level of the prediction and
                its grid (a truth with one latitude more, like the 721-row 0.25-degree grid, is cropped as
                `Batch.crop` does).  Its last history slice is used.  It is read where it lives when that is the
                prediction's device; otherwise it is first copied there whole with `Batch.to` (at 0.25 degrees about
                0.3 GB per history slice, which costs far more than the scoring itself).
        """
        md = pred.metadata
        if getattr(pred, "slab_plans", None) is not None:
            raise ValueError("Scorer.step needs a whole-grid prediction; gather the latitude bands first "
                             "(aurora_b200.sharding.gather_bands)")
        if md.lat.dim() != 1 or md.lon.dim() != 1:
            raise ValueError("Scorer.step needs 1-D latitudes and longitudes")
        if tuple(truth.metadata.time) != tuple(md.time):
            raise ValueError(f"the truth is valid at {tuple(truth.metadata.time)}, "
                             f"the prediction at {tuple(md.time)}")
        surf, atmos = self._names(pred, truth)
        _, truth_levels = self._check("truth", truth, pred, surf, atmos)
        clim = self.climatology
        if clim is not None:
            clim_b, clim_levels = self._check("climatology", clim, pred, surf, atmos)
        for k, t in [(k, pred.surf_vars[k]) for k in surf] + [(k, pred.atmos_vars[k]) for k in atmos]:
            if not t.is_cuda:
                raise cabi.AbError(f"Scorer.step needs the prediction on a CUDA device ({k} is on {t.device}); "
                                   "libaurora_b200 has no CPU path")
            if t.dtype != torch.float32:
                raise TypeError(f"Scorer.step needs float32 fields, the prediction's {k} is {t.dtype}")
        device = pred.surf_vars[surf[0]].device if surf else pred.atmos_vars[atmos[0]].device
        h = md.lat.numel()

        with torch.cuda.device(device):
            if any(t.device != device for t in list(truth.surf_vars.values()) + list(truth.atmos_vars.values())):
                truth = truth.to(device)
            if clim is not None:
                clim = self._clim_on.get(device)
                if clim is None:
                    clim = self.climatology
                    if any(t.device != device for t in list(clim.surf_vars.values()) + list(clim.atmos_vars.values())):
                        clim = clim.to(device)
                    self._clim_on[device] = clim
            weights = self._row_weights(md.lat, device)

            fields, rows, keep = [], [], []
            for b, time in enumerate(md.time):
                for k in surf + atmos:
                    is_atmos = k in atmos
                    group = "atmos_vars" if is_atmos else "surf_vars"
                    p = getattr(pred, group)[k][b, -1]
                    t = getattr(truth, group)[k][b, -1]
                    c = None if clim is None else getattr(clim, group)[k][min(b, clim_b - 1), -1]
                    if is_atmos:
                        t = _select_levels(t, truth_levels)
                        c = None if c is None else _select_levels(c, clim_levels)
                    views = [v if v is None or v.stride(-1) == 1 else v.contiguous()
                             for v in (p, t[..., :h, :], None if c is None else c[..., :h, :])]
                    keep += views
                    fields.append(_field(*views))
                    levels = md.atmos_levels if is_atmos else (float("nan"),)
                    rows += [(time, md.rollout_step, b, k, float(lv), clim is not None) for lv in levels]

            sums = self._append(len(rows), device)
            done = 0
            for s0 in range(0, len(fields), cabi.AB_SCORE_MAX_FIELDS):
                chunk = fields[s0:s0 + cabi.AB_SCORE_MAX_FIELDS]
                nbytes = cabi.score_workspace_bytes(chunk)
                if self._workspace is None or self._workspace.numel() < nbytes:
                    self._workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)
                planes = sum(f.levels for f in chunk)
                cabi.score_fields(chunk, weights, sums[done:done + planes], self._workspace)
                done += planes
            self._rows += rows

    def results(self):
        """The scores as a pandas DataFrame, one row per (step call, batch member, variable, level), with columns
        time, rollout_step, member, variable, level (NaN for surface variables), rmse, bias, mae, acc (NaN without a
        climatology) and count (valid points).  One device-to-host copy of every sum accumulated so far."""
        import pandas as pd

        n = len(self._rows)
        s = self._sums[:n].cpu().numpy() if n else np.zeros((0, cabi.AB_SCORE_SUMS))
        time, step, member, variable, level, has_clim = zip(*self._rows) if n else ((),) * 6
        with np.errstate(divide="ignore", invalid="ignore"):
            w = s[:, 0]
            den = np.sqrt(s[:, 5] * s[:, 6])
            acc = np.where(np.asarray(has_clim, dtype=bool) & (den != 0), s[:, 4] / den, np.nan)
            return pd.DataFrame({
                "time": pd.Series(list(time), dtype="datetime64[ns]"),
                "rollout_step": np.asarray(step, dtype=np.int64), "member": np.asarray(member, dtype=np.int64),
                "variable": pd.Series(list(variable), dtype="str"), "level": np.asarray(level, dtype=np.float64),
                "rmse": np.sqrt(s[:, 2] / w), "bias": s[:, 1] / w, "mae": s[:, 3] / w, "acc": acc,
                "count": s[:, 7].astype(np.int64)})
