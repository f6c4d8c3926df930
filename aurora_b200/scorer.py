"""``Scorer``: latitude-weighted RMSE, bias, MAE and anomaly correlation of predictions against a truth (an analysis
such as ERA5 or HRES T0) and, optionally, a climatology, computed where the prediction lives.  ``EnsembleScorer``: the
probabilistic counterparts for an ensemble of predictions: ensemble-mean RMSE and bias, spread, spread-skill ratio,
the fair CRPS and the ensemble-mean ACC.

Every `step` is one `ab_score_fields` call (`csrc/score.cu`): one descriptor per variable and batch member, seven
float64 sums and a count per level plane, appended to a device tensor the scorer owns.  Nothing is read back until
`results`, which copies all accumulated sums to the host at once and forms the scores there.

Definitions, with row weights ``w_i = cos(deg2rad(lat_i))`` (float64, from the prediction's latitudes) and a point
valid when prediction, truth and (if given) climatology are all not NaN (±inf is not skipped and propagates); every
sum runs over the valid points, ``d = p - t``, ``af = p - c``, ``ao = t - c`` in float64 and ``W = Σ w``:

    rmse = sqrt(Σ w d² / W)      bias = Σ w d / W      mae = Σ w |d| / W
    acc  = Σ w af ao / sqrt(Σ w af² · Σ w ao²)         (uncentred, as WeatherBench 2; NaN for a zero denominator)

Normalising by the valid weights makes the common ``cos / mean(cos)`` convention cancel.

`EnsembleScorer.step` is one `ab_ensemble_score_fields` call per 16 variables: one descriptor per variable holding
all M members, nine float64 sums and a count per level plane.  A point is valid when the truth, every member and (if
given) the climatology are all not NaN (±inf is not skipped).  With the member values ``x_k`` (k = 1..M), their mean
``x̄`` and unbiased variance ``s² = Σ_k (x_k - x̄)² / (M - 1)`` in float64, ``y`` the truth, the same weights and
``W = Σ w`` over the valid points:

    ens_rmse    = sqrt(Σ w (x̄ - y)² / W)                ens_bias = Σ w (x̄ - y) / W
    spread      = sqrt(Σ w s² / W)                      ssr      = sqrt((M + 1) / M) · spread / ens_rmse
    crps_skill  = Σ w (1/M) Σ_k |x_k - y| / W
    crps_spread = Σ w (1/(M(M-1))) Σ_{k≠l} |x_k - x_l| / W           (the fair estimator, WeatherBench 2's CRPSSpread)
    crps        = crps_skill - crps_spread / 2
    acc         = the uncentred ACC above of x̄ against the climatology

``ssr`` is the unbiased spread-skill ratio (Fortin et al. 2014): 1 for a reliable ensemble.  The kernel sorts each
point's member values and forms everything from the sorted order, so the scores do not depend on the order of the
members, bit for bit.
"""

from __future__ import annotations

from typing import Iterable, Optional

import numpy as np
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch

__all__ = ["Scorer", "EnsembleScorer"]

COLUMNS = ("time", "rollout_step", "member", "variable", "level", "rmse", "bias", "mae", "acc", "count")
ENSEMBLE_COLUMNS = ("time", "rollout_step", "variable", "level", "members", "ens_rmse", "ens_bias", "spread", "ssr",
                    "crps", "crps_skill", "crps_spread", "acc", "count")


def _select_levels(t: torch.Tensor, idx: list[int]) -> torch.Tensor:
    """Levels `idx` of a (C, H, W) tensor: a strided view when they are evenly spaced, else a gathered copy."""
    step = idx[1] - idx[0] if len(idx) > 1 else 1
    if step > 0 and all(b - a == step for a, b in zip(idx, idx[1:])):
        return t[idx[0]:idx[-1] + 1:step]
    return t[idx]


def _layout(t: torch.Tensor) -> tuple[int, int, int, int, int]:
    """(levels, h, w, row pitch, level stride) of an (H, W) or (C, H, W) view with unit column stride."""
    levels, h, w = (1, *t.shape) if t.dim() == 2 else t.shape
    return (levels, h, w, t.stride(-2) if h > 1 else max(t.stride(-2), w),
            t.stride(0) if t.dim() == 3 and levels > 1 else 0)


def _field(pred: torch.Tensor, truth: torch.Tensor, clim: Optional[torch.Tensor]) -> cabi.AbScoreField:
    """Descriptor of (H, W) or (C, H, W) views with equal shapes."""
    f = cabi.AbScoreField()
    for name, t in (("pred", pred), ("truth", truth), ("clim", clim)):
        if t is None:
            continue
        f.levels, f.h, f.w, ld, stride = _layout(t)
        setattr(f, name, t.data_ptr())
        setattr(f, f"ld_{name}", ld)
        setattr(f, f"{name}_level_stride", stride)
    return f


def _ensemble_field(members: list[torch.Tensor], truth: torch.Tensor,
                    clim: Optional[torch.Tensor]) -> cabi.AbEnsembleField:
    """Descriptor of (H, W) or (C, H, W) views with equal shapes; the members share one row pitch and level stride."""
    f = cabi.AbEnsembleField()
    f.levels, f.h, f.w, f.ld_member, f.member_level_stride = _layout(members[0])
    f.n_members = len(members)
    for k, t in enumerate(members):
        f.members[k] = t.data_ptr()
    for name, t in (("truth", truth), ("clim", clim)):
        if t is not None:
            _, _, _, ld, stride = _layout(t)
            setattr(f, name, t.data_ptr())
            setattr(f, f"ld_{name}", ld)
            setattr(f, f"{name}_level_stride", stride)
    return f


class _StepScorer:
    """What `Scorer`, `EnsembleScorer` and `ZonalSpectra` share: the climatology and variable selection, the checks of
    a truth or climatology against a prediction, host copies of coordinates, row weights and the device sums that
    `step` appends to: one row per plane, `_SUMS` values wide unless a call says otherwise, packed end to end."""

    _SUMS = cabi.AB_SCORE_SUMS

    def __init__(self, climatology: Optional[Batch] = None, variables: Optional[Iterable[str]] = None) -> None:
        self.climatology = climatology
        self.variables = None if variables is None else tuple(variables)
        self._rows: list[tuple] = []  # one per plane
        self._sums: Optional[torch.Tensor] = None  # float64 [capacity] on the predictions' device
        self._used = 0  # values of `_sums` the rows fill
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

    def _check(self, what: str, other: Batch, pred: Batch, surf: list[str], atmos: list[str],
               b: Optional[int] = None) -> tuple[int, list]:
        """Refuse `other` (truth or climatology) unless it has the variables, levels and grid of the prediction and
        batch size `b` (by default the prediction's; 1 also for a climatology); returns its batch size and the index
        in its levels of every prediction level."""
        md, om = pred.metadata, other.metadata
        if om.lat.dim() != 1 or om.lon.dim() != 1:
            raise ValueError(f"{type(self).__name__}.step needs 1-D latitudes and longitudes (the {what}'s are not)")
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
        b = len(md.time) if b is None else b
        tensors = [other.surf_vars[k] for k in surf] + [other.atmos_vars[k] for k in atmos]
        sizes = {t.shape[0] for t in tensors}
        if not sizes <= ({b} if what == "truth" else {1, b}):
            raise ValueError(f"the {what} has batch size {sorted(sizes)}, the prediction {b}")
        for t in tensors:
            if t.dtype != torch.float32:
                raise TypeError(f"{type(self).__name__}.step needs float32 fields, the {what} has {t.dtype}")
            if t.shape[-2] != lat.size or t.shape[-1] != md.lon.numel():
                raise ValueError(f"a field of the {what} has shape {tuple(t.shape)}, its grid is "
                                 f"{lat.size} x {md.lon.numel()}")
        return sizes.pop(), [levels.index(lv) for lv in md.atmos_levels if lv in levels]

    def _append(self, n: int, device: torch.device, width: int) -> torch.Tensor:
        """`n` fresh rows of `width` values at the end of the device sums (grown by copying on the device, never read
        back), as an [n, width] view."""
        used = self._used
        if self._sums is not None and self._sums.device != device:
            raise ValueError(f"{type(self).__name__} holds scores on {self._sums.device}; "
                             f"the prediction is on {device}")
        need = used + n * width
        if self._sums is None or self._sums.numel() < need:
            cap = max(need, 256 * self._SUMS, 0 if self._sums is None else 2 * self._sums.numel())
            grown = torch.empty(cap, dtype=torch.float64, device=device)
            if used:
                grown[:used].copy_(self._sums[:used])
            self._sums = grown
        return self._sums[used:need].view(n, width)

    def _check_prediction(self, pred: Batch, what: str = "prediction") -> None:
        """Refuse a sharded or 2-D-coordinate prediction."""
        name = type(self).__name__
        if getattr(pred, "slab_plans", None) is not None:
            raise ValueError(f"{name}.step needs a whole-grid {what}; gather the latitude bands first "
                             "(aurora_b200.sharding.gather_bands)")
        if pred.metadata.lat.dim() != 1 or pred.metadata.lon.dim() != 1:
            raise ValueError(f"{name}.step needs 1-D latitudes and longitudes")

    def _check_tensors(self, pred: Batch, surf: list[str], atmos: list[str], what: str = "prediction") -> None:
        for k, t in [(k, pred.surf_vars[k]) for k in surf] + [(k, pred.atmos_vars[k]) for k in atmos]:
            if not t.is_cuda:
                raise cabi.AbError(f"{type(self).__name__}.step needs the {what} on a CUDA device ({k} is on "
                                   f"{t.device}); libaurora_b200 has no CPU path")
            if t.dtype != torch.float32:
                raise TypeError(f"{type(self).__name__}.step needs float32 fields, the {what}'s {k} is {t.dtype}")

    def _resident(self, truth: Batch, device: torch.device) -> tuple[Batch, Optional[Batch]]:
        """The truth and the climatology on `device` (the climatology copied there once); call under that device."""
        if any(t.device != device for t in list(truth.surf_vars.values()) + list(truth.atmos_vars.values())):
            truth = truth.to(device)
        clim = self.climatology
        if clim is not None:
            clim = self._clim_on.get(device)
            if clim is None:
                clim = self.climatology
                if any(t.device != device for t in list(clim.surf_vars.values()) + list(clim.atmos_vars.values())):
                    clim = clim.to(device)
                self._clim_on[device] = clim
        return truth, clim

    def _score(self, fields: list, rows: list, weights: torch.Tensor, device: torch.device, max_fields: int,
               workspace_bytes, score, width: Optional[int] = None) -> None:
        """Score `fields` in calls of at most `max_fields` into fresh rows (one per plane, `width` values, by default
        `_SUMS`) of the device sums."""
        width = self._SUMS if width is None else width
        sums = self._append(len(rows), device, width)
        done = 0
        for s0 in range(0, len(fields), max_fields):
            chunk = fields[s0:s0 + max_fields]
            nbytes = workspace_bytes(chunk)
            if self._workspace is None or self._workspace.numel() < nbytes:
                self._workspace = torch.empty(nbytes, dtype=torch.uint8, device=device)
            planes = sum(f.levels for f in chunk)
            score(chunk, weights, sums[done:done + planes], self._workspace)
            done += planes
        self._rows += rows
        self._used += len(rows) * width

    def _host_sums(self) -> np.ndarray:
        """Every value accumulated so far, flat, in one device-to-host copy."""
        return self._sums[:self._used].cpu().numpy() if self._used else np.zeros(0)


class Scorer(_StepScorer):
    """Scores predictions against a truth, step by step, without copying them to the host.

    Args:
        climatology: Optional `Batch` with the scored variables on the truth's levels and grid; its last history
            slice is the climatology of every step (batch size 1, or that of the predictions).  Needed for `acc`.
            A climatology that is not on the predictions' device is copied there once with `Batch.to`.
        variables: Surface / atmospheric variable names to score.  By default every variable present in both the
            prediction and the truth.  Static variables are never scored.
    """

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
        self._check_prediction(pred)
        if tuple(truth.metadata.time) != tuple(md.time):
            raise ValueError(f"the truth is valid at {tuple(truth.metadata.time)}, "
                             f"the prediction at {tuple(md.time)}")
        surf, atmos = self._names(pred, truth)
        _, truth_levels = self._check("truth", truth, pred, surf, atmos)
        clim = self.climatology
        if clim is not None:
            clim_b, clim_levels = self._check("climatology", clim, pred, surf, atmos)
        self._check_tensors(pred, surf, atmos)
        device = pred.surf_vars[surf[0]].device if surf else pred.atmos_vars[atmos[0]].device
        h = md.lat.numel()

        with torch.cuda.device(device):
            truth, clim = self._resident(truth, device)
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

            self._score(fields, rows, weights, device, cabi.AB_SCORE_MAX_FIELDS, cabi.score_workspace_bytes,
                        cabi.score_fields)

    def results(self):
        """The scores as a pandas DataFrame, one row per (step call, batch member, variable, level), with columns
        time, rollout_step, member, variable, level (NaN for surface variables), rmse, bias, mae, acc (NaN without a
        climatology) and count (valid points).  One device-to-host copy of every sum accumulated so far."""
        import pandas as pd

        n = len(self._rows)
        s = self._host_sums().reshape(-1, self._SUMS)
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


class EnsembleScorer(_StepScorer):
    """Scores an ensemble of predictions against a truth, step by step, without copying them to the host.

    Args:
        climatology: Optional `Batch` of batch size 1 with the scored variables on the truth's levels and grid; its
            last history slice is the climatology of every step.  Needed for `acc`.  A climatology that is not on the
            members' device is copied there once with `Batch.to`.
        variables: Surface / atmospheric variable names to score.  By default every variable present in both the
            members and the truth.  Static variables are never scored.
    """

    _SUMS = cabi.AB_ENS_SUMS

    def step(self, members, truth: Batch) -> None:
        """Score one step of an ensemble.  Enqueues the work on the current stream; nothing is read back.

        Args:
            members: A `Batch` or a sequence of `Batch`es as `Aurora.forward` returns them, on one CUDA device, with
                1-D coordinates and whole grids.  The ensemble is every batch entry of every `Batch`, so one forward
                with batch size M and M roll-outs of batch size 1 describe the same ensemble.  All members must share
                the valid time, `rollout_step`, grid, levels and variables; 2 <= M <= 64.
            truth: A `Batch` of batch size 1 valid at the members' time, as `Scorer.step` takes it.
        """
        name = type(self).__name__
        members = [members] if isinstance(members, Batch) else list(members)
        if not members:
            raise ValueError(f"{name}.step needs at least one Batch of members")
        for b in members:
            self._check_prediction(b, "member")
        first = members[0]
        md = first.metadata
        m = sum(len(b.metadata.time) for b in members)
        if m < 2:
            raise ValueError(f"{name}.step needs at least 2 members, got {m}")
        if m > cabi.AB_ENS_MAX_MEMBERS:
            raise ValueError(f"{name}.step scores at most {cabi.AB_ENS_MAX_MEMBERS} members, got {m}")
        times = sorted({t for b in members for t in b.metadata.time})
        if len(times) != 1:
            raise ValueError(f"the members are valid at different times: {times}")
        for i, b in enumerate(members[1:], 1):
            bm = b.metadata
            if bm.rollout_step != md.rollout_step:
                raise ValueError(f"members differ in rollout_step: {md.rollout_step} and {bm.rollout_step} "
                                 f"(Batch {i})")
            if (not np.array_equal(self._coords(bm.lat), self._coords(md.lat))
                    or not np.array_equal(self._coords(bm.lon), self._coords(md.lon))):
                raise ValueError(f"members differ in grid: Batch {i}'s latitudes or longitudes are not Batch 0's")
            if tuple(bm.atmos_levels) != tuple(md.atmos_levels):
                raise ValueError(f"members differ in levels: {tuple(md.atmos_levels)} and {tuple(bm.atmos_levels)} "
                                 f"(Batch {i})")
            if list(b.surf_vars) != list(first.surf_vars) or list(b.atmos_vars) != list(first.atmos_vars):
                raise ValueError(f"members differ in variables: {list(first.surf_vars) + list(first.atmos_vars)} "
                                 f"and {list(b.surf_vars) + list(b.atmos_vars)} (Batch {i})")
        surf, atmos = self._names(first, truth)
        for what, other in (("truth", truth), ("climatology", self.climatology)):
            sizes = set() if other is None else {t.shape[0] for d in (other.surf_vars, other.atmos_vars)
                                                 for k, t in d.items() if k in surf + atmos}
            if sizes - {1}:
                raise ValueError(f"{name}.step needs a {what} of batch size 1, it has {sorted(sizes)}")
        if tuple(truth.metadata.time) != (times[0],):
            raise ValueError(f"the truth is valid at {tuple(truth.metadata.time)}, the members at {times[0]}")
        _, truth_levels = self._check("truth", truth, first, surf, atmos, b=1)
        clim = self.climatology
        if clim is not None:
            _, clim_levels = self._check("climatology", clim, first, surf, atmos, b=1)
        for b in members:
            self._check_tensors(b, surf, atmos, "member")
        device = first.surf_vars[surf[0]].device if surf else first.atmos_vars[atmos[0]].device
        for b in members:
            for k, t in [(k, b.surf_vars[k]) for k in surf] + [(k, b.atmos_vars[k]) for k in atmos]:
                if t.device != device:
                    raise ValueError(f"members are on {device} and {t.device} ({k})")
        h = md.lat.numel()

        with torch.cuda.device(device):
            truth, clim = self._resident(truth, device)
            weights = self._row_weights(md.lat, device)
            fields, rows, keep = [], [], []
            for k in surf + atmos:
                is_atmos = k in atmos
                group = "atmos_vars" if is_atmos else "surf_vars"
                xs = [getattr(b, group)[k][j, -1] for b in members for j in range(len(b.metadata.time))]
                xs = [x if x.stride(-1) == 1 else x.contiguous() for x in xs]
                if any(_layout(x)[3:] != _layout(xs[0])[3:] for x in xs):
                    xs = [x.contiguous() for x in xs]  # one row pitch and level stride for all members
                t = getattr(truth, group)[k][0, -1]
                c = None if clim is None else getattr(clim, group)[k][0, -1]
                if is_atmos:
                    t = _select_levels(t, truth_levels)
                    c = None if c is None else _select_levels(c, clim_levels)
                t, c = [v if v is None or v.stride(-1) == 1 else v.contiguous()
                        for v in (t[..., :h, :], None if c is None else c[..., :h, :])]
                keep += xs + [t, c]
                fields.append(_ensemble_field(xs, t, c))
                levels = md.atmos_levels if is_atmos else (float("nan"),)
                rows += [(times[0], md.rollout_step, k, float(lv), m, clim is not None) for lv in levels]
            self._score(fields, rows, weights, device, cabi.AB_ENS_MAX_FIELDS, cabi.ensemble_score_workspace_bytes,
                        cabi.ensemble_score_fields)

    def results(self):
        """The scores as a pandas DataFrame, one row per (step call, variable, level), with columns time,
        rollout_step, variable, level (NaN for surface variables), members, ens_rmse, ens_bias, spread, ssr, crps,
        crps_skill, crps_spread, acc (NaN without a climatology) and count (valid points).  One device-to-host copy
        of every sum accumulated so far."""
        import pandas as pd

        n = len(self._rows)
        s = self._host_sums().reshape(-1, self._SUMS)
        time, step, variable, level, members, has_clim = zip(*self._rows) if n else ((),) * 6
        m = np.asarray(members, dtype=np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            w = s[:, 0]
            rmse, spread = np.sqrt(s[:, 2] / w), np.sqrt(s[:, 3] / w)
            skill, pair = s[:, 4] / w, s[:, 5] / w
            den = np.sqrt(s[:, 7] * s[:, 8])
            acc = np.where(np.asarray(has_clim, dtype=bool) & (den != 0), s[:, 6] / den, np.nan)
            return pd.DataFrame({
                "time": pd.Series(list(time), dtype="datetime64[ns]"),
                "rollout_step": np.asarray(step, dtype=np.int64),
                "variable": pd.Series(list(variable), dtype="str"), "level": np.asarray(level, dtype=np.float64),
                "members": np.asarray(members, dtype=np.int64),
                "ens_rmse": rmse, "ens_bias": s[:, 1] / w, "spread": spread,
                "ssr": np.sqrt((m + 1) / m) * spread / rmse, "crps": skill - pair / 2, "crps_skill": skill,
                "crps_spread": pair, "acc": acc, "count": s[:, 9].astype(np.int64)})
