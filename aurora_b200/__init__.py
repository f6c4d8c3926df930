"""aurora_b200 — Hopper (H100, sm_90a) implementation of Aurora's forward pass behind the reference's API
(`aurora/__init__.py:3-30`): ``Aurora*`` model classes, ``Batch``, ``Metadata``, ``rollout`` and ``Tracker``,
plus ``Scorer`` and ``EnsembleScorer``, which score predictions and ensembles against an analysis on the GPU, and
``ZonalSpectra``, which takes their latitude-band zonal power spectra there."""

from aurora_b200.batch import Batch, Metadata
from aurora_b200.model import (
    Aurora,
    Aurora12hPretrained,
    AuroraAirPollution,
    AuroraHighRes,
    AuroraPretrained,
    AuroraSmall,
    AuroraSmallPretrained,
    AuroraWave,
)
from aurora_b200.rollout import rollout
from aurora_b200.scorer import EnsembleScorer, Scorer
from aurora_b200.spectra import ZonalSpectra
from aurora_b200.tracker import Tracker

__all__ = [
    "Aurora", "AuroraPretrained", "AuroraSmallPretrained", "AuroraSmall", "Aurora12hPretrained", "AuroraHighRes",
    "AuroraAirPollution", "AuroraWave", "Batch", "Metadata", "rollout",
    "Tracker", "Scorer", "EnsembleScorer", "ZonalSpectra",
]
