"""CPU-side checks of the scorer: the public import, the argument validation of `ab_score_fields` (which needs no GPU
because it happens before any launch), the input checks of `Scorer.step` and the schema of an empty result."""

import ctypes as C
from datetime import timedelta

import numpy as np
import pytest
import torch

from aurora_b200 import cabi
from aurora_b200.batch import Batch, Metadata
from tests import fixtures as fx

FAKE = 0x1000  # a non-null, 16-byte aligned pointer; validation fails before anything could dereference it


def test_public_import():
    from aurora_b200 import Scorer  # noqa: F401

    import aurora_b200

    assert "Scorer" in aurora_b200.__all__


def _field(**kw):
    f = cabi.AbScoreField(pred=FAKE, truth=FAKE, clim=FAKE, h=16, w=32, ld_pred=32, ld_truth=32, ld_clim=32, levels=13,
                          pred_level_stride=512, truth_level_stride=512, clim_level_stride=512)
    for k, v in kw.items():
        setattr(f, k, v)
    return f


def _call(fields, field_bytes=None, weights=FAKE, sums=FAKE, workspace=FAKE, workspace_bytes=1 << 30):
    lib = cabi.lib()
    arr = (cabi.AbScoreField * max(len(fields), 1))(*fields)
    size = C.sizeof(cabi.AbScoreField) if field_bytes is None else field_bytes
    status = lib.ab_score_fields(arr, len(fields), C.c_size_t(size), C.c_void_p(weights), C.c_void_p(sums),
                                 C.c_void_p(workspace), C.c_size_t(workspace_bytes), None)
    return status, lib.ab_last_error().decode()


def test_score_fields_rejects_null_pointers():
    for kw in ({"weights": None}, {"sums": None}, {"workspace": None}):
        status, msg = _call([_field()], **kw)
        assert status == -1 and "null argument" in msg, kw
    for name in ("pred", "truth"):
        status, msg = _call([_field(**{name: None})])
        assert status == -1 and "field 0: null pred or truth" in msg
    lib = cabi.lib()
    assert lib.ab_score_fields(None, 1, C.c_size_t(C.sizeof(cabi.AbScoreField)), C.c_void_p(FAKE), C.c_void_p(FAKE),
                               C.c_void_p(FAKE), C.c_size_t(1 << 30), None) == -1
    assert "null argument" in lib.ab_last_error().decode()


def test_score_fields_checks_the_descriptor_size_and_count():
    status, msg = _call([_field()], field_bytes=C.sizeof(cabi.AbScoreField) - 8)
    assert status == -1 and "sizeof(AbScoreField)" in msg
    status, msg = _call([_field()] * (cabi.AB_SCORE_MAX_FIELDS + 1))
    assert status == -3 and "at most 64" in msg
    status, msg = _call([_field()], field_bytes=0)
    assert status == -1 and "field_bytes 0" in msg
    assert _call([], weights=None, sums=None, workspace=None)[0] == 0  # an empty list is a no-op


def test_score_fields_rejects_bad_extents_and_pitches():
    for kw in ({"h": 0}, {"w": 0}, {"levels": 0}, {"h": -3}):
        status, msg = _call([_field(), _field(**kw)])
        assert status == -1 and "field 1: bad extent" in msg, kw
    for kw in ({"ld_pred": 31}, {"ld_truth": 16}, {"ld_clim": 0}):
        status, msg = _call([_field(**kw)])
        assert status == -1 and "row pitch smaller than the width" in msg, kw
    assert cabi.score_workspace_bytes([_field(clim=None, ld_clim=0)]) > 0  # no climatology: its pitch is unused
    status, msg = _call([_field(truth_level_stride=-512)])
    assert status == -1 and "negative level stride" in msg


def test_score_fields_rejects_a_small_workspace():
    lib = cabi.lib()
    fields = [_field(), _field(h=721, w=1440, ld_pred=1440, ld_truth=1440, ld_clim=1440, levels=1)]
    arr = (cabi.AbScoreField * 2)(*fields)
    need = C.c_size_t()
    assert lib.ab_score_workspace_bytes(arr, 2, C.c_size_t(C.sizeof(cabi.AbScoreField)), C.byref(need)) == 0
    # 13 planes of 16 x 32 are one work item each; 721 rows of 1440 points go in chunks of 11 rows
    assert need.value == (13 + -(-721 // 11)) * 8 * 8
    assert cabi.score_workspace_bytes(fields) == need.value
    status, msg = _call(fields, workspace_bytes=need.value - 1)
    assert status == -1 and f"workspace of {need.value - 1} bytes, {need.value} needed" in msg
    status, msg = _call(fields, sums=FAKE + 4)
    assert status == -1 and "8-byte aligned" in msg
    with pytest.raises(cabi.AbError, match="field 0: bad extent"):
        cabi.score_workspace_bytes([_field(w=0)])


# ---- Scorer.step refusals ---------------------------------------------------------------------------------------------
def _batch(h=16, w=32, b=1, levels=fx.LEVELS4, seed=0):
    return fx.make_batch(fx.CONFIGS["tiny"], h, w, levels=levels, b=b, seed=seed)


def _pred(b=1, levels=fx.LEVELS4):
    """A CPU batch shaped like a prediction: one history slice."""
    x = _batch(b=b, levels=levels)
    one = lambda d: {k: v[:, -1:] for k, v in d.items()}  # noqa: E731
    return Batch(one(x.surf_vars), x.static_vars, one(x.atmos_vars), x.metadata)


def test_step_refuses_cpu_predictions():
    from aurora_b200 import Scorer

    with pytest.raises(cabi.AbError, match="needs the prediction on a CUDA device"):
        Scorer().step(_pred(), _batch(seed=1))


def test_step_refuses_mismatched_times_levels_and_grids():
    from aurora_b200 import Scorer

    pred, sc = _pred(), Scorer()
    late = _batch(seed=1)
    late.metadata = Metadata.derived(late.metadata.lat, late.metadata.lon,
                                     tuple(t + timedelta(hours=6) for t in late.metadata.time), fx.LEVELS4)
    with pytest.raises(ValueError, match="the truth is valid at"):
        sc.step(pred, late)
    with pytest.raises(ValueError, match=r"the truth lacks the pressure levels \[500\]"):
        sc.step(pred, _batch(levels=(100, 250, 850), seed=1))
    shifted = _batch(seed=1)
    shifted.metadata = Metadata(shifted.metadata.lat * 0.5, shifted.metadata.lon, shifted.metadata.time, fx.LEVELS4)
    with pytest.raises(ValueError, match="the truth's latitudes differ"):
        sc.step(pred, shifted)
    with pytest.raises(ValueError, match="the truth has 18 latitudes, the prediction 16"):
        sc.step(pred, _batch(h=18, seed=1))
    with pytest.raises(ValueError, match="the truth's longitudes differ"):
        sc.step(pred, Batch(*_shift_lon(_batch(seed=1))))
    with pytest.raises(ValueError, match="the climatology's latitudes differ"):
        Scorer(climatology=shifted).step(pred, _batch(seed=1))
    with pytest.raises(ValueError, match=r"the truth lacks the variables \['msl'\]"):
        Scorer(variables=("msl",)).step(pred, Batch({}, {}, _batch(seed=1).atmos_vars, _batch(seed=1).metadata))
    with pytest.raises(ValueError, match=r"\['lsm'\] are not surface or atmospheric variables"):
        Scorer(variables=("msl", "lsm")).step(pred, _batch(seed=1))
    with pytest.raises(ValueError, match="the truth has batch size"):
        sc.step(_pred(b=2), Batch(*_times(_batch(seed=1), _pred(b=2))))


def _shift_lon(b):
    md = b.metadata
    return b.surf_vars, b.static_vars, b.atmos_vars, Metadata(md.lat, md.lon + 1.0, md.time, md.atmos_levels)


def _times(b, like):
    md = b.metadata
    return b.surf_vars, b.static_vars, b.atmos_vars, Metadata(md.lat, md.lon, like.metadata.time, md.atmos_levels)


def test_step_refuses_2d_coordinates_and_sharded_bands():
    from aurora_b200 import Scorer

    pred, truth = _pred(), _batch(seed=1)
    lat2, lon2 = torch.meshgrid(pred.metadata.lat, pred.metadata.lon, indexing="ij")
    pred2 = Batch(pred.surf_vars, pred.static_vars, pred.atmos_vars,
                  Metadata.derived(lat2, lon2, pred.metadata.time, pred.metadata.atmos_levels))
    with pytest.raises(ValueError, match="1-D latitudes and longitudes"):
        Scorer().step(pred2, truth)
    truth2 = Batch(truth.surf_vars, truth.static_vars, truth.atmos_vars,
                   Metadata.derived(lat2, lon2, truth.metadata.time, truth.metadata.atmos_levels))
    with pytest.raises(ValueError, match=r"1-D latitudes and longitudes \(the truth's are not\)"):
        Scorer().step(pred, truth2)
    pred.slab_plans = [object()]
    with pytest.raises(ValueError, match="gather the latitude bands first"):
        Scorer().step(pred, truth)


def test_step_refuses_other_dtypes():
    from aurora_b200 import Scorer

    pred, truth = _pred(), _batch(seed=1)
    truth.surf_vars["msl"] = truth.surf_vars["msl"].double()
    with pytest.raises(TypeError, match="needs float32 fields, the truth has torch.float64"):
        Scorer().step(pred, truth)


def test_empty_results_schema():
    from aurora_b200 import Scorer
    from aurora_b200.scorer import COLUMNS

    df = Scorer().results()
    assert tuple(df.columns) == COLUMNS == ("time", "rollout_step", "member", "variable", "level", "rmse", "bias",
                                           "mae", "acc", "count")
    assert len(df) == 0
    assert str(df["time"].dtype) == "datetime64[ns]"
    assert [str(df[c].dtype) for c in ("rollout_step", "member", "count")] == ["int64"] * 3
    assert all(df[c].dtype == np.float64 for c in ("level", "rmse", "bias", "mae", "acc"))
